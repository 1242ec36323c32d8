// merging.cu — MergingPress (reference kvpress/presses/merging_press.py): fold every evicted value into the kept row
// whose key is most cosine-similar, before the evicted rows are dropped. Keys are only gathered.
//
// Per row (b, kv head j) with the kept slots t = 0 .. n_kept-1 (ascending positions) and the evicted slots
// e = 0 .. n_evict-1 (the complement, ascending), include/kvpress_b200.h has the definition:
//   sim(e, t) = K[e].K[t] / (max(|K[e]|, 1e-6) max(|K[t]|, 1e-6)), target(e) = argmax_t (ties and NaN to the lowest t),
//   ok(e) = max_sim >= similarity_threshold, and, when merge_fraction < 1, max_sim >= torch.quantile of the ok
//   similarities (the others at -inf) at q = 1 - merge_fraction,
//   w(e) = clamp(max_sim, 0) ok |V[e]| / (|V[e]| + |V[target]| + 1e-6),
//   V_out[t] = (V[t] + sum w V[e]) / (1 + sum w) over the e with target t in ascending e, where sum w > 0; else V[t].
//
// Four kernels, chained by programmatic dependent launch:
//   1. merging_prologue_kernel: one warp per position. Its slot from a binary search of the kept list; the key row is
//      gathered into a [R][S_pad][Dp] workspace (kept slots first, then evicted slots) with zero columns up to Dp (a
//      multiple of 64), with the inverse clamped key norm and the value norm next to it.
//   2. merging_argmax_kernel: persistent, one CTA per SM, a TMA producer and two wgmma consumer warpgroups. An item is
//      128 evicted rows of one row, resident as the A operand (64 rows per consumer). The kept keys stream through a
//      TMA ring in 128-row tiles; each tile is one m64n128 product per consumer, scaled by the columns' inverse norms
//      and folded into a running (max, argmax) per row in ascending column order. Only target and max_sim leave the SM.
//   3. merging_plan_kernel: one CTA per row. The gate threshold by an exact radix select of two order statistics over
//      order-preserving 32-bit keys (four 8-bit passes, as select_compact.cu ranks 16-bit keys in two), the weights,
//      then a stable counting sort of the evicted slots by target: counts, exclusive offsets, and 1024-slot chunks in
//      ascending e, each sorted by (target, e) in shared memory so each target's run takes its offset in one step.
//   4. merging_merge_kernel: one warp per kept slot sums its contributions in that order and writes V_out.
// No float atomics anywhere: two calls are bitwise equal and a row's result does not depend on the batch it is in.
#include <limits.h>
#include <math.h>

#include <algorithm>

#include "qk_tiles.cuh"

namespace kvp {

constexpr int kMgThreads = 256;     // prologue and merge kernels: one warp per position / kept slot
constexpr int kMgPlanThreads = 1024;
constexpr float kMgEps = 1e-6f;

// The scratch in ws.scorer; every per-row array has row stride S_pad. Slots [0, n_kept) are the kept rows and
// [n_kept, S) the evicted rows, so its size does not depend on n_kept.
struct MgScratch {
    uint16_t* keys;  // [R][S_pad][Dp] gathered keys, zero columns past D
    float* inv;      // [R][S_pad] 1 / max(|K|, 1e-6) by slot
    float* vnorm;    // [R][S_pad] |V| by slot
    int32_t* pos;    // [R][S_pad] evicted slot e -> position
    int32_t* target; // [R][S_pad] evicted slot e -> kept slot
    float* sim;      // [R][S_pad] evicted slot e -> max_sim
    float* weight;   // [R][S_pad] evicted slot e -> w
    int32_t* end;    // [R][S_pad] kept slot t -> counts, then offsets, then the end of its contributions in perm
    int32_t* perm;   // [R][S_pad] evicted slots grouped by target, ascending within a target
    int32_t* kept;   // [R][S_pad] kept positions when the caller's idx_out is null (compress)
};

static int mg_dp(int D) { return (D + 63) / 64 * 64; }

static MgScratch carve_mg(const Dims& d, void* base, size_t* bytes = nullptr) {
    const size_t S_pad = (size_t)(d.S + kTile - 1) / kTile * kTile, n = (size_t)d.R * S_pad;
    Carve c(base);
    MgScratch s;
    s.keys = c.take<uint16_t>(n * mg_dp(d.D));
    s.inv = c.take<float>(n);
    s.vnorm = c.take<float>(n);
    s.pos = c.take<int32_t>(n);
    s.target = c.take<int32_t>(n);
    s.sim = c.take<float>(n);
    s.weight = c.take<float>(n);
    s.end = c.take<int32_t>(n);
    s.perm = c.take<int32_t>(n);
    s.kept = c.take<int32_t>(n);
    if (bytes) *bytes = c.bytes;
    return s;
}

size_t merging_scratch_bytes(const Dims& d) {
    size_t bytes;
    carve_mg(d, nullptr, &bytes);
    return bytes;
}

int32_t* merging_scratch_kept(const Dims& d, const Workspace& ws) { return carve_mg(d, ws.scorer).kept; }

struct MgArgs {
    const void* K;
    const void* V;
    Strides3 ks, vs;
    const int32_t* kept;  // [R][n_kept] ascending positions
    int H, S, S_pad, D, Dp, n_kept;
    MgScratch sc;
};

// ---- 1. prologue ------------------------------------------------------------------------------------------------------
// Sum of x over a warp by an xor butterfly (every lane gets it).
__device__ __forceinline__ float mg_warp_sum(float x) {
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) x += __shfl_xor_sync(0xFFFFFFFFu, x, o);
    return x;
}

// Sum of squares of the 8 elements of a 16-byte piece: two interleaved FMA chains.
template <typename T>
__device__ __forceinline__ float mg_sq8(const int4& v) {
    const uint32_t w[4] = {(uint32_t)v.x, (uint32_t)v.y, (uint32_t)v.z, (uint32_t)v.w};
    float f0 = 0.f, f1 = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float2 f = F16Traits<T>::unpack2(w[j]);
        f0 = fmaf(f.x, f.x, f0);
        f1 = fmaf(f.y, f.y, f1);
    }
    return f0 + f1;
}

template <typename T>
__global__ void __launch_bounds__(kMgThreads) merging_prologue_kernel(MgArgs a) {
    pdl_launch_dependents();
    pdl_wait();  // the kept list of a compress comes from the selection kernel
    const int lane = threadIdx.x & 31;
    const int s = blockIdx.x * (kMgThreads / 32) + (threadIdx.x >> 5), row = blockIdx.y;
    if (s >= a.S) return;
    const int b = row / a.H, h = row % a.H;
    // kept positions below s: the first index whose position is >= s
    const int32_t* kept = a.kept + (size_t)row * a.n_kept;
    int lo = 0, hi = a.n_kept;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(kept + mid) < s) lo = mid + 1;
        else hi = mid;
    }
    const bool is_kept = lo < a.n_kept && __ldg(kept + lo) == s;
    const int e = s - lo;
    const size_t slot = (size_t)row * a.S_pad + (is_kept ? lo : a.n_kept + e);
    const int nvec = a.D >> 3;
    const T* k = static_cast<const T*>(a.K) + (int64_t)b * a.ks.b + (int64_t)h * a.ks.h + (int64_t)s * a.ks.s;
    const T* v = static_cast<const T*>(a.V) + (int64_t)b * a.vs.b + (int64_t)h * a.vs.h + (int64_t)s * a.vs.s;
    int4 kv4 = make_int4(0, 0, 0, 0), vv4 = make_int4(0, 0, 0, 0);
    if (lane < nvec) {
        kv4 = ldg_plain(k + lane * 8);
        vv4 = ldg_plain(v + lane * 8);
    }
    if (lane < (a.Dp >> 3)) reinterpret_cast<int4*>(a.sc.keys + slot * a.Dp)[lane] = kv4;
    const float kss = mg_warp_sum(mg_sq8<T>(kv4)), vss = mg_warp_sum(mg_sq8<T>(vv4));
    if (lane == 0) {
        float kn = sqrtf(kss);
        kn = kn < kMgEps ? kMgEps : kn;  // clamp(min=1e-6); NaN stays NaN
        a.sc.inv[slot] = 1.f / kn;
        a.sc.vnorm[slot] = sqrtf(vss);
        if (!is_kept) a.sc.pos[(size_t)row * a.S_pad + e] = s;
    }
}

// ---- 2. similarity argmax -----------------------------------------------------------------------------------------------
// (v, c) is a better candidate than (bv, bc): NaN first, then the larger value, then the lower column.
__device__ __forceinline__ bool mg_better(float v, int c, float bv, int bc) {
    if (bv != bv) return v != v && c < bc;
    if (v != v) return true;
    return v > bv || (v == bv && c < bc);
}

template <typename T, int DP>
__global__ void __launch_bounds__(umma::kTmaCtaThreads, 1)
merging_argmax_kernel(const __grid_constant__ CUtensorMap mapE, const __grid_constant__ CUtensorMap mapT, int S_pad,
                      int n_kept, int n_evict, int R, MgScratch sc) {
    using L = SnSmem<DP, 128>;  // resident: 128 evicted rows; ring: 128 kept rows per stage
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* smem = umma::smem_align_1024(smem_raw);
    unsigned char* s_a = smem + L::kQOff;
    unsigned char* s_stage = smem + L::kStageOff;
    auto* b_ring = reinterpret_cast<umma::TmaRing<L::kStages>*>(smem + L::kBarOff);
    auto* a_ring = reinterpret_cast<umma::TmaRing<1>*>(b_ring + 1);  // the resident evicted block

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
    if (tid == 0) {
        umma::prefetch_tmap(&mapE);
        umma::prefetch_tmap(&mapT);
        b_ring->init(umma::kTmaConsumerWarps);
        a_ring->init(umma::kTmaConsumerWarps);
        umma::mbar_fence_init();
    }
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();  // the gathered keys and norms come from the prologue

    const int n_blocks = (n_evict + 127) / 128, n_tiles = (n_kept + kSnTile - 1) / kSnTile;
    const int n_items = R * n_blocks;
    if (wg == 0) {
        if (tid == 0) {
            // ===== TMA producer =====
            uint32_t b_it = 0, a_it = 0;
            for (int u = blockIdx.x; u < n_items; u += gridDim.x, ++a_it) {
                const int row = u / n_blocks, blk = u % n_blocks;
                a_ring->acquire(a_it, L::kQBytes);  // rows past n_evict read as zero
                for (int kp = 0; kp < L::kPanels; ++kp)
                    umma::tma_load_3d(s_a + kp * L::kQPanel, &mapE, a_ring->full(0), kp * 64, blk * 128, row);
                for (int t = 0; t < n_tiles; ++t, ++b_it) {
                    const int stage = b_ring->acquire(b_it, L::kStageBytes);  // rows past n_kept read as zero
                    for (int kp = 0; kp < L::kPanels; ++kp)
                        umma::tma_load_3d(s_stage + stage * L::kStageBytes + kp * kSnTile * 128, &mapT,
                                          b_ring->full(stage), kp * 64, t * kSnTile, row);
                }
            }
        }
    } else {
        // ===== consumers: warpgroup cw owns evicted rows 64 cw .. 64 cw + 63 of the item =====
        const int cw = wg - 1, w4 = warp & 3, qd = lane & 3;
        uint32_t b_it = 0, a_it = 0;
        for (int u = blockIdx.x; u < n_items; u += gridDim.x, ++a_it) {
            const int row = u / n_blocks, blk = u % n_blocks;
            const float* inv_kept = sc.inv + (size_t)row * S_pad;
            float bv[2] = {-INFINITY, -INFINITY};
            int bc[2] = {INT_MAX, INT_MAX};
            a_ring->wait(a_it);
            const uint32_t abase = umma::smem_u32(s_a) + cw * 64 * 128;
#pragma unroll 1
            for (int t = 0; t < n_tiles; ++t, ++b_it) {
                const int stage = b_ring->wait(b_it);
                float acc[64];
                snap_mma<T, DP>(acc, abase, L::kQPanel, umma::smem_u32(s_stage + stage * L::kStageBytes),
                                kSnTile * 128);
                b_ring->release(stage);  // the product has completed
                // columns 8 jj + 2 qd + {0, 1} of the tile, ascending per thread
#pragma unroll
                for (int jj = 0; jj < 16; ++jj) {
                    const int c = t * kSnTile + 8 * jj + 2 * qd;
                    const float2 ic = *reinterpret_cast<const float2*>(inv_kept + c);
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        if (c < n_kept) {
                            const float v = acc[4 * jj + 2 * hh] * ic.x;
                            if (mg_better(v, c, bv[hh], bc[hh])) bv[hh] = v, bc[hh] = c;
                        }
                        if (c + 1 < n_kept) {
                            const float v = acc[4 * jj + 2 * hh + 1] * ic.y;
                            if (mg_better(v, c + 1, bv[hh], bc[hh])) bv[hh] = v, bc[hh] = c + 1;
                        }
                    }
                }
            }
            a_ring->release(0);  // every product on the block has completed
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                float v = bv[hh];
                int c = bc[hh];
#pragma unroll
                for (int o = 1; o <= 2; o <<= 1) {  // the four threads of a row
                    const float v2 = __shfl_xor_sync(0xFFFFFFFFu, v, o);
                    const int c2 = __shfl_xor_sync(0xFFFFFFFFu, c, o);
                    if (mg_better(v2, c2, v, c)) v = v2, c = c2;
                }
                const int e = blk * 128 + cw * 64 + w4 * 16 + (lane >> 2) + 8 * hh;
                if (qd == 0 && e < n_evict) {
                    const size_t i = (size_t)row * S_pad + e;
                    sc.target[i] = c;
                    sc.sim[i] = v * sc.inv[(size_t)row * S_pad + n_kept + e];  // the row's positive scale keeps the order
                }
            }
        }
    }
}

// ---- 3. gate, weights and the stable counting sort --------------------------------------------------------------------
// ordered_f32, except that -0 and +0 share a key
__device__ __forceinline__ uint32_t mg_key32(float f) {
    return ordered_f32(__float_as_uint(f) == 0x80000000u ? 0.f : f);
}

struct MgPlanArgs {
    int S_pad, n_kept, n_evict;
    float threshold;
    float q;  // 1 - merge_fraction rounded to fp32; 0 when merge_fraction == 1 (no fraction gate)
    bool fraction;
    MgScratch sc;
    int32_t* target_out;  // [R][n_evict] or null
    float* sim_out;
};

// The gate's input of slot e: max_sim where it passes the threshold, -inf elsewhere (NaN never passes).
__device__ __forceinline__ uint32_t mg_gate_key(const float* sim, int e, float threshold) {
    const float x = sim[e];
    return mg_key32(x >= threshold ? x : -INFINITY);
}

// The k-th smallest (0-based) gate key of the row: four 8-bit radix passes over 256-bin shared histograms.
__device__ uint32_t mg_select(const float* sim, int n, float threshold, uint32_t k, uint32_t* hist, uint32_t* bc) {
    const int tid = threadIdx.x;
    uint32_t prefix = 0, mask = 0;
#pragma unroll 1
    for (int shift = 24; shift >= 0; shift -= 8) {
        if (tid < 256) hist[tid] = 0;
        __syncthreads();
        for (int e = tid; e < n; e += kMgPlanThreads) {
            const uint32_t key = mg_gate_key(sim, e, threshold);
            if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (tid < 32) {  // ascending bins: the bin where the running count passes k
            uint32_t h[8], sum = 0;
#pragma unroll
            for (int i = 0; i < 8; ++i) sum += (h[i] = hist[8 * tid + i]);
            uint32_t incl = sum;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t x = __shfl_up_sync(0xFFFFFFFFu, incl, o);
                if (tid >= o) incl += x;
            }
            const unsigned hit = __ballot_sync(0xFFFFFFFFu, incl > k);
            const int first = __ffs(hit) - 1;
            if (tid == first) {
                uint32_t run = incl - sum;
                int bin = 8 * tid + 7;
                for (int i = 0; i < 8; ++i) {
                    if (run + h[i] > k) {
                        bin = 8 * tid + i;
                        break;
                    }
                    run += h[i];
                }
                bc[0] = (uint32_t)bin;
                bc[1] = run;
            }
        }
        __syncthreads();
        prefix |= bc[0] << shift;
        mask |= 255u << shift;
        k -= bc[1];
        __syncthreads();  // bc is rewritten by the next pass
    }
    return prefix;
}

// Inclusive max-scan over the CTA (every thread's value), through `red` [32].
__device__ __forceinline__ int mg_block_max_scan(int x, int* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xFFFFFFFFu, x, o);
        if (lane >= o) x = max(x, y);
    }
    if (lane == 31) red[warp] = x;
    __syncthreads();
    if (warp == 0) {
        int w = red[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xFFFFFFFFu, w, o);
            if (lane >= o) w = max(w, y);
        }
        red[lane] = w;
    }
    __syncthreads();
    const int r = warp > 0 ? max(x, red[warp - 1]) : x;
    __syncthreads();  // red is reused
    return r;
}

// Exclusive sum-scan over the CTA; *total gets the sum. Through `red` [32].
__device__ __forceinline__ int mg_block_excl_sum(int x, int* red, int* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int incl = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xFFFFFFFFu, incl, o);
        if (lane >= o) incl += y;
    }
    if (lane == 31) red[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        int w = red[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xFFFFFFFFu, w, o);
            if (lane >= o) w += y;
        }
        red[lane] = w;
    }
    __syncthreads();
    const int r = incl - x + (warp > 0 ? red[warp - 1] : 0);
    *total = red[31];
    __syncthreads();
    return r;
}

__global__ void __launch_bounds__(kMgPlanThreads) merging_plan_kernel(MgPlanArgs a) {
    __shared__ uint32_t hist[256];
    __shared__ uint32_t bc[2];
    __shared__ int red[32];
    __shared__ unsigned long long skey[kMgPlanThreads];
    __shared__ int sbase[kMgPlanThreads];
    __shared__ float s_thr;
    pdl_launch_dependents();
    pdl_wait();  // target and max_sim come from the argmax kernel
    const int tid = threadIdx.x, row = blockIdx.x;
    const size_t base = (size_t)row * a.S_pad;
    const float* sim = a.sc.sim + base;
    const int32_t* target = a.sc.target + base;
    int32_t* end = a.sc.end + base;
    const int n = a.n_evict;
    for (int t = tid; t < a.n_kept; t += kMgPlanThreads) end[t] = 0;

    // ---- the fraction gate: torch.quantile's two order statistics and its lerp, in fp32 ----
    float thr = -INFINITY;
    if (a.fraction && n > 0) {
        const float rank = a.q * (float)(n - 1);
        const uint32_t lo = min((uint32_t)rank, (uint32_t)(n - 1)), hi = min((uint32_t)ceilf(rank), (uint32_t)(n - 1));
        const float w = rank - (float)lo;
        const uint32_t klo = mg_select(sim, n, a.threshold, lo, hist, bc);
        uint32_t khi = klo;
        if (hi != lo) {  // the next order statistic: klo again if more than hi keys are <= klo, else the next key up
            if (tid == 0) bc[0] = 0, bc[1] = 0xFFFFFFFFu;
            __syncthreads();
            for (int e = tid; e < n; e += kMgPlanThreads) {
                const uint32_t key = mg_gate_key(sim, e, a.threshold);
                if (key <= klo) atomicAdd(&bc[0], 1u);
                else atomicMin(&bc[1], key);
            }
            __syncthreads();
            khi = bc[0] > hi ? klo : bc[1];
        }
        const float below = ordered_f32_to_float(klo), above = ordered_f32_to_float(khi);
        const float diff = above - below;  // -inf - -inf = NaN: no merge in the row, as in torch
        thr = fabsf(w) < 0.5f ? fmaf(w, diff, below) : fmaf(-diff, 1.f - w, above);
    }
    if (tid == 0) s_thr = thr;
    __syncthreads();
    thr = s_thr;

    // ---- weights and counts ----
    const float* vn_kept = a.sc.vnorm + base;
    const float* vn_ev = vn_kept + a.n_kept;
    for (int e = tid; e < n; e += kMgPlanThreads) {
        const float ms = sim[e];
        const int t = target[e];
        const bool ok = ms >= a.threshold && (!a.fraction || ms >= thr);
        float w = ms != ms ? ms : fmaxf(ms, 0.f);  // clamp(min=0) keeps NaN
        w = w * (ok ? 1.f : 0.f);
        const float en = vn_ev[e];
        w = __fdiv_rn(__fmul_rn(w, en), __fadd_rn(__fadd_rn(en, vn_kept[t]), kMgEps));
        a.sc.weight[base + e] = w;
        if (a.target_out) a.target_out[(size_t)row * n + e] = t;
        if (a.sim_out) a.sim_out[(size_t)row * n + e] = ms;
        atomicAdd(&end[t], 1);  // integer counts: exact in any order
    }
    __syncthreads();

    // ---- exclusive offsets over the kept slots ----
    int carry = 0;
    for (int t0 = 0; t0 < a.n_kept; t0 += kMgPlanThreads) {
        const int t = t0 + tid;
        const int c = t < a.n_kept ? end[t] : 0;
        int total;
        const int off = mg_block_excl_sum(c, red, &total);
        if (t < a.n_kept) end[t] = carry + off;
        carry += total;
    }
    __syncthreads();

    // ---- stable placement, 1024 evicted slots at a time in ascending e ----
    int32_t* perm = a.sc.perm + base;
    for (int e0 = 0; e0 < n; e0 += kMgPlanThreads) {
        const int e = e0 + tid;
        skey[tid] = e < n ? ((unsigned long long)(uint32_t)target[e] << 32) | (uint32_t)tid : ~0ull;
        __syncthreads();
        for (int k = 2; k <= kMgPlanThreads; k <<= 1) {  // bitonic sort of the chunk by (target, e)
            for (int j = k >> 1; j > 0; j >>= 1) {
                const int ixj = tid ^ j;
                if (ixj > tid) {
                    const unsigned long long x = skey[tid], y = skey[ixj];
                    if (((tid & k) == 0) == (x > y)) skey[tid] = y, skey[ixj] = x;
                }
                __syncthreads();
            }
        }
        const unsigned long long key = skey[tid];
        const bool valid = key != ~0ull;
        const uint32_t t = (uint32_t)(key >> 32);
        const bool first = tid == 0 || (uint32_t)(skey[tid - 1] >> 32) != t;
        const bool last = tid == kMgPlanThreads - 1 || skey[tid + 1] == ~0ull || (uint32_t)(skey[tid + 1] >> 32) != t;
        const int start = mg_block_max_scan(first ? tid : 0, red);
        if (valid && last) {  // one thread per target of the chunk: its run takes the next places of the target
            const int at = end[t];
            end[t] = at + (tid - start + 1);
            sbase[start] = at;
        }
        __syncthreads();
        if (valid) perm[sbase[start] + (tid - start)] = e0 + (int)(uint32_t)key;
        __syncthreads();  // skey and sbase are reused
    }
}

// ---- 4. merge ----------------------------------------------------------------------------------------------------------
struct MgMergeArgs {
    const void* V;
    Strides3 vs;
    const int32_t* kept;
    void* V_out;  // contiguous [R][n_kept][D]
    int H, S_pad, D, n_kept;
    MgScratch sc;
};

template <typename T>
__device__ __forceinline__ void mg_unpack8(const int4& v, float (&f)[8]) {
    const uint32_t w[4] = {(uint32_t)v.x, (uint32_t)v.y, (uint32_t)v.z, (uint32_t)v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float2 p = F16Traits<T>::unpack2(w[j]);
        f[2 * j] = p.x;
        f[2 * j + 1] = p.y;
    }
}

template <typename T>
__global__ void __launch_bounds__(kMgThreads) merging_merge_kernel(MgMergeArgs a) {
    pdl_wait();  // weights and the placement come from the plan kernel
    const int lane = threadIdx.x & 31;
    const int t = blockIdx.x * (kMgThreads / 32) + (threadIdx.x >> 5), row = blockIdx.y;
    if (t >= a.n_kept) return;
    const int b = row / a.H, h = row % a.H;
    const size_t base = (size_t)row * a.S_pad;
    const T* Vrow = static_cast<const T*>(a.V) + (int64_t)b * a.vs.b + (int64_t)h * a.vs.h;
    const bool mine = lane < (a.D >> 3);
    const int begin = t > 0 ? a.sc.end[base + t - 1] : 0, stop = a.sc.end[base + t];
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, accw = 0.f;
    constexpr int kAhead = 4;  // value rows in flight
#pragma unroll 1
    for (int p0 = begin; p0 < stop; p0 += 32) {
        // 32 contributions' slot, weight and position, one per lane, then broadcast in order
        const int my = p0 + lane;
        int e = 0, pos = 0;
        float w = 0.f;
        if (my < stop) {
            e = a.sc.perm[base + my];
            w = a.sc.weight[base + e];
            pos = a.sc.pos[base + e];
        }
        const int cnt = min(32, stop - p0);
#pragma unroll 1
        for (int i0 = 0; i0 < cnt; i0 += kAhead) {
            int4 v4[kAhead];
            float wi[kAhead];
#pragma unroll
            for (int u = 0; u < kAhead; ++u) {
                const int src = min(i0 + u, 31);
                const int ps = __shfl_sync(0xFFFFFFFFu, pos, src);
                wi[u] = __shfl_sync(0xFFFFFFFFu, w, src);
                v4[u] = make_int4(0, 0, 0, 0);
                if (mine && i0 + u < cnt) v4[u] = ldg_plain(Vrow + (int64_t)ps * a.vs.s + lane * 8);
            }
#pragma unroll
            for (int u = 0; u < kAhead; ++u) {
                if (i0 + u >= cnt) break;
                float f[8];
                mg_unpack8<T>(v4[u], f);
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[j] = __fadd_rn(acc[j], __fmul_rn(wi[u], f[j]));
                accw = __fadd_rn(accw, wi[u]);
            }
        }
    }
    if (!mine) return;
    const int kp = a.kept[(size_t)row * a.n_kept + t];
    const int4 kv = ldg_plain(Vrow + (int64_t)kp * a.vs.s + lane * 8);
    int4 out = kv;
    if (accw > 0.f) {
        float f[8];
        mg_unpack8<T>(kv, f);
        const float den = __fadd_rn(1.f, accw);
        uint32_t w[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint16_t lo = F16Traits<T>::from_float(__fdiv_rn(__fadd_rn(f[2 * j], acc[2 * j]), den));
            const uint16_t hi = F16Traits<T>::from_float(__fdiv_rn(__fadd_rn(f[2 * j + 1], acc[2 * j + 1]), den));
            w[j] = (uint32_t)lo | ((uint32_t)hi << 16);
        }
        out = make_int4((int)w[0], (int)w[1], (int)w[2], (int)w[3]);
    }
    reinterpret_cast<int4*>(static_cast<T*>(a.V_out) + ((size_t)row * a.n_kept + t) * a.D)[lane] = out;
}

// ---- host launcher ------------------------------------------------------------------------------------------------------
template <typename T, int DP>
static cudaError_t launch_mg_argmax(const Dims& d, const MgScratch& sc, int S_pad, cudaStream_t st) {
    using L = SnSmem<DP, 128>;
    const int n_evict = d.S - d.n_kept;
    const int n_items = d.R * ((n_evict + 127) / 128);
    const int grid = std::min(device_sm_count(), n_items);
    CUtensorMap mapE, mapT;
    cudaError_t e;
    const uint64_t head_stride = (uint64_t)S_pad * DP;
    if ((e = make_tmap_rows(&mapE, sc.keys + (size_t)d.n_kept * DP, DP, n_evict, DP, d.R, head_stride, 128)) !=
        cudaSuccess)
        return e;
    if ((e = make_tmap_rows(&mapT, sc.keys, DP, d.n_kept, DP, d.R, head_stride, 128)) != cudaSuccess) return e;
    constexpr int smem = umma::smem_request(L::kTotal);
    constexpr auto k = merging_argmax_kernel<T, DP>;
    if ((e = ensure_dynamic_smem<k>(smem)) != cudaSuccess) return e;
    return launch_pdl(k, dim3(grid), dim3(umma::kTmaCtaThreads), smem, st, mapE, mapT, S_pad, d.n_kept, n_evict, d.R,
                      sc);
}

template <typename T>
static cudaError_t launch_mg_t(const Dims& d, const void* K, const void* V, const int32_t* kept, float threshold,
                               double merge_fraction, void* V_out, int32_t* target_out, float* sim_out,
                               const Workspace& ws, cudaStream_t st) {
    if (d.n_kept == 0) return cudaSuccess;  // nothing is kept: nothing to write
    const MgScratch sc = carve_mg(d, ws.scorer);
    const int Dp = mg_dp(d.D), n_evict = d.S - d.n_kept;
    MgArgs a = {K, V, d.ks, d.vs, kept, d.H, d.S, ws.S_pad, d.D, Dp, d.n_kept, sc};
    cudaError_t e = launch_pdl(merging_prologue_kernel<T>, dim3((d.S + 7) / 8, d.R), dim3(kMgThreads), 0, st, a);
    if (e != cudaSuccess) return e;
    if (n_evict > 0) {
        if (Dp == 64) e = launch_mg_argmax<T, 64>(d, sc, ws.S_pad, st);
        else if (Dp == 128) e = launch_mg_argmax<T, 128>(d, sc, ws.S_pad, st);
        else if (Dp == 192) e = launch_mg_argmax<T, 192>(d, sc, ws.S_pad, st);
        else e = launch_mg_argmax<T, 256>(d, sc, ws.S_pad, st);
        if (e != cudaSuccess) return e;
    }
    MgPlanArgs pa = {ws.S_pad, d.n_kept, n_evict, threshold, (float)(1.0 - merge_fraction), merge_fraction < 1.0, sc,
                     target_out, sim_out};
    if ((e = launch_pdl(merging_plan_kernel, dim3(d.R), dim3(kMgPlanThreads), 0, st, pa)) != cudaSuccess) return e;
    MgMergeArgs ma = {V, d.vs, kept, V_out, d.H, ws.S_pad, d.D, d.n_kept, sc};
    return launch_pdl(merging_merge_kernel<T>, dim3((d.n_kept + 7) / 8, d.R), dim3(kMgThreads), 0, st, ma);
}

cudaError_t launch_merging(const Dims& d, int dtype, const void* K, const void* V, const int32_t* kept, float threshold,
                           double merge_fraction, void* V_out, int32_t* target_out, float* sim_out, const Workspace& ws,
                           cudaStream_t st) {
    return with_dtype(dtype, [&](auto t) {
        return launch_mg_t<decltype(t)>(d, K, V, kept, threshold, merge_fraction, V_out, target_out, sim_out, ws, st);
    });
}

}  // namespace kvp
