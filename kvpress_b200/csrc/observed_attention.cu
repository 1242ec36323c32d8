// observed_attention.cu — stage S for ObservedAttentionPress (sm_90a: TMA + wgmma).
//
// Reference semantics (kvpress/presses/observed_attention_press.py, the H2O score), per (b, kv head j, key s), with
// G = Hq / Hkv, the query heads h = j G + g of kv head j and the n_q query rows i of the current forward at positions
// p_i = S - n_q + i:
//     y[h, i, s]  = scaling * q[h, i] . k[j, s]        if s <= p_i, else -inf                (causal)
//     P[h, i, :]  = softmax_s(y[h, i, :])              (exact normaliser over the whole row)
//     score(s)    = (1/G) sum_g sum_i P[h, i, s] / c(S - s)
// where c(n) is n rounded to the cache dtype, as the reference divides by torch.arange(S, 0, -1) cast to the
// attention dtype: in bf16 counts above 256 round, in fp16 counts >= 65520 become inf and those positions score 0.
// The reference reduces the [B, Hq, S, S] weights an eager attention forward materialises; here they never exist:
//   pass 1 (obs_stats_kernel)  item = (b, j, block of qpos query positions), the G heads' rows resident in shared memory
//          ([G qpos rows, padded to 128 / 256 / 512] x D); K tiles stream from 0 to the block's diagonal, only the
//          diagonal tiles are masked; every row keeps an online (max, sum exp2). Out: cb = -(m + log2 Z) per query row.
//   pass 2 (obs_colsum_kernel) item = (b, j, 128-key tile), the K tile resident; the 128-row Q chunks of the G heads
//          from the tile's diagonal to n_q stream through a TMA ring; each key sums exp2(c y + cb) = P over all rows
//          in registers. Only the first chunk of each head is masked. No atomics.
//   finalize (obs_finalize_kernel): / (G c(S - s)), ONE rounding to the cache dtype, keys + histogram for selection.
// Both MMA kernels are persistent (one CTA per SM) with one TMA producer thread and two wgmma consumer warpgroups.
// The work of an item grows (pass 1) or shrinks (pass 2) linearly along the sequence: items are enumerated in order of
// non-increasing work and dealt round-robin to the CTAs, which bounds every CTA's load by the mean plus one item
// (obs_stats_item / obs_colsum_item; restated by tests/test_observed_attention_host.py). One CTA owns each item, so
// the summation order depends only on the shape and two calls give bitwise-equal scores.
#include <algorithm>

#include "qk_tiles.cuh"

namespace kvp {

struct ObsScratch {
    float* cb;      // [B Hq][n_q]  -(max + log2 sum) of every query row, log2 units
    float* colsum;  // [R][S_pad]   sum over the query rows of the group of P[., s]
};

// The scratch in ws.scorer for n_q query rows; with a null base only its size (*bytes).
static ObsScratch carve_obs(const Dims& d, int n_q, void* base, size_t* bytes = nullptr) {
    const size_t S_pad = (size_t)((d.S + kTile - 1) / kTile) * kTile;
    Carve c(base);
    ObsScratch s;
    s.cb = c.take<float>((size_t)d.B * d.Hq * n_q);
    s.colsum = c.take<float>((size_t)d.R * S_pad);
    if (bytes) *bytes = c.bytes;
    return s;
}

size_t observed_attention_scratch_bytes(const Dims& d, int n_q) {
    size_t bytes;
    carve_obs(d, n_q, nullptr, &bytes);
    return bytes;
}

// ---- schedule (host and device) ----------------------------------------------------------------------------------
// Pass 1: query positions per item (G heads x obs_qpos(G) rows resident, qk_tiles.cuh), items = R * ceil(n_q / qpos).
// Item u is the block qb = n_blocks - 1 - u / R of row u % R: later blocks see more keys, so the work (K tiles,
// obs_stats_tiles) never increases with u.
// Pass 2: items = R * ceil(S / 128). Item u is the key tile kt = u / R of row u % R; its query rows start at
// i_min = max(0, 128 kt - (S - n_q)), so its work (G x Q chunks) never increases with u.
__host__ __device__ inline int obs_colsum_imin(int S, int n_q, int kt) { return max(0, kt * kSnTile - (S - n_q)); }
__host__ __device__ inline int obs_colsum_chunks(int S, int n_q, int kt) {
    return (n_q - obs_colsum_imin(S, n_q, kt) + kSnTile - 1) / kSnTile;
}

// Pass 2 layout: one resident K tile [128 x D], a ring of 128-row Q chunks.
template <int D>
struct ObsColSmem {
    static constexpr int kPanels = D / 64;
    static constexpr int kTileBytes = kPanels * kSnTile * 128;  // a K tile or a Q chunk
    static constexpr int kPanel = kSnTile * 128;                // bytes of one 64-column panel of either
    static constexpr int kStages = umma::ring_stages(kTileBytes + 256, kTileBytes);
    static constexpr int kKOff = 0;
    static constexpr int kStageOff = kTileBytes;
    static constexpr int kBarOff = kStageOff + kStages * kTileBytes;
    static constexpr int kTotal = kBarOff + 256;
    static_assert(umma::smem_request(kTotal) <= umma::kSmemBudget, "shared memory budget");
};

// ---- pass 1: per-query-row softmax normalisers --------------------------------------------------------------------
// Resident row r = g qpos + i is query position p0 + i of head j G + g (rows of padding heads, g >= G, are computed
// and ignored). Consumer warpgroup cw computes D[qrow, key] for the 64-row blocks mb = cw, cw + 2, ... against every K
// tile; a thread holds rows (16 w + l/4, +8) of a block and 32 of the 128 keys, keeps an online (max, sum exp2) per
// row, and the four threads that share a row merge theirs at the end of the item.
template <typename T, int D, int NQP>
__global__ void __launch_bounds__(umma::kTmaCtaThreads, 1)
obs_stats_kernel(const __grid_constant__ CUtensorMap mapK, const __grid_constant__ CUtensorMap mapQ, int H, int G,
                 int S, int n_q, int qpos, int R, int n_blocks, float c, ObsScratch sc) {
    using L = SnSmem<D, NQP>;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* smem = umma::smem_align_1024(smem_raw);
    unsigned char* s_q = smem + L::kQOff;
    unsigned char* s_stage = smem + L::kStageOff;
    auto* k_ring = reinterpret_cast<umma::TmaRing<L::kStages>*>(smem + L::kBarOff);
    uint64_t* q_full = reinterpret_cast<uint64_t*>(k_ring + 1);

    constexpr int kMyBlocks = NQP / 128;  // 64-row blocks of Q per consumer warpgroup
    const int NQ = G * qpos;
    const int off = S - n_q;  // position of query row 0
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;

    if (tid == 0) {
        umma::prefetch_tmap(&mapK);
        umma::prefetch_tmap(&mapQ);
        k_ring->init(umma::kTmaConsumerWarps);
        umma::mbar_init(q_full, 1);
        umma::mbar_fence_init();
    }
    __syncthreads();

    const int n_items = R * n_blocks;
    uint32_t k_it = 0, q_it = 0;
    for (int u = blockIdx.x; u < n_items; u += gridDim.x) {
        const int qb = n_blocks - 1 - u / R, row = u % R;
        const int b = row / H, j = row % H;
        const int p0 = qb * qpos;
        const int n_tiles = obs_stats_tiles(S, n_q, p0, qpos);
        __syncthreads();  // previous item fully consumed: s_q reusable

        if (wg == 0) {
            if (tid == 0) {
                // rows past n_q read as zero; rows of padding heads are not loaded
                umma::mbar_arrive_expect_tx(q_full, (uint32_t)(G * L::kPanels * qpos * 128));
                for (int g = 0; g < G; ++g)
                    for (int kp = 0; kp < L::kPanels; ++kp)
                        umma::tma_load_3d(s_q + kp * L::kQPanel + g * qpos * 128, &mapQ, q_full, kp * 64, p0,
                                          (b * H + j) * G + g);
                for (int t = 0; t < n_tiles; ++t, ++k_it) {
                    const int stage = k_ring->acquire(k_it, L::kStageBytes);
                    for (int kp = 0; kp < L::kPanels; ++kp)
                        umma::tma_load_4d(s_stage + stage * L::kStageBytes + kp * (kSnTile * 128), &mapK,
                                          k_ring->full(stage), kp * 64, t * kSnTile, j, b);
                }
            }
        } else {
            const int cw = wg - 1, w4 = warp & 3, qd = lane & 3;
            float run_m[kMyBlocks][2], run_z[kMyBlocks][2];
#pragma unroll
            for (int i = 0; i < kMyBlocks; ++i)
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    run_m[i][hh] = -INFINITY;
                    run_z[i][hh] = 0.f;
                }
            umma::mbar_wait(q_full, q_it & 1);
            for (int t = 0; t < n_tiles; ++t, ++k_it) {
                const int stage = k_ring->wait(k_it);
                const uint32_t kb = umma::smem_u32(s_stage + stage * L::kStageBytes);
                const int key0 = t * kSnTile + 2 * qd;
                const bool interior = (t + 1) * kSnTile <= off + p0 + 1;  // every key visible to every row
#pragma unroll
                for (int i = 0; i < kMyBlocks; ++i) {
                    const int mb = 2 * i + cw;
                    if (mb * 64 >= NQ) continue;  // warpgroup-uniform
                    float acc[64];
                    snap_mma<T, D>(acc, umma::smem_u32(s_q + mb * 64 * 128), L::kQPanel, kb, kSnTile * 128);
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        const int r = mb * 64 + w4 * 16 + (lane >> 2) + 8 * hh;  // resident row
                        const int limit = off + p0 + r % qpos;                  // last visible key position
                        online_row_update(acc, hh, c, interior, key0, limit, S, run_m[i][hh], run_z[i][hh]);
                    }
                }
                k_ring->release(stage);
            }
            ++q_it;
#pragma unroll
            for (int i = 0; i < kMyBlocks; ++i) {
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    float m = run_m[i][hh], z = run_z[i][hh];
                    quad_merge(m, z, c);
                    const int r = (2 * i + cw) * 64 + w4 * 16 + (lane >> 2) + 8 * hh;
                    const int g = r / qpos, pos = p0 + r % qpos;
                    if (qd == 0 && g < G && pos < n_q)
                        sc.cb[(size_t)((b * H + j) * G + g) * n_q + pos] = -m * c - log2f(z);
                }
            }
        }
    }
}

// ---- pass 2: normalised column sums ---------------------------------------------------------------------------------
// Consumer warpgroup cw computes D[key, qrow] for keys [64 cw, 64 cw + 64) of the resident tile against each streamed
// 128-row Q chunk; a thread holds keys (16 w + l/4, +8) and adds exp2(c y + cb_r) = P[r, key] over its 32 columns. The
// chunks of an item come in (head, chunk) order, each thread adds them in that order into one fp32 sum per key, and
// the four threads that share a key add theirs at the end of the item (xor 1, then xor 2).
template <typename T, int D>
__global__ void __launch_bounds__(umma::kTmaCtaThreads, 1)
obs_colsum_kernel(const __grid_constant__ CUtensorMap mapK, const __grid_constant__ CUtensorMap mapQ, int H, int G,
                  int S, int n_q, int R, int n_ktiles, float c, ObsScratch sc, int S_pad) {
    using L = ObsColSmem<D>;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* smem = umma::smem_align_1024(smem_raw);
    unsigned char* s_k = smem + L::kKOff;
    unsigned char* s_stage = smem + L::kStageOff;
    auto* q_ring = reinterpret_cast<umma::TmaRing<L::kStages>*>(smem + L::kBarOff);
    auto* k_ring = reinterpret_cast<umma::TmaRing<1>*>(q_ring + 1);  // the resident K tile

    const int off = S - n_q;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
    if (tid == 0) {
        umma::prefetch_tmap(&mapK);
        umma::prefetch_tmap(&mapQ);
        q_ring->init(umma::kTmaConsumerWarps);
        k_ring->init(umma::kTmaConsumerWarps);
        umma::mbar_fence_init();
    }
    __syncthreads();

    const int n_items = R * n_ktiles;
    if (wg == 0) {
        if (tid == 0) {
            // ===== TMA producer =====
            uint32_t q_it = 0, k_it = 0;
            for (int u = blockIdx.x; u < n_items; u += gridDim.x, ++k_it) {
                const int kt = u / R, row = u % R;
                const int b = row / H, j = row % H;
                const int i_min = obs_colsum_imin(S, n_q, kt), n_chunks = obs_colsum_chunks(S, n_q, kt);
                k_ring->acquire(k_it, L::kTileBytes);
                for (int kp = 0; kp < L::kPanels; ++kp)
                    umma::tma_load_4d(s_k + kp * L::kPanel, &mapK, k_ring->full(0), kp * 64, kt * kSnTile, j, b);
                for (int g = 0; g < G; ++g)
                    for (int ch = 0; ch < n_chunks; ++ch, ++q_it) {
                        const int stage = q_ring->acquire(q_it, L::kTileBytes);
                        for (int kp = 0; kp < L::kPanels; ++kp)
                            umma::tma_load_3d(s_stage + stage * L::kTileBytes + kp * L::kPanel, &mapQ,
                                              q_ring->full(stage), kp * 64, i_min + ch * kSnTile,
                                              (b * H + j) * G + g);
                    }
            }
        }
    } else {
        // ===== consumers =====
        const int cw = wg - 1, w4 = warp & 3, qd = lane & 3;
        uint32_t q_it = 0, k_it = 0;
        for (int u = blockIdx.x; u < n_items; u += gridDim.x, ++k_it) {
            const int kt = u / R, row = u % R;
            const int b = row / H, j = row % H;
            const int i_min = obs_colsum_imin(S, n_q, kt), n_chunks = obs_colsum_chunks(S, n_q, kt);
            const int key = kt * kSnTile + cw * 64 + w4 * 16 + (lane >> 2);  // and key + 8
            const uint32_t ka = umma::smem_u32(s_k) + cw * 64 * 128;
            k_ring->wait(k_it);
            float tot0 = 0.f, tot1 = 0.f;
            for (int g = 0; g < G; ++g) {
                const float* cb_h = sc.cb + (size_t)((b * H + j) * G + g) * n_q;
                for (int ch = 0; ch < n_chunks; ++ch, ++q_it) {
                    const int i0 = i_min + ch * kSnTile;
                    const int stage = q_ring->wait(q_it);
                    float acc[64];
                    const uint32_t qa = umma::smem_u32(s_stage + stage * L::kTileBytes);
                    umma::wgmma_fence();
#pragma unroll
                    for (int k = 0; k < D / 16; ++k) {
                        const int kp = k >> 2, kk = k & 3;
                        umma::wgmma_ss<128, F16Traits<T>::kMmaFormat>(
                            acc, umma::smem_desc_sw128(ka + kp * L::kPanel + kk * 32),
                            umma::smem_desc_sw128(qa + kp * L::kPanel + kk * 32), k > 0);
                    }
                    umma::wgmma_commit();
                    // the normalisers of the thread's 32 columns load while the MMAs run; rows past n_q add 0
                    float cbx[16], cby[16];
#pragma unroll
                    for (int jj = 0; jj < 16; ++jj) {
                        const int i = i0 + 8 * jj + 2 * qd;
                        cbx[jj] = i < n_q ? __ldg(cb_h + i) : -INFINITY;
                        cby[jj] = i + 1 < n_q ? __ldg(cb_h + i + 1) : -INFINITY;
                    }
                    umma::wgmma_wait_all();
                    q_ring->release(stage);
                    // key s is visible to row i iff s <= off + i, i.e. iff (s - off - i0) <= column; only the first
                    // chunk of a head reaches below the diagonal
                    const int dk0 = ch == 0 ? key - off - i0 : -(1 << 30), dk1 = dk0 + 8;
                    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
                    for (int jj = 0; jj < 16; ++jj) {
                        const int col = 8 * jj + 2 * qd;
                        const float x0 = dk0 > col ? -INFINITY : fmaf(acc[4 * jj], c, cbx[jj]);
                        const float x1 = dk0 > col + 1 ? -INFINITY : fmaf(acc[4 * jj + 1], c, cby[jj]);
                        const float x2 = dk1 > col ? -INFINITY : fmaf(acc[4 * jj + 2], c, cbx[jj]);
                        const float x3 = dk1 > col + 1 ? -INFINITY : fmaf(acc[4 * jj + 3], c, cby[jj]);
                        a0 += fast_exp2(x0);
                        a1 += fast_exp2(x1);
                        a2 += fast_exp2(x2);
                        a3 += fast_exp2(x3);
                    }
                    tot0 += a0 + a1;
                    tot1 += a2 + a3;
                }
            }
            k_ring->release(0);  // every MMA on the K tile has completed
            quad_sum(tot0, tot1);
            if (qd == 0 && key < S) sc.colsum[(size_t)row * S_pad + key] = tot0;
            if (qd == 0 && key + 8 < S) sc.colsum[(size_t)row * S_pad + key + 8] = tot1;
        }
    }
}

// ---- finalize: / (G c(S - s)), ONE rounding, keys + histogram --------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kTileThreads)
obs_finalize_kernel(int S, int G, ObsScratch sc, Workspace ws, uint16_t* __restrict__ scores_out) {
    __shared__ uint16_t skeys[kTile];
    __shared__ uint16_t sscores[kTile];
    __shared__ uint32_t shist[256];
    const int tile = blockIdx.x, row = blockIdx.y, tid = threadIdx.x;
    shist[tid] = 0;
    pdl_launch_dependents();  // the select+compact kernel behind this one may start to take residency
    score_tile_epilogue<T, 1>(skeys, sscores, shist, row, tile * kTile, S, 0, 0, ws, scores_out, nullptr, [&](int, int s) {
        // the reference's divisor, S - s in the cache dtype (fp16: inf from 65520 on, so the score is exactly 0);
        // G times it is exact in fp32
        const float div = F16Traits<T>::to_float(F16Traits<T>::from_float((float)(S - s)));
        return sc.colsum[(size_t)row * ws.S_pad + s] / ((float)G * div);
    });
}

// ---- host launchers -----------------------------------------------------------------------------------------------
// Pass 2 over the key tiles [0, n_ktiles) of every row (see qk_tiles.cuh, launch_attention_colsum).
template <typename T, int D>
static cudaError_t launch_obs_colsum_t(const Dims& d, const void* K, const void* q, int n_q, int n_ktiles, float c,
                                       const float* cb, float* colsum, int S_pad, cudaStream_t st) {
    using L2 = ObsColSmem<D>;
    const int grid2 = (int)std::min<long long>(device_sm_count(), (long long)d.R * n_ktiles);
    if (grid2 == 0) return cudaSuccess;
    CUtensorMap mapK, mapQ2;
    cudaError_t e;
    if ((e = make_tmap_cache(&mapK, K, d, d.ks, kSnTile)) != cudaSuccess) return e;
    const uint64_t n_heads = (uint64_t)d.B * d.Hq, head_stride = (uint64_t)n_q * D;
    if ((e = make_tmap_rows(&mapQ2, q, D, n_q, D, n_heads, head_stride, kSnTile)) != cudaSuccess) return e;
    constexpr int smem2 = umma::smem_request(L2::kTotal);
    constexpr auto k2 = obs_colsum_kernel<T, D>;
    if ((e = ensure_dynamic_smem<k2>(smem2)) != cudaSuccess) return e;
    const ObsScratch sc = {const_cast<float*>(cb), colsum};
    k2<<<grid2, umma::kTmaCtaThreads, smem2, st>>>(mapK, mapQ2, d.H, d.Hq / d.H, d.S, n_q, d.R, n_ktiles, c, sc, S_pad);
    return cudaPeekAtLastError();
}

cudaError_t launch_attention_colsum(const Dims& d, int dtype, const void* K, const void* q, int n_q, int n_ktiles,
                                    float c, const float* cb, float* colsum, int S_pad, cudaStream_t st) {
    return with_dtype(dtype, [&](auto t) -> cudaError_t {
        using T = decltype(t);
        if (d.D == 128) return launch_obs_colsum_t<T, 128>(d, K, q, n_q, n_ktiles, c, cb, colsum, S_pad, st);
        if (d.D == 64) return launch_obs_colsum_t<T, 64>(d, K, q, n_q, n_ktiles, c, cb, colsum, S_pad, st);
        return cudaErrorNotSupported;
    });
}

template <typename T, int D, int NQP>
static cudaError_t launch_obs_t(const Dims& d, const void* K, const void* q, int n_q, float scaling,
                                const Workspace& ws, void* scores_out, cudaStream_t st) {
    using L1 = SnSmem<D, NQP>;
    const int sm_count = device_sm_count();
    const int G = d.Hq / d.H, qpos = obs_qpos(G);
    const ObsScratch sc = carve_obs(d, n_q, ws.scorer);
    const int n_blocks = (n_q + qpos - 1) / qpos;
    const int n_ktiles = (d.S + kSnTile - 1) / kSnTile;
    const int grid1 = (int)std::min<long long>(sm_count, (long long)d.R * n_blocks);
    const float c = kLog2e * scaling;  // logits -> log2 domain

    CUtensorMap mapK, mapQ1;
    cudaError_t e;
    if ((e = make_tmap_cache(&mapK, K, d, d.ks, kSnTile)) != cudaSuccess) return e;
    // q [B Hq, n_q, D] contiguous: rows past n_q of a head read as zero
    const uint64_t n_heads = (uint64_t)d.B * d.Hq, head_stride = (uint64_t)n_q * D;
    if ((e = make_tmap_rows(&mapQ1, q, D, n_q, D, n_heads, head_stride, qpos)) != cudaSuccess) return e;
    constexpr int smem1 = umma::smem_request(L1::kTotal);
    constexpr auto k1 = obs_stats_kernel<T, D, NQP>;
    if ((e = ensure_dynamic_smem<k1>(smem1)) != cudaSuccess) return e;

    k1<<<grid1, umma::kTmaCtaThreads, smem1, st>>>(mapK, mapQ1, d.H, G, d.S, n_q, qpos, d.R, n_blocks, c, sc);
    if ((e = cudaPeekAtLastError()) != cudaSuccess) return e;
    if ((e = launch_obs_colsum_t<T, D>(d, K, q, n_q, n_ktiles, c, sc.cb, sc.colsum, ws.S_pad, st)) != cudaSuccess)
        return e;
    obs_finalize_kernel<T><<<dim3(ws.n_tiles, d.R), kTileThreads, 0, st>>>(d.S, G, sc, ws,
                                                                            static_cast<uint16_t*>(scores_out));
    return cudaPeekAtLastError();
}

template <typename T>
static cudaError_t launch_obs_d(const Dims& d, const void* K, const void* q, int n_q, float scaling,
                                const Workspace& ws, void* scores_out, cudaStream_t st) {
    const int G = d.Hq / d.H;
    // 1 <= G <= 8: the G heads' query blocks (G qpos rows) are padded to 128 / 256 / 512 resident rows
    if (G < 1 || G > 8) return cudaErrorNotSupported;
    const int NQ = G * obs_qpos(G);
    const int NQP = NQ <= 128 ? 128 : (NQ <= 256 ? 256 : 512);
#define KVP_OBS(DD, NN) \
    if (d.D == DD && NQP == NN) return launch_obs_t<T, DD, NN>(d, K, q, n_q, scaling, ws, scores_out, st)
    KVP_OBS(128, 128);
    KVP_OBS(128, 256);
    KVP_OBS(128, 512);
    KVP_OBS(64, 128);
    KVP_OBS(64, 256);
    KVP_OBS(64, 512);
#undef KVP_OBS
    return cudaErrorNotSupported;
}

cudaError_t launch_observed_attention_score(const Dims& d, int dtype, const void* K, const void* q, int n_q,
                                            float scaling, const Workspace& ws, void* scores_out, cudaStream_t st) {
    return with_dtype(dtype, [&](auto t) { return launch_obs_d<decltype(t)>(d, K, q, n_q, scaling, ws, scores_out, st); });
}

}  // namespace kvp
