// cam.cu — CAMPress's merge-before-prune compaction (kvp_cam_compress, include/kvpress_b200.h).
//
// One call, per batch element b (all kv heads share one selection):
//   1. cam_mean_kernel: m[s] = (sum of the Hkv scores, ascending head, fp32) / Hkv, rounded once; its ordered 16-bit
//      key and the key histogram go to the shared selection workspace, laid out for B rows of S positions.
//   2. select_compact_kernel (select_compact.cu), selection only: the n_kept best m, ties to the lowest positions.
//   3. cam_candidates_kernel: the n_merge best evicted positions by (m descending, position descending), from two
//      256-bin histograms of the keys of the evicted positions, then one ordered pass that writes them ascending with
//      t_i, the number of kept positions below candidate i.
//   4. cam_prob_kernel: per (b, head, candidate) the window mean of the running sum, p_i and the weight mask_i / n_i.
//   5. cam_merge_kernel: per output row r, the candidates whose window holds r (a binary search over t, which is
//      nondecreasing), summed into V[kept[r]] in fp32 in ascending i; K, V and the running sum are compacted in the
//      same pass. No atomics: every sum has a fixed order, so results are bitwise repeatable.
#include "common.cuh"

namespace kvp {

constexpr int kCandThreads = 1024;  // cam_candidates_kernel: one CTA per batch element, 8 keys per thread per pass
constexpr int kMergeThreads = 256;

// The CAM regions of the scratch area, sized for n_merge = S - n_kept: kept positions [B][n_kept], candidates and
// their kept counts t [B][n_merge], the merge weights mask / n [B][Hkv][n_merge].
struct CamScratch {
    int32_t* kept;
    int32_t* cand;
    int32_t* t;
    float* weight;
    size_t bytes;
};

static CamScratch cam_carve(const Dims& d, void* base) {
    Carve c(base);
    const size_t n_ev = (size_t)(d.S - d.n_kept);
    CamScratch s;
    s.kept = c.take<int32_t>((size_t)d.B * d.n_kept);
    s.cand = c.take<int32_t>((size_t)d.B * n_ev);
    s.t = c.take<int32_t>((size_t)d.B * n_ev);
    s.weight = c.take<float>((size_t)d.B * d.H * n_ev);
    s.bytes = c.bytes;
    return s;
}

size_t cam_scratch_bytes(const Dims& d) { return cam_carve(d, nullptr).bytes; }

Dims cam_selection_dims(const Dims& d) {
    Dims s = d;
    s.H = s.Hq = 1;
    s.R = d.B;
    s.ks = s.vs = {0, 0, 0};
    return s;
}

template <typename T>
__global__ void __launch_bounds__(kTileThreads)
cam_mean_kernel(const uint16_t* __restrict__ scores, int64_t sb, int64_t sh, int H, int S, Workspace ws) {
    __shared__ uint16_t skeys[kTile];
    __shared__ uint32_t shist[256];
    const int tile = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    shist[tid] = 0;
    pdl_launch_dependents();  // the selection kernel behind this one may start to take residency
    const int s = tile * kTile + tid;
    uint16_t key = 0;
    if (s < S) {
        const uint16_t* src = scores + (int64_t)b * sb + s;
        float sum = 0.f;
        for (int h = 0; h < H; ++h) sum += F16Traits<T>::to_float(src[(int64_t)h * sh]);
        key = ordered_key16(round_once<T>(sum / (float)H), F16Traits<T>::kInfBits);
    }
    skeys[tid] = key;
    __syncthreads();
    flush_chunk_keys<1>(skeys, nullptr, shist, b, tile * kTile, S, ws, nullptr);
}

__device__ __forceinline__ uint32_t key_at(const uint4& v, int j) {
    const uint32_t w = j < 2 ? v.x : j < 4 ? v.y : j < 6 ? v.z : v.w;
    return (j & 1) ? (w >> 16) : (w & 0xFFFFu);
}

// The 8 keys of positions [s0, s0 + 8) of a row; zero (no key) from S on. s0 is a multiple of 8, and a row's keys are
// padded to a multiple of kTile, so the load never leaves the row.
__device__ __forceinline__ uint4 load_keys8(const uint16_t* keys, int s0, int S) {
    return s0 < S ? __ldcg(reinterpret_cast<const uint4*>(keys + s0)) : make_uint4(0, 0, 0, 0);
}

// Exclusive prefix over the CTA of three per-thread counts, and their CTA totals. Call with every thread.
__device__ __forceinline__ void block_scan3(uint32_t (&v)[3], uint32_t (&before)[3], uint32_t (&total)[3],
                                            uint32_t (*wsum)[kCandThreads / 32]) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint32_t incl[3] = {v[0], v[1], v[2]};
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const uint32_t x = __shfl_up_sync(0xFFFFFFFFu, incl[k], off);
            if (lane >= off) incl[k] += x;
        }
    }
    if (lane == 31) {
#pragma unroll
        for (int k = 0; k < 3; ++k) wsum[k][warp] = incl[k];
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        uint32_t b = incl[k] - v[k], t = 0;
        for (int w = 0; w < kCandThreads / 32; ++w) {
            const uint32_t x = wsum[k][w];
            b += w < warp ? x : 0u;
            t += x;
        }
        before[k] = b;
        total[k] = t;
    }
    __syncthreads();  // wsum is rewritten by the next call
}

// One CTA per batch element. The kept positions get key 0, which no number has (every NaN's key is 0xFFFF); the
// n_merge best of the other keys, ties to the LATER position, are the candidates.
__global__ void __launch_bounds__(kCandThreads)
cam_candidates_kernel(int S, int n_kept, int n_merge, Workspace ws, const int32_t* __restrict__ kept,
                      int32_t* __restrict__ cand, int32_t* __restrict__ t_out, int32_t* __restrict__ merge_idx_out) {
    __shared__ uint32_t hist[256];
    __shared__ uint32_t wsum[3][kCandThreads / 32];
    __shared__ uint32_t thr[3];
    const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    uint16_t* keys = ws.keys + (size_t)b * ws.S_pad;
    pdl_wait();  // the kept positions are complete
    pdl_launch_dependents();
    for (int r = tid; r < n_kept; r += kCandThreads) keys[kept[(size_t)b * n_kept + r]] = 0;
    if (tid < 256) hist[tid] = 0;
    __syncthreads();

    constexpr int kStep = 8 * kCandThreads;
    for (int base = 0; base < S; base += kStep) {
        const uint4 v = load_keys8(keys, base + 8 * tid, S);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const uint32_t key = key_at(v, j);
            warp_hist_add(hist, key ? (key >> 8) : 256u);
        }
    }
    __syncthreads();
    if (warp == 0) {
        int b1;
        uint32_t above;
        warp_suffix_find(hist, (uint32_t)n_merge, lane, b1, above);
        if (lane == 0) {
            thr[0] = (uint32_t)b1;
            thr[1] = (uint32_t)n_merge - above;  // >= 1
        }
    }
    __syncthreads();
    const uint32_t b1 = thr[0], need = thr[1];
    if (tid < 256) hist[tid] = 0;
    __syncthreads();
    for (int base = 0; base < S; base += kStep) {
        const uint4 v = load_keys8(keys, base + 8 * tid, S);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const uint32_t key = key_at(v, j);
            warp_hist_add(hist, key && (key >> 8) == b1 ? (key & 255u) : 256u);
        }
    }
    __syncthreads();
    if (warp == 0) {
        int lo1;
        uint32_t above;
        warp_suffix_find(hist, need, lane, lo1, above);
        if (lane == 0) {
            thr[0] = (b1 << 8) | (uint32_t)lo1;
            thr[1] = hist[lo1] - (need - above);  // ties at T that are NOT taken: the earliest ones
        }
    }
    __syncthreads();
    const uint32_t T = thr[0], skip = thr[1];

    // Ascending pass. Position s is a candidate if key > T, or key == T with at least `skip` ties before it; its slot is
    // (keys > T before s) + (taken ties before s), and t = s - (evicted positions before s).
    uint32_t run[3] = {0, 0, 0};  // keys > T, keys == T, evicted (non-zero keys) before this pass step
    const int64_t out0 = (int64_t)b * n_merge;
    for (int base = 0; base < S; base += kStep) {
        const int s0 = base + 8 * tid;
        const uint4 v = load_keys8(keys, s0, S);
        uint32_t cnt[3] = {0, 0, 0};
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const uint32_t key = key_at(v, j);
            cnt[0] += key > T;
            cnt[1] += key == T;
            cnt[2] += key != 0;
        }
        uint32_t before[3], total[3];
        block_scan3(cnt, before, total, wsum);
        uint32_t gt = run[0] + before[0], eq = run[1] + before[1], ev = run[2] + before[2];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const uint32_t key = key_at(v, j);
            const bool take = key > T || (key == T && eq >= skip);
            if (take) {
                const int64_t slot = out0 + gt + (eq > skip ? eq - skip : 0u);
                const int s = s0 + j;
                cand[slot] = s;
                t_out[slot] = s - (int)ev;
                if (merge_idx_out != nullptr) merge_idx_out[slot] = s;
            }
            gt += key > T;
            eq += key == T;
            ev += key != 0;
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) run[k] += total[k];
    }
}

// One thread per (candidate i, row b * Hkv + h): the window of kept ranks [t_i, t_i + n_i), its mean running sum, p_i
// and the weight mask_i / n_i (0 when the draw fails).
__global__ void __launch_bounds__(256)
cam_prob_kernel(int H, int n_kept, int n_merge, int budget, const float* __restrict__ A, int64_t ab, int64_t ah,
                const float* __restrict__ u, const int32_t* __restrict__ kept, const int32_t* __restrict__ cand,
                const int32_t* __restrict__ t, float* __restrict__ weight, float* __restrict__ prob_out) {
    pdl_wait();  // candidates and t are complete
    pdl_launch_dependents();
    const int i = blockIdx.x * blockDim.x + threadIdx.x, row = blockIdx.y, b = row / H, h = row % H;
    if (i >= n_merge) return;
    const float* a = A + (int64_t)b * ab + (int64_t)h * ah;
    const int32_t* kp = kept + (int64_t)b * n_kept;
    const int64_t ci = (int64_t)b * n_merge + i;
    const int ti = t[ci];
    const int n = min(budget, n_kept - ti);
    float sum = 0.f;
    for (int r = ti; r < ti + n; ++r) sum += a[kp[r]];
    float p = a[cand[ci]] / (sum / (float)max(n, 1));
    if (isnan(p)) p = 0.f;
    p = fminf(fmaxf(p, 0.f), 1.f);  // +inf -> 1, -inf -> 0
    const int64_t o = (int64_t)row * n_merge + i;
    weight[o] = u[o] < p ? 1.f / (float)max(n, 1) : 0.f;
    if (prob_out != nullptr) prob_out[o] = p;
}

// First index in t[0, n) whose value exceeds x (t nondecreasing).
__device__ __forceinline__ int first_above(const int32_t* __restrict__ t, int n, int x) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (t[mid] > x) hi = mid;
        else lo = mid + 1;
    }
    return lo;
}

// LPR lanes per output row, 8 elements per lane and 16-byte vector. Output row r of (b, h) gets K[kept[r]] and
// A[kept[r]] exactly, and V[kept[r]] + sum of weight_i V[e_i] over the candidates with t_i <= r < t_i + budget, in
// ascending i, each term one fused multiply-add in fp32, rounded once. A row may receive up to n_merge terms.
template <typename T, int LPR>
__global__ void __launch_bounds__(kMergeThreads)
cam_merge_kernel(const char* __restrict__ K, const char* __restrict__ V, Strides3 ks, Strides3 vs,
                 const float* __restrict__ A, int64_t ab, int64_t ah, char* __restrict__ K_out, char* __restrict__ V_out,
                 float* __restrict__ A_out, int64_t ob, int64_t oh, int H, int D, int n_kept, int n_merge, int budget,
                 const int32_t* __restrict__ kept, const int32_t* __restrict__ cand, const int32_t* __restrict__ t,
                 const float* __restrict__ weight) {
    pdl_wait();  // kept positions and weights are complete
    constexpr int kRows = kMergeThreads / LPR;
    const int lane = threadIdx.x % LPR, r = blockIdx.x * kRows + threadIdx.x / LPR;
    const int row = blockIdx.y, b = row / H, h = row % H;
    if (r >= n_kept) return;
    const int64_t s = kept[(int64_t)b * n_kept + r];
    const char* k_row = K + ((int64_t)b * ks.b + (int64_t)h * ks.h + s * ks.s) * 2;
    const char* v_base = V + ((int64_t)b * vs.b + (int64_t)h * vs.h) * 2;
    const char* v_row = v_base + s * vs.s * 2;
    const int64_t out_row = ((int64_t)row * n_kept + r) * D * 2;
    // the candidates whose window holds rank r: r - budget < t_i <= r
    const int32_t* tb = t + (int64_t)b * n_merge;
    const int i_lo = n_merge > 0 ? first_above(tb, n_merge, r - budget) : 0;
    const int i_hi = n_merge > 0 ? first_above(tb, n_merge, r) : 0;
    const int32_t* cb = cand + (int64_t)b * n_merge;
    const float* wb = weight + (int64_t)row * n_merge;
    const uint64_t pol_first = l2_policy_evict_first();
    for (int c = lane; c < (D >> 3); c += LPR) {
        stg_hint(K_out + out_row + c * 16, ldg_plain(k_row + c * 16), pol_first);
        const int4 vk = ldg_plain(v_row + c * 16);
        float acc[8];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float2 f = F16Traits<T>::unpack2(reinterpret_cast<const uint32_t*>(&vk)[q]);
            acc[2 * q] = f.x;
            acc[2 * q + 1] = f.y;
        }
        for (int i = i_lo; i < i_hi; ++i) {
            const float w = wb[i];
            const int4 ve = ldg_plain(v_base + (int64_t)cb[i] * vs.s * 2 + c * 16);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float2 f = F16Traits<T>::unpack2(reinterpret_cast<const uint32_t*>(&ve)[q]);
                acc[2 * q] = fmaf(w, f.x, acc[2 * q]);
                acc[2 * q + 1] = fmaf(w, f.y, acc[2 * q + 1]);
            }
        }
        int4 o;
        uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
        for (int q = 0; q < 4; ++q)
            ow[q] = (uint32_t)round_once<T>(acc[2 * q]) | ((uint32_t)round_once<T>(acc[2 * q + 1]) << 16);
        stg_hint(V_out + out_row + c * 16, o, pol_first);
    }
    if (lane == 0) A_out[(int64_t)b * ob + (int64_t)h * oh + r] = A[(int64_t)b * ab + (int64_t)h * ah + s];
}

cudaError_t launch_cam_compress(const Dims& d, int dtype, const void* scores, int64_t sb, int64_t sh, const void* K,
                                const void* V, const float* A, int64_t ab, int64_t ah, int n_merge, int budget,
                                const float* u, void* K_out, void* V_out, float* A_out, int64_t ob, int64_t oh,
                                int32_t* idx_out, int32_t* merge_idx_out, float* prob_out, const Workspace& ws,
                                cudaStream_t st) {
    const CamScratch cs = cam_carve(d, ws.scorer);
    int32_t* kept = idx_out != nullptr ? idx_out : cs.kept;
    return with_dtype(dtype, [&](auto tv) -> cudaError_t {
        using T = decltype(tv);
        cam_mean_kernel<T><<<dim3(ws.n_tiles, d.B), kTileThreads, 0, st>>>(static_cast<const uint16_t*>(scores), sb,
                                                                          sh, d.H, d.S, ws);
        cudaError_t e = cudaPeekAtLastError();
        if (e != cudaSuccess) return e;
        if ((e = launch_select_compact(cam_selection_dims(d), nullptr, nullptr, nullptr, nullptr, kept, ws, st)))
            return e;
        if (n_merge > 0) {
            if ((e = launch_pdl(cam_candidates_kernel, dim3(d.B), dim3(kCandThreads), 0, st, d.S, d.n_kept, n_merge,
                                ws, kept, cs.cand, cs.t, merge_idx_out)))
                return e;
            if ((e = launch_pdl(cam_prob_kernel, dim3((n_merge + 255) / 256, d.R), dim3(256), 0, st, d.H, d.n_kept,
                                n_merge, budget, A, ab, ah, u, kept, cs.cand, cs.t, cs.weight, prob_out)))
                return e;
        }
        with_lanes_per_row(d.D, [&](auto lpr) {
            constexpr int L = decltype(lpr)::value;
            constexpr int kRows = kMergeThreads / L;
            e = launch_pdl(cam_merge_kernel<T, L>, dim3((d.n_kept + kRows - 1) / kRows, d.R), dim3(kMergeThreads), 0,
                           st, static_cast<const char*>(K), static_cast<const char*>(V), d.ks, d.vs, A, ab, ah,
                           static_cast<char*>(K_out), static_cast<char*>(V_out), A_out, ob, oh, d.H, d.D, d.n_kept,
                           n_merge, budget, static_cast<const int32_t*>(kept), static_cast<const int32_t*>(cs.cand),
                           static_cast<const int32_t*>(cs.t), static_cast<const float*>(cs.weight));
        });
        return e;
    });
}

}  // namespace kvp
