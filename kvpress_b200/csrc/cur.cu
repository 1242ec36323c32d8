// cur.cu — CURPress scores (reference kvpress/presses/cur_press.py; CurDKV, https://arxiv.org/abs/2509.15038).
//
// Per row (b, kv head j) with S positions, w = local_window_size (0: no local approximation), evaluated in fp32 from
// the 16-bit inputs and rounded once to the cache dtype:
//   - a_k(s) = sum_d k_d^2, or with a projection G [D, r] (float32, row-major): a_k(s) = sum_c (sum_d k_d G_dc)^2.
//     a_v(s) likewise from V.
//   - w >= 1: window c covers [cw, (c+1)w) within [0, S); p_k(s) = a_k(s) / sum_{t in window} a_k(t), IEEE rules
//     (0/0 = NaN). The last, short window sums its real positions only. w = 0: p_k = a_k. p_v likewise.
//   - u(s) = p_k | p_v | (p_k + p_v) / 2 | p_k p_v for leverage_type 0 | 1 | 2 | 3 (key, value, kv_avg, kv_product).
//     Type 0 does not read V and type 1 does not read K.
//   - T = sum_s u(s) over all S positions; score(s) = u(s) / T; positions s < num_sinks score exactly 1.
// NaN and inf propagate as in torch: one NaN u (an all-zero window gives 0/0) makes T and so every non-sink score of the
// row NaN; an inf u makes T inf, its own score NaN and the others 0. fp32 overflow departs from the definition only for
// bf16 inputs near the top of their range (a sum of squares, or a product of two of them, beyond 3.4e38).
//
// Schedule: two kernels.
//   1. cur_unit_kernel, grid (CTAs per row, B Hkv), 256 threads. A unit is ceil(256 / w) whole windows of a row (256
//      positions without local approximation): 256 to 1024 positions, fixed by S and w alone. A CTA strides over the
//      units of its row. Per unit: a_k and a_v of its positions go to shared memory (row_norm_span of knorm_chunk.cuh,
//      one 128-bit load per lane and row; with a projection one thread per row against G in shared memory, its columns
//      padded to 32), every window is summed by one warp in a fixed lane order and divided through, u(s) is written to
//      the fp32 [B Hkv, S] scratch and the unit's sum of u, taken in fp64 in a fixed order, to partials[row][unit].
//   2. cur_finalize_kernel, one CTA per 256 positions: T from the row's partials in a fixed order in fp64, u / T, the
//      sinks, the one rounding, then scores, ordered keys and the row histogram (flush_chunk_keys). The shared
//      select+compact stage follows it by programmatic dependent launch.
// The units, the window sums and T do not depend on how many CTAs share a row, so a row's scores are bitwise
// independent of the SM count, of the batch it sits in and of the strides of the cache.
#include <math.h>

#include "knorm_chunk.cuh"

namespace kvp {

constexpr int kCurThreads = 256;
constexpr int kCurWarps = kCurThreads / 32;
constexpr int kCurUnitMax = 1024;   // positions of the largest unit: kCurWindowMax, or 255 + 256 for w <= 256
constexpr int kCurCtasPerSm = 4;    // CTAs per SM the grid of the unit kernel is sized for
constexpr int kCurGCols = 32;       // columns of G in shared memory (kCurRankMax, zero padded)
static_assert(kCurUnitMax >= kCurWindowMax && kCurGCols == kCurRankMax, "unit and projection limits");

struct CurArgs {
    const void* K;
    const void* V;
    Strides3 ks, vs;
    int H, S, D;
    int w;          // window length; 0 without local approximation
    int unit;       // positions per unit
    int n_units;    // units per row
    int type;       // 0 key, 1 value, 2 kv_avg, 3 kv_product
    const float* G; // [D][r] or null
    int r;
    float* u;           // [R][S]
    double* partials;   // [R][part_stride]
    int part_stride;
};

struct CurScratch {
    float* u;
    double* partials;
    int part_stride;
};

static CurScratch cur_scratch(const Dims& d, const Workspace& ws) {
    Carve c(ws.scorer);
    CurScratch sc;
    sc.u = c.take<float>((size_t)d.R * d.S);
    sc.part_stride = (d.S + kTile - 1) / kTile;  // a unit has at least 256 positions
    sc.partials = c.take<double>((size_t)d.R * sc.part_stride);
    return sc;
}

size_t cur_scratch_bytes(const Dims& d) {
    Carve c(nullptr);
    c.take<float>((size_t)d.R * d.S);
    c.take<double>((size_t)d.R * ((d.S + kTile - 1) / kTile));
    return c.bytes;
}

// Sum of x over the CTA in fp64: the lanes of a warp by an xor butterfly, then the warps in index order.
__device__ __forceinline__ double cur_block_sum(double x, double* red) {
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) x += __shfl_xor_sync(0xFFFFFFFFu, x, off);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = x;
    __syncthreads();
    double t = red[0];
#pragma unroll
    for (int i = 1; i < kCurWarps; ++i) t += red[i];
    __syncthreads();  // red is reused
    return t;
}

// sum_c (sum_d x_d G_dc)^2 of one row, by one thread: d ascending per column, then c ascending.
template <typename T>
__device__ __forceinline__ float cur_projected(const T* __restrict__ x, int D, int r, const float* __restrict__ sG) {
    float acc[kCurGCols];
#pragma unroll
    for (int c = 0; c < kCurGCols; ++c) acc[c] = 0.f;
#pragma unroll 1
    for (int v = 0; v < (D >> 3); ++v) {
        const int4 w4 = __ldg(reinterpret_cast<const int4*>(x) + v);
        const uint32_t w[4] = {(uint32_t)w4.x, (uint32_t)w4.y, (uint32_t)w4.z, (uint32_t)w4.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 f = F16Traits<T>::unpack2(w[j]);
            const float4* g0 = reinterpret_cast<const float4*>(sG + (size_t)(v * 8 + 2 * j) * kCurGCols);
            const float4* g1 = g0 + kCurGCols / 4;
#pragma unroll
            for (int q = 0; q < kCurGCols / 4; ++q) {
                const float4 a = g0[q];
                acc[4 * q] = fmaf(f.x, a.x, acc[4 * q]);
                acc[4 * q + 1] = fmaf(f.x, a.y, acc[4 * q + 1]);
                acc[4 * q + 2] = fmaf(f.x, a.z, acc[4 * q + 2]);
                acc[4 * q + 3] = fmaf(f.x, a.w, acc[4 * q + 3]);
            }
#pragma unroll
            for (int q = 0; q < kCurGCols / 4; ++q) {
                const float4 a = g1[q];
                acc[4 * q] = fmaf(f.y, a.x, acc[4 * q]);
                acc[4 * q + 1] = fmaf(f.y, a.y, acc[4 * q + 1]);
                acc[4 * q + 2] = fmaf(f.y, a.z, acc[4 * q + 2]);
                acc[4 * q + 3] = fmaf(f.y, a.w, acc[4 * q + 3]);
            }
        }
    }
    float ss = 0.f;
#pragma unroll
    for (int c = 0; c < kCurGCols; ++c)
        if (c < r) ss = fmaf(acc[c], acc[c], ss);  // the padding columns take no part (inf * 0 would be NaN)
    return ss;
}

template <typename T, int LPR, bool kProj>
__global__ void __launch_bounds__(kCurThreads) cur_unit_kernel(CurArgs a) {
    __shared__ float sa[2][kCurUnitMax];  // a_k and a_v of the unit, then p_k and p_v
    __shared__ double red[kCurWarps];
    extern __shared__ __align__(16) float sG[];  // [D][kCurGCols], kProj only
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int row = blockIdx.y, b = row / a.H, h = row % a.H;
    const bool use_k = a.type != 1, use_v = a.type != 0;
    if (kProj) {
        for (int i = tid; i < a.D * kCurGCols; i += kCurThreads) {
            const int d = i / kCurGCols, c = i % kCurGCols;
            sG[i] = c < a.r ? a.G[(size_t)d * a.r + c] : 0.f;
        }
        __syncthreads();
    }
    for (int unit = blockIdx.x; unit < a.n_units; unit += gridDim.x) {
        const int s0 = unit * a.unit, s1 = min(a.S, s0 + a.unit), len = s1 - s0;
        if (kProj) {
            const T* Kb = static_cast<const T*>(a.K) + (int64_t)b * a.ks.b + (int64_t)h * a.ks.h;
            const T* Vb = static_cast<const T*>(a.V) + (int64_t)b * a.vs.b + (int64_t)h * a.vs.h;
            for (int i = tid; i < len; i += kCurThreads) {
                if (use_k) sa[0][i] = cur_projected<T>(Kb + (int64_t)(s0 + i) * a.ks.s, a.D, a.r, sG);
                if (use_v) sa[1][i] = cur_projected<T>(Vb + (int64_t)(s0 + i) * a.vs.s, a.D, a.r, sG);
            }
        } else {
            constexpr int kLoads = LPR == 4 ? 4 : 8;  // 128-bit loads in flight per lane and tensor
            if (use_k)
                row_norm_span<T, LPR, kLoads, false>(static_cast<const T*>(a.K), a.ks, b, h, s0, s1, a.D, sa[0] - s0, warp,
                                                kCurWarps);
            if (use_v)
                row_norm_span<T, LPR, kLoads, false>(static_cast<const T*>(a.V), a.vs, b, h, s0, s1, a.D, sa[1] - s0, warp,
                                                kCurWarps);
        }
        __syncthreads();
        if (a.w > 0) {
            // one warp per window: lane l sums positions l, l + 32, ... in order, then an xor butterfly; each lane
            // divides the positions it summed
            const int n_win = (len + a.w - 1) / a.w;
            for (int win = warp; win < n_win; win += kCurWarps) {
                const int lo = win * a.w, hi = min(len, lo + a.w);
                float fk = 0.f, fv = 0.f;
                for (int i = lo + lane; i < hi; i += 32) {
                    if (use_k) fk += sa[0][i];
                    if (use_v) fv += sa[1][i];
                }
#pragma unroll
                for (int off = 16; off >= 1; off >>= 1) {
                    fk += __shfl_xor_sync(0xFFFFFFFFu, fk, off);
                    fv += __shfl_xor_sync(0xFFFFFFFFu, fv, off);
                }
                for (int i = lo + lane; i < hi; i += 32) {
                    if (use_k) sa[0][i] = sa[0][i] / fk;
                    if (use_v) sa[1][i] = sa[1][i] / fv;
                }
            }
            __syncthreads();
        }
        double part = 0.0;
        for (int i = tid; i < len; i += kCurThreads) {
            const float pk = use_k ? sa[0][i] : 0.f, pv = use_v ? sa[1][i] : 0.f;
            const float u = a.type == 0 ? pk : a.type == 1 ? pv : a.type == 2 ? (pk + pv) * 0.5f : pk * pv;
            a.u[(size_t)row * a.S + s0 + i] = u;
            part += (double)u;
        }
        part = cur_block_sum(part, red);  // its barriers also free sa for the next unit
        if (tid == 0) a.partials[(size_t)row * a.part_stride + unit] = part;
    }
}

template <typename T>
__global__ void __launch_bounds__(kTileThreads)
cur_finalize_kernel(int S, int n_units, int num_sinks, CurScratch sc, Workspace ws, uint16_t* __restrict__ scores_out) {
    __shared__ uint16_t skeys[kTile];
    __shared__ uint16_t sscores[kTile];
    __shared__ uint32_t shist[256];
    __shared__ double red[kCurWarps];
    const int tile = blockIdx.x, row = blockIdx.y, tid = threadIdx.x;
    shist[tid] = 0;
    pdl_launch_dependents();  // the select+compact kernel behind this one may start to take residency
    double t = 0.0;
    for (int i = tid; i < n_units; i += kTileThreads) t += sc.partials[(size_t)row * sc.part_stride + i];
    const double total = cur_block_sum(t, red);
    score_tile_epilogue<T, 1>(skeys, sscores, shist, row, tile * kTile, S, 0, 0, ws, scores_out, nullptr, [&](int, int s) {
        return s < num_sinks ? 1.f : (float)((double)sc.u[(size_t)row * S + s] / total);
    });
}

template <typename T>
static cudaError_t launch_cur_t(const CurArgs& a, const Dims& d, int num_sinks, const CurScratch& sc,
                                const Workspace& ws, void* scores_out, cudaStream_t st) {
    const int per_row = min(a.n_units, max(1, (kCurCtasPerSm * device_sm_count() + d.R - 1) / d.R));
    const dim3 grid(per_row, d.R);
    if (a.r > 0) {
        cur_unit_kernel<T, 4, true><<<grid, kCurThreads, (size_t)a.D * kCurGCols * sizeof(float), st>>>(a);
    } else {
        with_lanes_per_row(a.D, [&](auto lpr) { cur_unit_kernel<T, lpr, false><<<grid, kCurThreads, 0, st>>>(a); });
    }
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) return e;
    cur_finalize_kernel<T><<<dim3(ws.n_tiles, d.R), kTileThreads, 0, st>>>(d.S, a.n_units, num_sinks, sc, ws,
                                                                           static_cast<uint16_t*>(scores_out));
    return cudaPeekAtLastError();
}

cudaError_t launch_cur_score(const Dims& d, int dtype, const void* K, const void* V, int num_sinks, int leverage_type,
                             int window, const float* G, int r, const Workspace& ws, void* scores_out,
                             cudaStream_t st) {
    if (d.D > 256 || window < 0 || window > kCurWindowMax || r < 0 || r > kCurRankMax || (G == nullptr) != (r == 0) ||
        leverage_type < 0 || leverage_type > 3 || num_sinks < 0)
        return cudaErrorNotSupported;
    const CurScratch sc = cur_scratch(d, ws);
    CurArgs a = {};
    a.K = K;
    a.V = V;
    a.ks = d.ks;
    a.vs = d.vs;
    a.H = d.H;
    a.S = d.S;
    a.D = d.D;
    a.w = window;
    a.unit = window > 0 ? window * ((kTile + window - 1) / window) : kTile;
    a.n_units = (d.S + a.unit - 1) / a.unit;
    a.type = leverage_type;
    a.G = G;
    a.r = r;
    a.u = sc.u;
    a.partials = sc.partials;
    a.part_stride = sc.part_stride;
    return with_dtype(dtype, [&](auto t) { return launch_cur_t<decltype(t)>(a, d, num_sinks, sc, ws, scores_out, st); });
}

}  // namespace kvp
