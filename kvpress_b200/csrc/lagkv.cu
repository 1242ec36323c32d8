// lagkv.cu — LagKVPress scores (reference kvpress/presses/lagkv_press.py; https://arxiv.org/abs/2504.04704).
//
// Per row (b, kv head j), with S positions and L = lag_size:
//   - Short cache, S < n_sink + 2L. Position s < n_sink scores 1. Position s >= n_sink scores
//     fp32(s - n_sink) / fp32(S - n_sink), rounded once to the cache dtype. This is the reference's float32
//     `arange / n`, then `.to(dtype)`.
//   - Otherwise:
//       - Let P = (S - n_sink) // L and end = n_sink + P L.
//       - Partition c covers positions [n_sink + cL, n_sink + (c+1)L).
//       - Partitions c = 0 ... P-2 are scored. Each uses partition c+1 as its reference.
//       - The sinks, partition P-1 and the remainder [end, S) score 1, so the tail has L + S - end positions.
//   - Within a scored partition, for each channel d:
//       - lo_d and hi_d are the min and max of the reference partition's L rows.
//       - x_{s,d} = (k_{s,d} - lo_d) / (hi_d - lo_d), with IEEE rules: x/0 = +-inf and 0/0 = NaN.
//       - sigma_k(s) is the unbiased standard deviation of x over d (divisor D - 1, as torch.std). sigma_v is the
//         same with V.
//       - a_k = softmax of sigma_k over the partition's L rows, and a_v likewise.
//       - c(s) = (a_k(s) + a_v(s)) / 2.
//   - The score of a scored position:
//       - cross_scoring: c(s), rounded once.
//       - Otherwise, the rank r(s) = #{t : c(t) < c(s)} + #{t < s : c(t) = c(s)} over the partition. NaN compares
//         above every number and equal to NaN, which is what torch.sort(stable=True) does. The score is
//         fp32(r) / fp32(L), rounded once. Given r, it is bitwise the reference's value.
// Everything is evaluated in fp32 from the 16-bit inputs; the reference runs the chain in the cache dtype.
// Degenerate reference partitions: a constant channel of the reference partition, in K or V, makes every sigma of the
// partition it scores NaN (x is +-inf or NaN in that channel), so that partition's cross scores are NaN and its ranks
// are in position order, as in the reference. A zeroed channel (ThinK-style pruning) is one; L = 1 makes every scored
// partition NaN. A NaN in a reference partition's K or V makes the partition it scores NaN too, as torch.min / max
// propagate it. The evaluation is fp32: where an intermediate leaves the fp32 range, which only bf16 inputs can cause (a
// reference range hi - lo that overflows, or one so small against the scored values that x or its square overflows),
// the kernel departs from the float64 definition, and an overflowing sigma makes the whole partition NaN.
//
// Schedule: one kernel, grid (items, B Hkv). An item is either
//   - a segment of consecutive scored partitions [c0, c1) of one row. The CTA first takes the per-channel min / max of
//     partition c1 (the reference of c1 - 1), then walks c = c1 - 1 down to c0. Each partition's rows are read from
//     HBM once: that one load is scored against the statistics held from c + 1 and yields the partition's own min /
//     max, which c - 1 needs. K and V are read once plus one partition per segment. Segments are sized so that a row
//     has ceil(kLagItemsPerSm * SMs / (B Hkv)) of them (at most one per scored partition), or
//   - 256 positions of the constant parts of a row: the sinks and the tail, or the whole short cache.
// Shared memory holds sigma_k / sigma_v (then c and its ordered keys) of the partition, and the four D-float statistic
// vectors. The rank is counted exactly over the partition in shared memory. min / max are exact, and every row's sums
// run in a fixed lane order, so a row's scores do not depend on the schedule or on the other rows of the batch.
// With keys wanted (compress), the kernel writes the ordered 16-bit keys and the row histograms for the shared
// select+compact stage, which follows it by programmatic dependent launch.
#include <math.h>

#include "common.cuh"

namespace kvp {

constexpr int kLagThreads = 256;
constexpr int kLagItemsPerSm = 2;  // scoring items per SM the segments are sized for (2 CTAs per SM are resident)

struct LagArgs {
    const void* K;
    const void* V;
    Strides3 ks, vs;
    int H, S, D, n_sink, L, cross;
    int n_scored;   // scored partitions per row (P - 1); 0 on the short path
    int seg_len;    // scored partitions per segment
    int n_seg;      // segments per row
    int n_fill_a;   // 256-position items of [0, end_a)
    int end_a;      // n_sink (long path) or fill_end (short path)
    int tail_start; // n_sink + (P - 1) L: the first position of the constant tail (long path)
    int fill_end;   // S_pad with keys (the key padding is written as 0), else S
    Workspace ws;
    uint16_t* scores_out;
    int want_keys;
};

// order-preserving int image of a float (min / max through integer atomics; exact, order independent)
__device__ __forceinline__ int f2o(float f) {
    const int i = __float_as_int(f);
    return i >= 0 ? i : i ^ 0x7FFFFFFF;
}
__device__ __forceinline__ float o2f(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7FFFFFFF); }

// the rank's comparison: ordered_f32, except that every NaN sorts above everything and -0 ties with +0 (as torch.sort)
__device__ __forceinline__ uint32_t rank_key(float f) {
    return isnan(f) ? 0xFFFFFFFFu : ordered_f32(f == 0.f ? 0.f : f);
}

// Writes one position's score (or, past S, its zero key padding) and counts its key in the CTA histogram.
// Every lane of the warp calls it; `valid` marks the lanes that own a position.
template <typename T>
__device__ __forceinline__ void emit(const LagArgs& a, int row, int s, bool valid, float value, uint32_t* shist) {
    unsigned bin = 256u;
    if (valid) {
        if (s < a.S) {
            const uint16_t bits = F16Traits<T>::from_float(value);
            if (a.scores_out) a.scores_out[(size_t)row * a.S + s] = bits;
            if (a.want_keys) {
                const uint16_t key = ordered_key16(bits, F16Traits<T>::kInfBits);
                a.ws.keys[(size_t)row * a.ws.S_pad + s] = key;
                bin = key >> 8;
            }
        } else if (a.want_keys) {
            a.ws.keys[(size_t)row * a.ws.S_pad + s] = 0;
        }
    }
    if (a.want_keys) warp_hist_add(shist, bin);
}

// sigma of one row: x = (v - lo) / (hi - lo) over this lane's 8 channels, mean and the two-pass unbiased std over the
// D channels of the LPR lanes of the row (xor butterflies: a fixed order).
template <int LPR>
__device__ __forceinline__ float row_sigma(const float (&v)[8], const float (&lo)[8], const float (&hi)[8],
                                           bool lane_ok, int D) {
    float x[8];
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        x[j] = lane_ok ? (v[j] - lo[j]) / (hi[j] - lo[j]) : 0.f;
        sum += x[j];
    }
#pragma unroll
    for (int off = LPR / 2; off >= 1; off >>= 1) sum += __shfl_xor_sync(0xFFFFFFFFu, sum, off);
    const float mean = sum / (float)D;
    float q = 0.f;
    if (lane_ok)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float d = x[j] - mean;
            q = fmaf(d, d, q);
        }
#pragma unroll
    for (int off = LPR / 2; off >= 1; off >>= 1) q += __shfl_xor_sync(0xFFFFFFFFu, q, off);
    return sqrtf(q / (float)(D - 1));
}

template <typename T>
__device__ __forceinline__ void unpack8(const int4& w4, float (&f)[8]) {
    const uint32_t w[4] = {(uint32_t)w4.x, (uint32_t)w4.y, (uint32_t)w4.z, (uint32_t)w4.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float2 p = F16Traits<T>::unpack2(w[j]);
        f[2 * j] = p.x;
        f[2 * j + 1] = p.y;
    }
}

struct LagSmem {
    float sk[kLagMax];  // sigma_k of the partition's rows, then c
    float sv[kLagMax];  // sigma_v, then the rank keys of c (as uint32)
    float stat[4][256]; // lo_k, hi_k, lo_v, hi_v of the reference partition
    int next[4][256];   // the same of the partition being read, as f2o images
    float red[2][kLagThreads / 32];
    uint32_t hist[256];
};

// Block reduction of two floats (max or sum) in a fixed order; every thread gets the results.
template <bool kMax>
__device__ __forceinline__ void block_reduce2(float& x, float& y, LagSmem& sm) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
        const float ox = __shfl_xor_sync(0xFFFFFFFFu, x, off), oy = __shfl_xor_sync(0xFFFFFFFFu, y, off);
        x = kMax ? fmaxf(x, ox) : x + ox;
        y = kMax ? fmaxf(y, oy) : y + oy;
    }
    if (lane == 0) {
        sm.red[0][warp] = x;
        sm.red[1][warp] = y;
    }
    __syncthreads();
    x = sm.red[0][0];
    y = sm.red[1][0];
#pragma unroll
    for (int w = 1; w < kLagThreads / 32; ++w) {
        x = kMax ? fmaxf(x, sm.red[0][w]) : x + sm.red[0][w];
        y = kMax ? fmaxf(y, sm.red[1][w]) : y + sm.red[1][w];
    }
    __syncthreads();  // sm.red is reused by the next reduction
}

// One segment: the statistics of partition c1, then partitions c1 - 1 ... c0 scored.
template <typename T, int LPR>
__device__ __forceinline__ void score_segment(const LagArgs& a, int row, int seg, LagSmem& sm) {
    constexpr int RPC = kLagThreads / LPR;  // rows per pass of the CTA
    constexpr int U = 2;                    // passes in flight per load batch
    const int tid = threadIdx.x;
    const int sub = tid % LPR, rsel = tid / LPR;
    const int b = row / a.H, h = row % a.H;
    const bool lane_ok = sub < (a.D >> 3);
    const T* Kb = static_cast<const T*>(a.K) + (int64_t)b * a.ks.b + (int64_t)h * a.ks.h + sub * 8;
    const T* Vb = static_cast<const T*>(a.V) + (int64_t)b * a.vs.b + (int64_t)h * a.vs.h + sub * 8;
    const int L = a.L;
    const int c0 = seg * a.seg_len;
    const int c1 = min(c0 + a.seg_len, a.n_scored);

    // the reference partition holds a NaN: torch.min / max propagate it, so every sigma it scores is NaN
    int ref_nan = 0;
    for (int c = c1; c >= c0; --c) {
        const bool score = c < c1;  // uniform over the CTA
        const int p0 = a.n_sink + c * L;
        float lk[8], hk[8], lv[8], hv[8];  // the reference statistics (c + 1)
        float nlk[8], nhk[8], nlv[8], nhv[8];  // this partition's (fminf / fmaxf skip NaN: it is flagged apart)
        bool has_nan = false;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int d = (sub * 8 + j) & 255;
            lk[j] = sm.stat[0][d];
            hk[j] = sm.stat[1][d];
            lv[j] = sm.stat[2][d];
            hv[j] = sm.stat[3][d];
            nlk[j] = nlv[j] = INFINITY;
            nhk[j] = nhv[j] = -INFINITY;
        }
#pragma unroll 1
        for (int r0 = 0; r0 < L; r0 += RPC * U) {
            int4 wk[U], wv[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int r = r0 + u * RPC + rsel;
                wk[u] = wv[u] = make_int4(0, 0, 0, 0);
                if (r < L && lane_ok) {
                    wk[u] = ldg_plain(Kb + (int64_t)(p0 + r) * a.ks.s);
                    wv[u] = ldg_plain(Vb + (int64_t)(p0 + r) * a.vs.s);
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int r = r0 + u * RPC + rsel;
                float k[8], v[8];
                unpack8<T>(wk[u], k);
                unpack8<T>(wv[u], v);
                if (r < L && lane_ok) {
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        nlk[j] = fminf(nlk[j], k[j]);
                        nhk[j] = fmaxf(nhk[j], k[j]);
                        nlv[j] = fminf(nlv[j], v[j]);
                        nhv[j] = fmaxf(nhv[j], v[j]);
                        has_nan |= isnan(k[j]) || isnan(v[j]);
                    }
                }
                if (score) {
                    const float sk = row_sigma<LPR>(k, lk, hk, lane_ok, a.D);
                    const float sv = row_sigma<LPR>(v, lv, hv, lane_ok, a.D);
                    if (sub == 0 && r < L) {
                        sm.sk[r] = sk;
                        sm.sv[r] = sv;
                    }
                }
            }
        }
        // this partition's min / max: lanes of one channel group meet (xor over the row-select bits), then the warps
        // through integer atomics
#pragma unroll
        for (int off = LPR; off < 32; off <<= 1)
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                nlk[j] = fminf(nlk[j], __shfl_xor_sync(0xFFFFFFFFu, nlk[j], off));
                nhk[j] = fmaxf(nhk[j], __shfl_xor_sync(0xFFFFFFFFu, nhk[j], off));
                nlv[j] = fminf(nlv[j], __shfl_xor_sync(0xFFFFFFFFu, nlv[j], off));
                nhv[j] = fmaxf(nhv[j], __shfl_xor_sync(0xFFFFFFFFu, nhv[j], off));
            }
        if ((tid & 31) < LPR && lane_ok)
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int d = sub * 8 + j;
                atomicMin(&sm.next[0][d], f2o(nlk[j]));
                atomicMax(&sm.next[1][d], f2o(nhk[j]));
                atomicMin(&sm.next[2][d], f2o(nlv[j]));
                atomicMax(&sm.next[3][d], f2o(nhv[j]));
            }
        const int this_nan = __syncthreads_or(has_nan);
        // publish them as the reference of c - 1 (every thread has read sm.stat above)
        if (tid < a.D) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                sm.stat[i][tid] = o2f(sm.next[i][tid]);
                sm.next[i][tid] = (i & 1) ? f2o(-INFINITY) : f2o(INFINITY);
            }
        }
        if (score) {
            // softmax of sigma_k and sigma_v over the L rows; a NaN sigma makes every c of the partition NaN
            float mk = -INFINITY, mv = -INFINITY;
            bool nan = ref_nan;
            for (int t = tid; t < L; t += kLagThreads) {
                const float sk = sm.sk[t], sv = sm.sv[t];
                nan |= isnan(sk) || isnan(sv);
                mk = fmaxf(mk, sk);
                mv = fmaxf(mv, sv);
            }
            nan = __syncthreads_or(nan);
            block_reduce2<true>(mk, mv, sm);
            float zk = 0.f, zv = 0.f;
            for (int t = tid; t < L; t += kLagThreads) {
                zk += expf(sm.sk[t] - mk);
                zv += expf(sm.sv[t] - mv);
            }
            block_reduce2<false>(zk, zv, sm);
            uint32_t* keys = reinterpret_cast<uint32_t*>(sm.sv);
            for (int t = tid; t < L; t += kLagThreads) {
                const float ak = expf(sm.sk[t] - mk) / zk, av = expf(sm.sv[t] - mv) / zv;
                const float cs = nan ? __int_as_float(0x7FFFFFFF) : (ak + av) * 0.5f;
                sm.sk[t] = cs;
                keys[t] = rank_key(cs);
            }
            __syncthreads();
            for (int base = 0; base < L; base += kLagThreads) {
                const int s = base + tid;
                const bool valid = s < L;
                float value = 0.f;
                if (valid) {
                    if (a.cross) {
                        value = sm.sk[s];
                    } else {
                        const uint32_t ks = keys[s];
                        int r = 0;
#pragma unroll 4
                        for (int t = 0; t < L; ++t) {
                            const uint32_t kt = keys[t];
                            r += (kt < ks) | ((kt == ks) & (t < s));
                        }
                        value = (float)r / (float)L;
                    }
                }
                emit<T>(a, row, p0 + s, valid, value, sm.hist);
            }
        }
        ref_nan = this_nan;
        __syncthreads();
    }
}

template <typename T, int LPR>
__global__ void __launch_bounds__(kLagThreads, 2) lagkv_kernel(LagArgs a) {
    __shared__ LagSmem sm;
    const int item = blockIdx.x, row = blockIdx.y;
    const int tid = threadIdx.x;
    sm.hist[tid] = 0;
    if (tid < 256)
#pragma unroll
        for (int i = 0; i < 4; ++i) sm.next[i][tid] = (i & 1) ? f2o(-INFINITY) : f2o(INFINITY);
    pdl_launch_dependents();  // the select+compact kernel behind this one may start to take residency
    __syncthreads();
    if (item < a.n_seg) {
        score_segment<T, LPR>(a, row, item, sm);
    } else {
        // 256 positions of [0, end_a) or [tail_start, fill_end)
        const int f = item - a.n_seg;
        const int begin = f < a.n_fill_a ? f * kLagThreads : a.tail_start + (f - a.n_fill_a) * kLagThreads;
        const int end = f < a.n_fill_a ? a.end_a : a.fill_end;
        const int s = begin + tid;
        float value = 1.f;
        if (a.n_scored == 0 && s >= a.n_sink) value = (float)(s - a.n_sink) / (float)(a.S - a.n_sink);
        emit<T>(a, row, s, s < end, value, sm.hist);
    }
    if (a.want_keys) {
        __syncthreads();
        flush_row_hist(sm.hist, row, a.ws);
    }
}

template <typename T>
static cudaError_t launch_lagkv_t(const LagArgs& a, int R, int n_items, cudaStream_t st) {
    const dim3 grid(n_items, R);
    with_lanes_per_row(a.D, [&](auto lpr) { lagkv_kernel<T, lpr><<<grid, kLagThreads, 0, st>>>(a); });
    return cudaPeekAtLastError();
}

cudaError_t launch_lagkv_score(const Dims& d, int dtype, const void* K, const void* V, int n_sink, int lag_size,
                               int cross, const Workspace& ws, void* scores_out, bool want_keys, cudaStream_t st) {
    if (d.D > 256 || lag_size < 1 || lag_size > kLagMax || n_sink < 0) return cudaErrorNotSupported;
    LagArgs a = {};
    a.K = K;
    a.V = V;
    a.ks = d.ks;
    a.vs = d.vs;
    a.H = d.H;
    a.S = d.S;
    a.D = d.D;
    a.n_sink = n_sink;
    a.L = lag_size;
    a.cross = cross ? 1 : 0;
    a.ws = ws;
    a.scores_out = static_cast<uint16_t*>(scores_out);
    a.want_keys = want_keys ? 1 : 0;
    a.fill_end = want_keys ? ws.S_pad : d.S;
    int n_items;
    if ((int64_t)d.S < (int64_t)n_sink + 2 * (int64_t)lag_size) {  // short cache: one ramp
        a.n_scored = a.seg_len = a.n_seg = 0;
        a.end_a = a.tail_start = a.fill_end;
        a.n_fill_a = (a.fill_end + kLagThreads - 1) / kLagThreads;
        n_items = a.n_fill_a;
    } else {
        const int P = (d.S - n_sink) / lag_size;
        a.n_scored = P - 1;
        const int target = kLagItemsPerSm * device_sm_count();
        const int per_row = min(a.n_scored, max(1, (target + d.R - 1) / d.R));
        a.seg_len = (a.n_scored + per_row - 1) / per_row;
        a.n_seg = (a.n_scored + a.seg_len - 1) / a.seg_len;
        a.end_a = n_sink;
        a.n_fill_a = (n_sink + kLagThreads - 1) / kLagThreads;
        a.tail_start = n_sink + (P - 1) * lag_size;
        n_items = a.n_seg + a.n_fill_a + (a.fill_end - a.tail_start + kLagThreads - 1) / kLagThreads;
    }
    return with_dtype(dtype, [&](auto t) { return launch_lagkv_t<decltype(t)>(a, d.R, n_items, st); });
}

}  // namespace kvp
