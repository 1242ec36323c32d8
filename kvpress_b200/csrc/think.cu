// think.cu — ThinKPress (reference kvpress/presses/think_press.py; ThinK, https://arxiv.org/abs/2407.21018).
//
// Per row (b, kv head j) with S positions, G = Hq / Hkv and w window-query rows (include/kvpress_b200.h,
// kvp_think_prune):
//   qn(c) = 1/(G w) sum_{g<G} sum_{i<w} q[b, jG+g, i, c]^2,   kn(c) = 1/S sum_s K[b, j, s, c]^2,
//   score(c) = qn(c) kn(c) rounded to fp32; the D - n_pruned largest scores are kept (ties to the lower channel, NaN
//   above every number) and every element of the other channels is set to +0 in place.
//
// Schedule: a memset of the row tickets, then two kernels.
//   1. think_reduce_select_kernel, grid (units, B Hkv), 256 threads. A unit is 256 consecutive positions of a row, so
//      the units depend on S alone. A sub-warp of LPR lanes covers a row with 128-bit loads; each lane sums the squares
//      of its 8 channels over its rows in ascending position (fp32), then the rows of the CTA are summed per channel in
//      ascending row order (fp32) and written as the unit's partial. The CTA that takes a row's last ticket sums the
//      row's partials in ascending unit order in fp64, reads the G w query rows of the kv head (fp64 squares and sums,
//      in a fixed lane / row order), forms the scores and ranks them. It writes the keep bitmask to the workspace and
//      the pruned channels and scores to the caller's outputs when those are non-null.
//   2. think_zero_kernel, launched behind the first by programmatic dependent launch: after pdl_wait() (the first
//      kernel has completed, so K is no longer read), every 16-byte vector of K that holds a pruned channel is read,
//      masked and written back; vectors with no pruned channel are not touched. On the H100 this read-modify-write
//      measured 2.3x faster than 2-byte stores of zeros to the pruned elements alone (DESIGN.md, ThinK).
// Every sum has a fixed order that depends on S, G and w alone, so a row's results are bitwise independent of the SM
// count, of the batch it sits in and of the strides.
#include <math.h>

#include "common.cuh"

namespace kvp {

constexpr int kThinkUnit = 256;     // positions per unit of the reduce kernel and per CTA of the zero kernel
constexpr int kThinkThreads = 256;
constexpr int kThinkMaskWords = 8;  // 256 channels
static_assert(kThinkThreads >= 256, "one thread per channel in the selection");

struct ThinkScratch {
    uint32_t* tickets;  // [R] units of the row done; cleared by the call's memset
    uint32_t* mask;     // [R][8] bit c set: channel c is pruned
    float* partials;    // [R][n_units][D]
};

static int think_units(const Dims& d) { return (d.S + kThinkUnit - 1) / kThinkUnit; }

static ThinkScratch think_scratch(const Dims& d, void* base, size_t* bytes) {
    Carve c(base);
    ThinkScratch sc;
    sc.tickets = c.take<uint32_t>(d.R);
    sc.mask = c.take<uint32_t>((size_t)d.R * kThinkMaskWords);
    sc.partials = c.take<float>((size_t)d.R * think_units(d) * d.D);
    *bytes = c.bytes;
    return sc;
}

size_t think_scratch_bytes(const Dims& d) {
    size_t bytes = 0;
    think_scratch(d, nullptr, &bytes);
    return bytes;
}

struct ThinkArgs {
    const void* K;
    Strides3 ks;
    const void* q;
    int H, G, S, D, w;
    int n_units;
    int n_keep;  // D - n_pruned
    ThinkScratch sc;
    int32_t* pruned_out;
    float* scores_out;
};

template <typename T>
__device__ __forceinline__ void add_squares(const int4& v, float (&acc)[8]) {
    const uint32_t w[4] = {(uint32_t)v.x, (uint32_t)v.y, (uint32_t)v.z, (uint32_t)v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float2 f = F16Traits<T>::unpack2(w[j]);
        acc[2 * j] = fmaf(f.x, f.x, acc[2 * j]);  // the square of a 16-bit value is exact in fp32
        acc[2 * j + 1] = fmaf(f.y, f.y, acc[2 * j + 1]);
    }
}

template <typename T>
__device__ __forceinline__ void add_squares(const int4& v, double (&acc)[8]) {
    const uint32_t w[4] = {(uint32_t)v.x, (uint32_t)v.y, (uint32_t)v.z, (uint32_t)v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float2 f = F16Traits<T>::unpack2(w[j]);
        acc[2 * j] = fma((double)f.x, (double)f.x, acc[2 * j]);
        acc[2 * j + 1] = fma((double)f.y, (double)f.y, acc[2 * j + 1]);
    }
}

template <typename T, int LPR>
__global__ void __launch_bounds__(kThinkThreads) think_reduce_select_kernel(ThinkArgs a) {
    constexpr int kRpp = kThinkThreads / LPR;     // rows per pass of the CTA
    constexpr int kPasses = kThinkUnit / kRpp;    // rows per lane in a unit (= LPR)
    constexpr int kU = kPasses < 8 ? kPasses : 8;  // 128-bit loads in flight per lane
    constexpr int kCols = LPR * 8;
    static_assert(kPasses % kU == 0, "unroll must divide the passes");
    __shared__ double sred[kRpp * kCols];  // per-lane sums: fp32 for K, then fp64 for q
    __shared__ uint32_t skey[256];
    __shared__ uint32_t swarp[kThinkThreads / 32];
    __shared__ int s_last;
    float* sredf = reinterpret_cast<float*>(sred);
    const int tid = threadIdx.x, sub = tid % LPR, rsel = tid / LPR;
    const int unit = blockIdx.x, row = blockIdx.y, b = row / a.H, h = row % a.H;
    const int nvec = a.D >> 3;
    pdl_launch_dependents();  // the zero kernel may take residency; it waits for this grid in pdl_wait()

    // ---- the unit's sum of squares per channel ----
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    if (sub < nvec) {
        const T* base = static_cast<const T*>(a.K) + (int64_t)b * a.ks.b + (int64_t)h * a.ks.h + (int64_t)sub * 8;
        const uint64_t pol = l2_policy_evict_first();
        const int s0 = unit * kThinkUnit + rsel;
#pragma unroll 1
        for (int p = 0; p < kPasses; p += kU) {
            int4 v[kU];
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                const int s = s0 + (p + u) * kRpp;
                v[u] = s < a.S ? ldg_hint(base + (int64_t)s * a.ks.s, pol) : make_int4(0, 0, 0, 0);
            }
#pragma unroll
            for (int u = 0; u < kU; ++u) add_squares<T>(v[u], acc);
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) sredf[rsel * kCols + sub * 8 + j] = acc[j];
    __syncthreads();
    if (tid < a.D) {
        float t = 0.f;
#pragma unroll 4
        for (int r = 0; r < kRpp; ++r) t += sredf[r * kCols + tid];
        a.sc.partials[((size_t)row * a.n_units + unit) * a.D + tid] = t;
    }

    // ---- the last unit of the row finishes it ----
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = atomicAdd(&a.sc.tickets[row], 1u) == (uint32_t)(a.n_units - 1);
    __syncthreads();
    if (!s_last) return;
    __threadfence();

    double kn = 0.0;
    if (tid < a.D) {
        // ascending unit order, 16 loads in flight (L2: the other units' partials bypass this SM's L1)
        const float* p = a.sc.partials + (size_t)row * a.n_units * a.D + tid;
        int u = 0;
        for (; u + 16 <= a.n_units; u += 16) {
            float x[16];
#pragma unroll
            for (int i = 0; i < 16; ++i) x[i] = __ldcg(p + (size_t)(u + i) * a.D);
#pragma unroll
            for (int i = 0; i < 16; ++i) kn += (double)x[i];
        }
        for (; u < a.n_units; ++u) kn += (double)__ldcg(p + (size_t)u * a.D);
        kn /= (double)a.S;
    }

    // the G w query rows of kv head h are consecutive: [b, hG .. hG+G-1, 0 .. w-1]
    double qacc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) qacc[j] = 0.0;
    const int64_t n_rows = (int64_t)a.G * a.w;
    if (sub < nvec) {
        const T* qb = static_cast<const T*>(a.q) + ((int64_t)b * a.H + h) * a.G * a.w * a.D + (int64_t)sub * 8;
        constexpr int kQ = 4;
#pragma unroll 1
        for (int64_t r0 = rsel; r0 < n_rows; r0 += kQ * kRpp) {
            int4 v[kQ];
#pragma unroll
            for (int u = 0; u < kQ; ++u) {
                const int64_t r = r0 + u * kRpp;
                v[u] = r < n_rows ? ldg_plain(qb + r * a.D) : make_int4(0, 0, 0, 0);
            }
#pragma unroll
            for (int u = 0; u < kQ; ++u) add_squares<T>(v[u], qacc);
        }
    }
    __syncthreads();  // sred held the K sums
#pragma unroll
    for (int j = 0; j < 8; ++j) sred[rsel * kCols + sub * 8 + j] = qacc[j];
    __syncthreads();

    float score = 0.f;
    uint32_t key = 0;
    if (tid < a.D) {
        double qn = 0.0;
#pragma unroll 4
        for (int r = 0; r < kRpp; ++r) qn += sred[r * kCols + tid];
        qn /= (double)n_rows;
        score = (float)(qn * kn);
        key = isnan(score) ? 0xFFFFFFFFu : ordered_f32(score);  // NaN above +inf, whatever its sign
        skey[tid] = key;
    }
    __syncthreads();

    // rank = the channels that beat this one: a larger key, or an equal key at a lower channel
    bool pruned = false;
    if (tid < a.D) {
        int rank = 0;
        for (int c = 0; c < a.D; ++c) {
            const uint32_t o = skey[c];
            rank += (o > key) | ((o == key) & (c < tid));
        }
        pruned = rank >= a.n_keep;
        if (a.scores_out) a.scores_out[(size_t)row * a.D + tid] = score;
    }
    const uint32_t bal = __ballot_sync(0xFFFFFFFFu, pruned);
    const int warp = tid >> 5, lane = tid & 31;
    if (lane == 0) {
        swarp[warp] = __popc(bal);
        a.sc.mask[(size_t)row * kThinkMaskWords + warp] = bal;
    }
    __syncthreads();
    if (pruned && a.pruned_out) {
        int pos = __popc(bal & ((1u << lane) - 1u));
        for (int i = 0; i < warp; ++i) pos += swarp[i];
        a.pruned_out[(size_t)row * (a.D - a.n_keep) + pos] = tid;
    }
}

template <typename T, int LPR>
__global__ void __launch_bounds__(kThinkThreads)
think_zero_kernel(void* K, Strides3 ks, int H, int S, int D, const uint32_t* __restrict__ mask) {
    constexpr int kRpp = kThinkThreads / LPR;
    constexpr int kPasses = kThinkUnit / kRpp;
    constexpr int kU = kPasses < 8 ? kPasses : 8;
    const int tid = threadIdx.x, sub = tid % LPR, rsel = tid / LPR;
    const int row = blockIdx.y, b = row / H, h = row % H;
    pdl_wait();  // the reduce kernel has completed: its mask is visible and K is no longer read
    if (sub >= (D >> 3)) return;
    const uint32_t bits = (mask[(size_t)row * kThinkMaskWords + (sub >> 2)] >> ((sub & 3) * 8)) & 0xFFu;
    if (bits == 0) return;
    uint32_t keep[4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
        keep[j] = (((bits >> (2 * j)) & 1u) ? 0u : 0x0000FFFFu) | (((bits >> (2 * j + 1)) & 1u) ? 0u : 0xFFFF0000u);
    T* base = static_cast<T*>(K) + (int64_t)b * ks.b + (int64_t)h * ks.h + (int64_t)sub * 8;
    const int s0 = blockIdx.x * kThinkUnit + rsel;
#pragma unroll 1
    for (int p = 0; p < kPasses; p += kU) {
        int4 v[kU];
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            const int s = s0 + (p + u) * kRpp;
            v[u] = make_int4(0, 0, 0, 0);
            if (s < S) v[u] = *reinterpret_cast<const int4*>(base + (int64_t)s * ks.s);
        }
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            const int s = s0 + (p + u) * kRpp;
            if (s < S) {
                const int4 m = make_int4((int)((uint32_t)v[u].x & keep[0]), (int)((uint32_t)v[u].y & keep[1]),
                                         (int)((uint32_t)v[u].z & keep[2]), (int)((uint32_t)v[u].w & keep[3]));
                *reinterpret_cast<int4*>(base + (int64_t)s * ks.s) = m;
            }
        }
    }
}

template <typename T, int LPR>
static cudaError_t launch_think_t(const ThinkArgs& a, const Dims& d, void* K, cudaStream_t st) {
    const dim3 grid(a.n_units, d.R);
    think_reduce_select_kernel<T, LPR><<<grid, kThinkThreads, 0, st>>>(a);
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) return e;
    return launch_pdl(think_zero_kernel<T, LPR>, grid, dim3(kThinkThreads), 0, st, K, d.ks, d.H, d.S, d.D,
                      static_cast<const uint32_t*>(a.sc.mask));
}

cudaError_t launch_think_prune(const Dims& d, int dtype, void* K, const void* q, int window, int n_pruned,
                               int32_t* pruned_out, float* scores_out, void* scratch, cudaStream_t st) {
    size_t bytes = 0;
    ThinkArgs a = {};
    a.sc = think_scratch(d, scratch, &bytes);
    a.K = K;
    a.ks = d.ks;
    a.q = q;
    a.H = d.H;
    a.G = d.Hq / d.H;
    a.S = d.S;
    a.D = d.D;
    a.w = window;
    a.n_units = think_units(d);
    a.n_keep = d.D - n_pruned;
    a.pruned_out = pruned_out;
    a.scores_out = scores_out;
    cudaError_t e = cudaMemsetAsync(a.sc.tickets, 0, (size_t)d.R * sizeof(uint32_t), st);
    if (e != cudaSuccess) return e;
    return with_dtype(dtype, [&](auto t) {
        cudaError_t r = cudaSuccess;
        with_lanes_per_row(d.D, [&](auto lpr) { r = launch_think_t<decltype(t), lpr>(a, d, K, st); });
        return r;
    });
}

}  // namespace kvp
