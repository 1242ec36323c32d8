// knorm_chunk.cuh — scoring of one 256-position chunk of one (b, h) row for KnormPress, shared by the
// standalone score kernel (knorm.cu) and the fused persistent Knorm kernel (select_compact.cu).
#pragma once
#include "common.cuh"

namespace kvp {

constexpr int kScoreChunk = 256;  // positions per score work item (== kTile)
static_assert(kScoreChunk == kTile, "score chunks and select tiles share the key layout");


// Sum of `v[u]` over the LPR lanes of a row group for the U rows a lane batch covers, WITHOUT reducing every row on
// every lane: a butterfly that halves the number of live values per step ("transpose-reduce"). Step with lane mask m:
// a lane keeps the upper half of its values if (sub & m), the lower half otherwise, sends the other half to its
// partner and adds what it receives. After min(log2 LPR, log2 U) steps a lane holds U / 2^steps totals-so-far; masks
// that are left reduce plainly. On return slot i of lane `sub` holds the full sum of row `row_of(sub) + i` for
// i < kSlots, and only lanes with (sub & kIdleMask) == 0 need to finish it: 8 shuffles instead of 32 per 8 rows of
// head_dim 128, and the sqrt / rounding / key tail runs once per lane batch with every active lane on a different row
// (the score kernels are co-limited by issue slots).
template <int LPR, int U>
struct RowSums {
    static constexpr int log2c(int x) { return x <= 1 ? 0 : 1 + log2c(x / 2); }
    static constexpr int kT = log2c(LPR) < log2c(U) ? log2c(LPR) : log2c(U);  // transpose steps
    static constexpr int kSlots = U >> kT;                                     // rows a lane ends up with
    static constexpr int kIdleMask = (LPR >> kT) - 1;                          // lanes with these bits set hold copies
    __device__ __forceinline__ static int row_of(int sub) {
        int u = 0;
#pragma unroll
        for (int t = 0; t < kT; ++t)
            if (sub & (LPR >> (t + 1))) u += U >> (t + 1);
        return u;
    }
    __device__ __forceinline__ static void reduce(float (&v)[U], int sub) {
#pragma unroll
        for (int t = 0; t < kT; ++t) {
            const int m = LPR >> (t + 1), half = U >> (t + 1);
            const bool upper = (sub & m) != 0;
#pragma unroll
            for (int i = 0; i < half; ++i) {
                const float send = upper ? v[i] : v[i + half];
                const float keep = upper ? v[i + half] : v[i];
                v[i] = keep + __shfl_xor_sync(0xFFFFFFFFu, send, m);
            }
        }
#pragma unroll
        for (int m = (LPR >> kT) / 2; m >= 1; m >>= 1)
#pragma unroll
            for (int i = 0; i < kSlots; ++i) v[i] += __shfl_xor_sync(0xFFFFFFFFu, v[i], m);
    }
};

// Writes -||k_s||_2 (rounded once to the storage dtype) and its ordered key for the 256 positions of
// `chunk` into shared memory. 256 threads; a sub-warp of LPR lanes per 2*D-byte row, U independent
// 128-bit loads in flight per lane. Caller synchronises before reading skeys / sscores.
// kEvictLast: the loads carry an L2 evict_last hint (rows that the compaction stage re-reads soon: they should survive
// in the 126 MB L2); otherwise they carry no hint.
template <typename T, int LPR, bool kEvictLast = false>
__device__ __forceinline__ void knorm_score_chunk(const T* __restrict__ K, Strides3 ks, int b, int h,
                                                  int chunk, int S, int D, uint16_t* skeys,
                                                  uint16_t* sscores) {
    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    constexpr int RPW = 32 / LPR;                                   // rows per warp-wide load
    constexpr int TOK_PER_WARP = kScoreChunk / (kTileThreads / 32);  // 32
    constexpr int ITERS = TOK_PER_WARP / RPW;
    constexpr int U = (ITERS < 8) ? ITERS : 8;  // independent 16-byte loads in flight per lane
    static_assert(ITERS % U == 0, "unroll must divide the iteration count");

    const int sub = lane % LPR;   // which 16-byte piece of the row
    const int rsel = lane / LPR;  // which row of the RPW rows
    const int nvec = D >> 3;      // 16-byte pieces per row
    const T* base = K + (int64_t)b * ks.b + (int64_t)h * ks.h + (int64_t)sub * 8;
    const int s_warp = chunk * kScoreChunk + warp * TOK_PER_WARP;
    const uint64_t pol = kEvictLast ? l2_policy_evict_last() : 0ull;

#pragma unroll 1
    for (int it = 0; it < ITERS; it += U) {
        int4 v[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int s = s_warp + (it + u) * RPW + rsel;
            v[u] = make_int4(0, 0, 0, 0);
            if (s < S && sub < nvec)
                v[u] = kEvictLast ? ldg_hint(base + (int64_t)s * ks.s, pol) : ldg_plain(base + (int64_t)s * ks.s);
        }
        float ssu[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const uint32_t w[4] = {(uint32_t)v[u].x, (uint32_t)v[u].y, (uint32_t)v[u].z,
                                   (uint32_t)v[u].w};
            float s0 = 0.f, s1 = 0.f;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2 f = F16Traits<T>::unpack2(w[j]);
                s0 = fmaf(f.x, f.x, s0);
                s1 = fmaf(f.y, f.y, s1);
            }
            ssu[u] = s0 + s1;
        }
        using RS = RowSums<LPR, U>;
        RS::reduce(ssu, sub);
        if ((sub & RS::kIdleMask) == 0) {
#pragma unroll
            for (int i = 0; i < RS::kSlots; ++i) {
                const int sl = warp * TOK_PER_WARP + (it + RS::row_of(sub) + i) * RPW + rsel;
                // -sqrt(ss) rounded once to the storage dtype (negation is exact)
                const uint16_t bits = F16Traits<T>::from_float(sqrtf(ssu[i])) ^ 0x8000u;
                sscores[sl] = bits;
                skeys[sl] = ordered_key16(bits, F16Traits<T>::kInfBits);
            }
        }
    }
}

// ||x_s||_2 in fp32 of positions [s_begin, s_end) of one (b, h) row, written to out[s]. `n_warps` warps share the span
// (this is warp `wi` of them) in batches of U loads per lane; a sub-warp of LPR lanes covers a 2*D-byte row. Loads are
// L2-evict-first: the rows are read exactly once. Each row's sum of squares is formed as in knorm_score_chunk (per lane
// an even/odd FMA pair over its 8 elements, then the lane tree over xor LPR/2 .. 1 of RowSums), so the norms do not
// depend on U, on the span or on how many warps share it. kSqrt = false writes the sum of squares itself (CUR).
template <typename T, int LPR, int U, bool kSqrt = true>
__device__ __forceinline__ void row_norm_span(const T* __restrict__ X, Strides3 xs, int b, int h, int s_begin,
                                              int s_end, int D, float* __restrict__ out, int wi, int n_warps) {
    const int lane = threadIdx.x & 31;
    constexpr int RPW = 32 / LPR;
    constexpr int kRows = RPW * U;  // rows per warp batch
    const int sub = lane % LPR, rsel = lane / LPR;
    const int nvec = D >> 3;
    const T* base = X + (int64_t)b * xs.b + (int64_t)h * xs.h + (int64_t)sub * 8;
    const uint64_t pol = l2_policy_evict_first();
#pragma unroll 1
    for (int s0 = s_begin + wi * kRows; s0 < s_end; s0 += n_warps * kRows) {
        int4 v[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int s = s0 + u * RPW + rsel;
            v[u] = make_int4(0, 0, 0, 0);
            if (s < s_end && sub < nvec) v[u] = ldg_hint(base + (int64_t)s * xs.s, pol);
        }
        float ssu[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const uint32_t w[4] = {(uint32_t)v[u].x, (uint32_t)v[u].y, (uint32_t)v[u].z, (uint32_t)v[u].w};
            float f0 = 0.f, f1 = 0.f;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2 f = F16Traits<T>::unpack2(w[j]);
                f0 = fmaf(f.x, f.x, f0);
                f1 = fmaf(f.y, f.y, f1);
            }
            ssu[u] = f0 + f1;
        }
        using RS = RowSums<LPR, U>;
        RS::reduce(ssu, sub);
        if ((sub & RS::kIdleMask) == 0) {
#pragma unroll
            for (int i = 0; i < RS::kSlots; ++i) {
                const int s = s0 + (RS::row_of(sub) + i) * RPW + rsel;
                if (s < s_end) out[s] = kSqrt ? sqrtf(ssu[i]) : ssu[i];
            }
        }
    }
}

}  // namespace kvp
