// qk_tiles.cuh — the sm_90a building blocks of the tensor-core attention scorers (snapkv.cu, observed_attention.cu,
// non_causal_attention.cu) and of merging.cu's similarity argmax: 128-key tiles, the resident-Q / streamed-K
// shared-memory layout, one K-major wgmma product per 64-row block, the MUFU exp2, and SnapKV's and ObservedAttention's
// softmax epilogues of a product tile: the online (max, sum exp2) of a query row, its four-thread merge, and the column
// sums against normalisers in shared memory.
#pragma once
#include "common.cuh"
#include "umma.cuh"

namespace kvp {

constexpr int kSnTile = 128;
constexpr float kLog2e = 1.4426950408889634f;

__device__ __forceinline__ float fast_exp2(float x) {  // MUFU.EX2, 2 ulp; exp2(-inf) = 0
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// Shared-memory layout shared by both passes. Q is resident ([NQP rows x D], K-major SW128 panels),
// K tiles stream through a ring of kStages.
template <int D, int NQP>
struct SnSmem {
    static constexpr int kPanels = D / 64;
    static constexpr int kQPanel = NQP * 128;             // bytes of one 64-column panel of Q
    static constexpr int kQBytes = kPanels * kQPanel;
    static constexpr int kStageBytes = kPanels * kSnTile * 128;
    static constexpr int kCbBytes = NQP * 4;              // pass 2: per query row -(max + log2 sum) in log2 units
    static constexpr int kStages = umma::ring_stages(kQBytes + kCbBytes + 256, kStageBytes);
    static_assert(kStages >= 2, "K ring needs two stages");
    static constexpr int kQOff = 0;
    static constexpr int kStageOff = kQBytes;
    static constexpr int kCbOff = kStageOff + kStages * kStageBytes;
    static constexpr int kBarOff = kCbOff + kCbBytes;
    static constexpr int kTotal = kBarOff + 256;
    static_assert(umma::smem_request(kTotal) <= umma::kSmemBudget, "shared memory budget");
};

// Query blocks of the scorers whose query rows have positions S - n_q + i (ObservedAttention, Finch): a block holds
// qpos consecutive positions of each of the G query heads of a kv head, resident as G qpos rows.
__host__ __device__ inline int obs_qpos(int G) { return G == 1 ? 128 : 64; }
// The K tiles the block starting at query row p0 sees (causal): keys [0, S - n_q + p0 + qpos), clipped to S.
__host__ __device__ inline int obs_stats_tiles(int S, int n_q, int p0, int qpos) {
    const int end = min(S, S - n_q + p0 + qpos);
    return (end + kSnTile - 1) / kSnTile;
}

// acc[64] (+)= A[64 rows x D] * B[128 rows x D]^T, both K-major SW128 panels (`a_panel` / `b_panel` bytes apart)
template <typename T, int D>
__device__ __forceinline__ void snap_mma(float (&acc)[64], uint32_t a, int a_panel, uint32_t b, int b_panel) {
    umma::wgmma_fence();
#pragma unroll
    for (int k = 0; k < D / 16; ++k) {
        const int kp = k >> 2, kk = k & 3;
        umma::wgmma_ss<128, F16Traits<T>::kMmaFormat>(acc, umma::smem_desc_sw128(a + kp * a_panel + kk * 32),
                                                      umma::smem_desc_sw128(b + kp * b_panel + kk * 32), k > 0);
    }
    umma::wgmma_commit();
    umma::wgmma_wait_all();
}

// Online softmax statistics of one query row against a 128-key tile of a D[qrow, key] product. The thread's 32 logits
// of the row are acc[4 j + 2 hh] and acc[4 j + 2 hh + 1], keys key0 + 8 j and key0 + 8 j + 1; unless `interior`, keys
// past `limit` or past S count as -inf. The running max m is kept in raw logit units (q.k): c > 0 keeps the order and
// folds the scale into one FFMA per element, exp2(fma(y, c, -m c)); z is the running sum of exp2(c (y - m)). While
// every logit of the row seen so far is -inf, (m, z) stay (-inf, 0).
__device__ __forceinline__ void online_row_update(const float (&acc)[64], int hh, float c, bool interior, int key0,
                                                  int limit, int S, float& m, float& z) {
    float v[32];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        v[2 * j] = acc[4 * j + 2 * hh];
        v[2 * j + 1] = acc[4 * j + 2 * hh + 1];
        if (!interior) {
            const int pos = key0 + 8 * j;
            if (pos > limit || pos >= S) v[2 * j] = -INFINITY;
            if (pos + 1 > limit || pos + 1 >= S) v[2 * j + 1] = -INFINITY;
        }
    }
    float m16[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) m16[j] = fmaxf(v[j], v[j + 16]);
#pragma unroll
    for (int j = 0; j < 8; ++j) m16[j] = fmaxf(m16[j], m16[j + 8]);
#pragma unroll
    for (int j = 0; j < 4; ++j) m16[j] = fmaxf(m16[j], m16[j + 4]);
    const float m_new = fmaxf(m, fmaxf(fmaxf(m16[0], m16[2]), fmaxf(m16[1], m16[3])));
    if (m_new > -INFINITY) {
        const float neg = -m_new * c;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;  // four independent sum chains
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
            a0 += fast_exp2(fmaf(v[j], c, neg));
            a1 += fast_exp2(fmaf(v[j + 1], c, neg));
            a2 += fast_exp2(fmaf(v[j + 2], c, neg));
            a3 += fast_exp2(fmaf(v[j + 3], c, neg));
        }
        z = z * fast_exp2((m - m_new) * c) + ((a0 + a1) + (a2 + a3));
        m = m_new;
    }
}

// The four threads that share a row (lanes 4k .. 4k + 3) merge their online (m, z), xor 1 then xor 2; all four end
// with the row's.
__device__ __forceinline__ void quad_merge(float& m, float& z, float c) {
#pragma unroll
    for (int off = 1; off <= 2; off <<= 1) {
        const float m2 = __shfl_xor_sync(0xFFFFFFFFu, m, off);
        const float z2 = __shfl_xor_sync(0xFFFFFFFFu, z, off);
        const float mn = fmaxf(m, m2);
        z = (mn == -INFINITY) ? 0.f : z * fast_exp2((m - mn) * c) + z2 * fast_exp2((m2 - mn) * c);
        m = mn;
    }
}

// Column sums of one D[key, qrow] product tile against per-query-row normalisers cb[0 .. 128) in shared memory
// (cb = -(m + log2 Z) in log2 units, -inf for rows that add nothing): the thread's keys add exp2(c y + cb) = P over its
// 32 query columns 8 j + 2 qd and +1, the first key into tot0, the key 8 rows further into tot1.
__device__ __forceinline__ void colsum_tile(const float (&acc)[64], const float* cb, int qd, float c, float& tot0,
                                            float& tot1) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const float2 cbv = *reinterpret_cast<const float2*>(cb + 8 * j + 2 * qd);
        a0 += fast_exp2(fmaf(acc[4 * j], c, cbv.x));
        a1 += fast_exp2(fmaf(acc[4 * j + 1], c, cbv.y));
        a2 += fast_exp2(fmaf(acc[4 * j + 2], c, cbv.x));
        a3 += fast_exp2(fmaf(acc[4 * j + 3], c, cbv.y));
    }
    tot0 += a0 + a1;
    tot1 += a2 + a3;
}

// The four threads that share a key add their two column sums, xor 1 then xor 2; all four end with the key's.
__device__ __forceinline__ void quad_sum(float& tot0, float& tot1) {
#pragma unroll
    for (int off = 1; off <= 2; off <<= 1) {
        tot0 += __shfl_xor_sync(0xFFFFFFFFu, tot0, off);
        tot1 += __shfl_xor_sync(0xFFFFFFFFu, tot1, off);
    }
}

}  // namespace kvp
