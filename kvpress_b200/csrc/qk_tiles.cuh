// qk_tiles.cuh — the sm_90a building blocks of the two query-key attention scorers (snapkv.cu,
// observed_attention.cu): 128-key tiles, the resident-Q / streamed-K shared-memory layout, one K-major
// wgmma product per 64-row block, and the MUFU exp2.
#pragma once
#include "common.cuh"
#include "umma.cuh"

namespace kvp {

constexpr int kSnTile = 128;
constexpr int kSnThreads = 384;  // warpgroup 0: TMA producer (one thread); warpgroups 1, 2: wgmma + epilogue
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
    static constexpr int kFit = (227 * 1024 - 1024 - kQBytes - kCbBytes - 256) / kStageBytes;
    static constexpr int kStages = kFit >= 4 ? 4 : kFit;
    static_assert(kStages >= 2, "K ring needs two stages");
    static constexpr int kQOff = 0;
    static constexpr int kStageOff = kQBytes;
    static constexpr int kCbOff = kStageOff + kStages * kStageBytes;
    static constexpr int kBarOff = kCbOff + kCbBytes;
    static constexpr int kTotal = kBarOff + 256;
    static_assert(kTotal + 1024 <= 227 * 1024, "shared memory budget");
};

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

}  // namespace kvp
