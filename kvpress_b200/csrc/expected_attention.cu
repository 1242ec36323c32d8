// expected_attention.cu — stage S for ExpectedAttentionPress (sm_90a: TMA + wgmma).
//
// Reference semantics (kvpress/presses/expected_attention_press.py:136-165), per kv head h and each
// of its G = Hq/Hkv query heads g, over positions s in [n_sink, S):
//     logit_g(s) = mu_g . k_s / sqrt(d) + k_s^T Sigma_g k_s / (2 d)              (:149-151)
//     p_g        = softmax_s(logit_g)                                              (:152)
//     score(s)   = mean_g p_g(s)          [* ||v_s||_2 after adding epsilon]       (:155-160)
//   and the n_sink first positions are forced to be kept (:163).
// The reference materialises repeat_kv(K)^T twice and a [B,Hq,D,S] einsum intermediate; here
//   kernel 1 (ea_logits_kernel, persistent, one CTA per SM, warp-specialised):
//       TMA streams 128-position K tiles (SWIZZLE_128B) into a ring; two consumer warpgroups compute
//       Y = K_tile[64 x D] * Sigma_g^T per head with wgmma (K rows from registers, accumulators in registers) and
//       finish logit = sum_n k_n (Y_n + 2 sqrt(d) mu_n) / (2d) with the same k registers,
//       keep online softmax statistics and store fp32 logits. Sigma of up to four heads (the unit) stays resident
//       in shared memory while the CTA works on that unit.
//       Three otherwise idle warps of the producer warpgroup stream V next to the MMAs and write ||v_s||.
//   kernel 2 (ea_finalize_kernel): combines the per-CTA softmax statistics, forms the final score in
//       fp32, rounds it ONCE to the cache dtype, and emits keys + histogram for the select stage.
// Covariance-free mode (use_covariance=False) is a plain streaming GEMV kernel that also writes ||v_s||.
#include <stdlib.h>

#include "common.cuh"
#include "knorm_chunk.cuh"
#include "umma.cuh"

namespace kvp {

constexpr int kEaTile = 128;      // key rows per MMA tile (M)
constexpr int kEaMaxParts = 160;  // upper bound on CTAs per (b,h) row (>= SM count)
constexpr int kEaVnormLoads = 8;  // 16-byte V loads in flight per lane of a value-norm warp

struct EaScratch {
    float* logits;    // [R][G][S_pad]
    float* vnorm;     // [R][S_pad]
    float2* partial;  // [R][G][n_parts] (max, sum exp) per CTA part
};

// The scratch in ws.scorer; with a null base only its size (*bytes).
static EaScratch carve_ea(const Dims& d, void* base, size_t* bytes = nullptr) {
    const int G = d.Hq / d.H;
    const size_t S_pad = (size_t)((d.S + kTile - 1) / kTile) * kTile;
    const size_t n_parts = (size_t)((d.S + kScoreChunkGeneric - 1) / kScoreChunkGeneric);
    Carve c(base);
    EaScratch s;
    s.logits = c.take<float>((size_t)d.R * G * S_pad);
    s.vnorm = c.take<float>((size_t)d.R * S_pad);
    s.partial = c.take<float2>((size_t)d.R * G * (n_parts > kEaMaxParts ? n_parts : kEaMaxParts));
    if (bytes) *bytes = c.bytes;
    return s;
}

size_t ea_scratch_bytes(const Dims& d) {
    size_t bytes;
    carve_ea(d, nullptr, &bytes);
    return bytes;
}

// ---- shared-memory carve-up of ea_logits_kernel ---------------------------------------------------
template <int D, int GR>
struct EaSmem {
    static constexpr int kPanels = D / 64;                 // 64-element (128 B) K panels
    static constexpr int kCovHeadPanel = D * 128;          // bytes of one head's [D x 64] panel
    static constexpr int kCovBytes = GR * kPanels * kCovHeadPanel;
    static constexpr int kStageBytes = kPanels * kEaTile * 128;
    static constexpr int kBiasBytes = GR * D * 4;          // 2 sqrt(d) mu_g in fp32
    static constexpr int kStages = umma::ring_stages(kCovBytes + kBiasBytes + 512, kStageBytes);
    static_assert(kStages >= 2, "K ring needs two stages");
    static constexpr int kCovOff = 0;
    static constexpr int kStageOff = kCovBytes;
    static constexpr int kBiasOff = kStageOff + kStages * kStageBytes;
    static constexpr int kBarOff = kBiasOff + kBiasBytes;
    static constexpr int kTotal = kBarOff + 512;
    static_assert(umma::smem_request(kTotal) <= umma::kSmemBudget, "shared memory budget");
};

// Work: unit = (row, group of GR query heads of its kv head); item = (unit, 128-position tile). The items are cut into
// equal contiguous ranges, one per CTA (a range may cross a unit boundary), so every SM gets the same number of tiles
// whatever the number of rows. Contiguous, balanced item ranges: CTA p owns [ea2_start(p), ea2_start(p + 1)).
__host__ __device__ inline long long ea2_start(int p, long long total, int n_workers) {
    return ((long long)p * total) / n_workers;
}
// the CTA whose (non-empty) range contains `item`
__host__ __device__ inline int ea2_pair_of(long long item, long long total, int n_workers) {
    int p = (int)((item * n_workers) / total);
    if (p >= n_workers) p = n_workers - 1;
    while (p + 1 < n_workers && ea2_start(p + 1, total, n_workers) <= item) ++p;
    while (p > 0 && ea2_start(p, total, n_workers) > item) --p;
    return p;
}

// Host-callable view of the partition for the CPU test of the schedule (tests/test_abi_symbols.py): for `pair` (CTA) of
// `n_pairs` over `n_units` units of `n_tp` items: out4 = {first item, one past the last item}; for `unit`:
// {first CTA that touches it, number of CTAs that touch it}. Returns -1 on bad arguments.
extern "C" int kvp_debug_ea_pair_partition(int n_units, int n_tp, int n_pairs, int pair, int unit, long long* out4) {
    if (n_units < 1 || n_tp < 1 || n_pairs < 1 || out4 == nullptr) return -1;
    const long long total = (long long)n_units * n_tp;
    if ((long long)n_pairs > total || pair < 0 || pair >= n_pairs || unit < 0 || unit >= n_units) return -1;
    out4[0] = ea2_start(pair, total, n_pairs);
    out4[1] = ea2_start(pair + 1, total, n_pairs);
    const int first = ea2_pair_of((long long)unit * n_tp, total, n_pairs);
    out4[2] = first;
    out4[3] = ea2_pair_of((long long)(unit + 1) * n_tp - 1, total, n_pairs) - first + 1;
    return 0;
}

// Warpgroup 0: one thread streams the covariance of the unit's heads (resident for the unit) and the K tiles through a
// ring; warps 1-3 stream the V rows of the CTA's tiles and write ||v_s|| (units with g_off == 0 only, so each row's
// norms are computed once). Consumer warpgroup cw loads its 64 rows of the tile into registers once (ldmatrix),
// releases the stage, computes Y_g = K[64 cw .. 64 cw + 64) * Sigma_g^T per head (wgmma, A from registers,
// accumulators in registers) and finishes logit_g = sum_n k_n (Y_g,n + 2 sqrt(d) mu_g,n) / (2d) with the same k
// registers: the A fragment of k-step kk holds columns 16 kk + 2 qd + {0, 1, 8, 9} of rows r0 and r0 + 8, which are the
// accumulator columns 8 j + 2 qd + {0, 1} for j = 2 kk, 2 kk + 1. A thread holds two rows and D/4 columns; the four
// threads of a row add their partial dot products.
template <typename T, int D, int GR>
__global__ void __launch_bounds__(umma::kTmaCtaThreads, 1)
ea_logits_kernel(const __grid_constant__ CUtensorMap mapK, const __grid_constant__ CUtensorMap mapCov,
                 const T* __restrict__ mu, const T* __restrict__ V, Strides3 vs, int use_vnorm, int H, int Hq, int S,
                 int n_sink, int R, int n_tiles128, int n_workers, int n_parts, EaScratch sc, int S_pad, int g_total,
                 int n_split) {
    using L = EaSmem<D, GR>;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    // dynamic shared memory is only guaranteed 16-B aligned: round up to 1024 B for the swizzle. The pointer is
    // offset from smem_raw (not rebuilt from an integer) so that the compiler still sees shared memory and emits LDS.
    unsigned char* smem = smem_raw + ((1024u - (umma::smem_u32(smem_raw) & 1023u)) & 1023u);
    unsigned char* s_cov = smem + L::kCovOff;
    unsigned char* s_stage = smem + L::kStageOff;
    float* s_bias = reinterpret_cast<float*>(smem + L::kBiasOff);
    auto* k_ring = reinterpret_cast<umma::TmaRing<L::kStages>*>(smem + L::kBarOff);
    uint64_t* cov_full = reinterpret_cast<uint64_t*>(k_ring + 1);
    float* s_red = reinterpret_cast<float*>(cov_full + 1);  // [8 warps][GR heads][2]

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
    const int P = blockIdx.x;

    if (tid == 0) {
        umma::prefetch_tmap(&mapK);
        umma::prefetch_tmap(&mapCov);
        k_ring->init(umma::kTmaConsumerWarps);
        umma::mbar_init(cov_full, 1);
        umma::mbar_fence_init();
    }
    __syncthreads();

    const float inv_2d = 1.0f / (2.0f * (float)D);
    const float bias_scale = 2.0f * sqrtf((float)D);
    const long long total = (long long)R * n_split * n_tiles128;
    const long long i_begin = ea2_start(P, total, n_workers), i_end = ea2_start(P + 1, total, n_workers);

    uint32_t k_it = 0, cov_it = 0;  // pipeline state, carried across units (barriers keep flipping)
    for (long long it = i_begin; it < i_end; ++cov_it) {
        const int unit = (int)(it / n_tiles128);
        const int t_begin = (int)(it - (long long)unit * n_tiles128);
        const int t_end = (int)min((long long)n_tiles128, t_begin + (i_end - it));
        it += t_end - t_begin;
        const int row = unit / n_split, g_off = (unit % n_split) * GR;
        const int b = row / H, h = row % H;
        const int hq0 = b * Hq + h * g_total + g_off;  // first head of the unit in [B*Hq]
        const int n_real = min(GR, g_total - g_off);   // heads of the unit (the last unit of an odd group is short)
        const long long unit_first = (long long)unit * n_tiles128;
        const int first_cta = ea2_pair_of(unit_first, total, n_workers);
        const int part = P - first_cta;                 // this CTA's slot among the unit's softmax partials

        __syncthreads();  // every MMA of the previous unit has completed: s_cov, s_bias, s_red reusable
        for (int n = tid; n < GR * D; n += umma::kTmaCtaThreads)
            s_bias[n] = (n / D < n_real)
                            ? bias_scale * F16Traits<T>::to_float(reinterpret_cast<const uint16_t*>(mu)[(size_t)hq0 * D + n])
                            : 0.f;
        __syncthreads();

        if (wg == 0) {
            if (tid == 0) {
                // ===== TMA producer =====
                umma::mbar_arrive_expect_tx(cov_full, (uint32_t)(n_real * L::kPanels * L::kCovHeadPanel));
                for (int kp = 0; kp < L::kPanels; ++kp)
                    for (int g = 0; g < n_real; ++g)
                        umma::tma_load_3d(s_cov + (kp * GR + g) * L::kCovHeadPanel, &mapCov, cov_full, kp * 64, 0,
                                          hq0 + g);
                for (int t = t_begin; t < t_end; ++t, ++k_it) {
                    const int stage = k_ring->acquire(k_it, L::kStageBytes);
                    for (int kp = 0; kp < L::kPanels; ++kp)
                        umma::tma_load_4d(s_stage + stage * L::kStageBytes + kp * (kEaTile * 128), &mapK,
                                          k_ring->full(stage), kp * 64, t * kEaTile, h, b);
                }
            } else if (warp > 0 && use_vnorm && g_off == 0) {
                // ===== value norms of this CTA's positions of the row, next to the MMAs =====
                row_norm_span<T, D / 8, kEaVnormLoads>(V, vs, b, h, t_begin * kEaTile, min(t_end * kEaTile, S), D,
                                                       sc.vnorm + (size_t)row * S_pad, warp - 1, 3);
            }
        } else {
            // ===== consumers: wgmma + epilogue; thread = rows r0, r0 + 8 of the tile =====
            const int cw = wg - 1, qd = lane & 3;
            const int r0 = cw * 64 + (warp & 3) * 16 + (lane >> 2);
            const int r_ld = cw * 64 + (warp & 3) * 16 + (lane & 15);  // the row this lane addresses for ldmatrix
            float run_m[GR], run_z[GR];
#pragma unroll
            for (int g = 0; g < GR; ++g) {
                run_m[g] = -INFINITY;
                run_z[g] = 0.f;
            }
            umma::mbar_wait(cov_full, cov_it & 1);
            for (int t = t_begin; t < t_end; ++t, ++k_it) {
                const int stage = k_ring->wait(k_it);
                const uint32_t k_base = umma::smem_u32(s_stage + stage * L::kStageBytes);
                uint32_t ka[D / 16][4];  // this warp's 16 rows of the tile: the A fragment of each k-step
#pragma unroll
                for (int kk = 0; kk < D / 16; ++kk)
                    umma::ldmatrix_x4(ka[kk], k_base + (kk >> 2) * (kEaTile * 128) +
                                                  umma::sw128_offset(r_ld, 2 * (kk & 3) + (lane >> 4)));
                k_ring->release(stage);  // the k rows are in registers: hand the stage back before the MMAs
                // Head g's logits are finished (quad sum, scale, store, online max / sum-exp) while the tensor cores
                // work on head g + 1: the MMAs are issued first, then the previous head's finish runs before the wait.
                // Only the last head's finish is exposed. Both rows' shuffles come before the store branch, since a
                // shuffle cannot be scheduled across a divergent branch.
                auto finish = [&](const int g, const float l0, const float l1) {
                    float l[2] = {l0, l1};
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) l[hh] += __shfl_xor_sync(0xFFFFFFFFu, l[hh], 1);
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        l[hh] += __shfl_xor_sync(0xFFFFFFFFu, l[hh], 2);
                        l[hh] *= inv_2d;
                    }
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        const int s = t * kEaTile + r0 + 8 * hh;
                        if (qd == 0 && s >= n_sink && s < S) {
                            sc.logits[((size_t)row * g_total + g_off + g) * S_pad + s] = l[hh];
                            const float m_new = fmaxf(run_m[g], l[hh]);
                            run_z[g] = run_z[g] * __expf(run_m[g] - m_new) + __expf(l[hh] - m_new);
                            run_m[g] = m_new;
                        }
                    }
                };
                float p0 = 0.f, p1 = 0.f;  // head g - 1's partial dot products of rows r0, r0 + 8
#pragma unroll
                for (int g = 0; g < GR; ++g) {
                    if (g >= n_real) continue;  // warpgroup-uniform
                    float acc[D / 2];
                    umma::wgmma_fence();
#pragma unroll
                    for (int kk = 0; kk < D / 16; ++kk) {
                        const int kp = kk >> 2, ks = kk & 3;
                        umma::wgmma_rs<D, F16Traits<T>::kMmaFormat>(
                            acc, ka[kk],
                            umma::smem_desc_sw128(umma::smem_u32(s_cov + (kp * GR + g) * L::kCovHeadPanel) + ks * 32),
                            kk > 0);
                    }
                    umma::wgmma_commit();
                    if (g > 0) finish(g - 1, p0, p1);
                    umma::wgmma_wait_all();
                    float l0 = 0.f, l1 = 0.f;
#pragma unroll
                    for (int j = 0; j < D / 8; ++j) {
                        // columns 8j + 2 qd, +1 of rows r0 (fragment register 0 or 2) and r0 + 8 (1 or 3)
                        const float2 k0 = F16Traits<T>::unpack2(ka[j >> 1][(j & 1) * 2]);
                        const float2 k1 = F16Traits<T>::unpack2(ka[j >> 1][(j & 1) * 2 + 1]);
                        const float2 bb = *reinterpret_cast<const float2*>(&s_bias[g * D + 8 * j + 2 * qd]);
                        l0 = fmaf(k0.x, acc[4 * j] + bb.x, l0);
                        l0 = fmaf(k0.y, acc[4 * j + 1] + bb.y, l0);
                        l1 = fmaf(k1.x, acc[4 * j + 2] + bb.x, l1);
                        l1 = fmaf(k1.y, acc[4 * j + 3] + bb.y, l1);
                    }
                    p0 = l0;
                    p1 = l1;
                    if (g + 1 == n_real) finish(g, l0, l1);
                }
            }
            // ---- warp-level (max, sum-exp) per head -> shared ---------------------------------------------------
#pragma unroll
            for (int g = 0; g < GR; ++g) {
                float m = run_m[g], z = run_z[g];
#pragma unroll
                for (int off = 16; off >= 1; off >>= 1) {
                    const float m2 = __shfl_xor_sync(0xFFFFFFFFu, m, off);
                    const float z2 = __shfl_xor_sync(0xFFFFFFFFu, z, off);
                    const float mn = fmaxf(m, m2);
                    z = (mn == -INFINITY) ? 0.f : z * __expf(m - mn) + z2 * __expf(m2 - mn);
                    m = mn;
                }
                if (lane == 0) {
                    s_red[((warp - 4) * GR + g) * 2] = m;
                    s_red[((warp - 4) * GR + g) * 2 + 1] = z;
                }
            }
        }
        // ---- CTA-level softmax statistics of this CTA's tiles of the unit -> partial[row][g][part] ---------------
        __syncthreads();
        if (tid < n_real) {
            float m = -INFINITY, z = 0.f;
            for (int w = 0; w < 8; ++w) {
                const float m2 = s_red[(w * GR + tid) * 2], z2 = s_red[(w * GR + tid) * 2 + 1];
                const float mn = fmaxf(m, m2);
                z = (mn == -INFINITY) ? 0.f : z * __expf(m - mn) + z2 * __expf(m2 - mn);
                m = mn;
            }
            sc.partial[((size_t)row * g_total + g_off + tid) * n_parts + part] = make_float2(m, z);
        }
        if (part == 0 && tid >= 32 && tid < 32 + n_real) {
            // the unit's first CTA neutralises the slots no CTA of this unit owns (units take a varying number of CTAs)
            const int used = ea2_pair_of(unit_first + n_tiles128 - 1, total, n_workers) - first_cta + 1;
            for (int p = used; p < n_parts; ++p)
                sc.partial[((size_t)row * g_total + g_off + (tid - 32)) * n_parts + p] = make_float2(-INFINITY, 0.f);
        }
    }
}

// ---- covariance-free logits: mu.k / sqrt(d) with plain streaming loads (use_covariance=False); the same CTA
// writes ||v_s|| of its positions first when the score uses the value norms -----------------------------------------
template <typename T, int LPR>
__global__ void __launch_bounds__(256)
ea_mu_logits_kernel(const T* __restrict__ K, Strides3 ks, const T* __restrict__ mu, const T* __restrict__ V,
                    Strides3 vs, int use_vnorm, int H, int Hq, int G, int S, int D, int n_sink, int n_parts,
                    EaScratch sc, int S_pad) {
    __shared__ float s_mu[8 * 256];
    __shared__ float s_red[8][8][2];
    const int chunk = blockIdx.x, row = blockIdx.y, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int b = row / H, h = row % H;
    const int hq0 = b * Hq + h * G;
    const float scale = 1.0f / sqrtf((float)D);
    for (int i = tid; i < G * D; i += 256)
        s_mu[i] = F16Traits<T>::to_float(reinterpret_cast<const uint16_t*>(mu)[(size_t)hq0 * D + i]);
    if (use_vnorm)
        row_norm_span<T, LPR, 8>(V, vs, b, h, chunk * kScoreChunkGeneric, min((chunk + 1) * kScoreChunkGeneric, S), D,
                                 sc.vnorm + (size_t)row * S_pad, warp, 8);
    __syncthreads();
    constexpr int RPW = 32 / LPR;
    constexpr int TOK_PER_WARP = kScoreChunkGeneric / 8;
    constexpr int ITERS = TOK_PER_WARP / RPW;
    constexpr int U = (ITERS < 4) ? ITERS : 4;
    const int sub = lane % LPR, rsel = lane / LPR;
    const int nvec = D >> 3;
    const T* base = K + (int64_t)b * ks.b + (int64_t)h * ks.h + (int64_t)sub * 8;
    const int s_warp = chunk * kScoreChunkGeneric + warp * TOK_PER_WARP;
    float run_m[8], run_z[8];
#pragma unroll
    for (int g = 0; g < 8; ++g) {
        run_m[g] = -INFINITY;
        run_z[g] = 0.f;
    }
#pragma unroll 1
    for (int it = 0; it < ITERS; it += U) {
        int4 v[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int s = s_warp + (it + u) * RPW + rsel;
            v[u] = make_int4(0, 0, 0, 0);
            if (s < S && sub < nvec) v[u] = ldg_plain(base + (int64_t)s * ks.s);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int s = s_warp + (it + u) * RPW + rsel;
            const uint32_t w4[4] = {(uint32_t)v[u].x, (uint32_t)v[u].y, (uint32_t)v[u].z, (uint32_t)v[u].w};
            float kf[8];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2 f = F16Traits<T>::unpack2(w4[j]);
                kf[2 * j] = f.x;
                kf[2 * j + 1] = f.y;
            }
#pragma unroll
            for (int g = 0; g < 8; ++g) {
                if (g < G) {
                    float dot = 0.f;
                    if (sub < nvec) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) dot = fmaf(kf[j], s_mu[g * D + sub * 8 + j], dot);
                    }
#pragma unroll
                    for (int off = LPR / 2; off >= 1; off >>= 1) dot += __shfl_xor_sync(0xFFFFFFFFu, dot, off);
                    const float lg = dot * scale;
                    if (sub == 0 && s >= n_sink && s < S) {
                        sc.logits[((size_t)row * G + g) * S_pad + s] = lg;
                        const float mn = fmaxf(run_m[g], lg);
                        run_z[g] = run_z[g] * __expf(run_m[g] - mn) + __expf(lg - mn);
                        run_m[g] = mn;
                    }
                }
            }
        }
    }
    // merge the per-lane statistics (only lanes with sub == 0 hold any)
#pragma unroll
    for (int g = 0; g < 8; ++g) {
        if (g < G) {
            float m = run_m[g], z = run_z[g];
#pragma unroll
            for (int off = 16; off >= 1; off >>= 1) {
                const float m2 = __shfl_xor_sync(0xFFFFFFFFu, m, off);
                const float z2 = __shfl_xor_sync(0xFFFFFFFFu, z, off);
                const float mn = fmaxf(m, m2);
                z = (mn == -INFINITY) ? 0.f : z * __expf(m - mn) + z2 * __expf(m2 - mn);
                m = mn;
            }
            if (lane == 0) {
                s_red[warp][g][0] = m;
                s_red[warp][g][1] = z;
            }
        }
    }
    __syncthreads();
    if (tid < G) {
        float m = -INFINITY, z = 0.f;
        for (int w = 0; w < 8; ++w) {
            const float m2 = s_red[w][tid][0], z2 = s_red[w][tid][1];
            const float mn = fmaxf(m, m2);
            z = (mn == -INFINITY) ? 0.f : z * __expf(m - mn) + z2 * __expf(m2 - mn);
            m = mn;
        }
        sc.partial[((size_t)row * G + tid) * n_parts + chunk] = make_float2(m, z);
    }
}

// ---- finalize: softmax normalisation, group mean, * ||v||, ONE rounding, keys + histogram -----------
// One CTA = kEaFinalPos consecutive positions of one row, 4 per thread: the G logits and the value norm arrive as
// 128-bit loads (all independent, issued before anything else), 1024 CTAs cover a 128k x 8-head cache in one wave.
constexpr int kEaFinalKpt = 4;
constexpr int kEaFinalPos = kTileThreads * kEaFinalKpt;
template <typename T>
__global__ void __launch_bounds__(kTileThreads)
ea_finalize_kernel(int G, int S, int n_sink, int use_vnorm, float eps, int n_parts, EaScratch sc,
                   Workspace ws, uint16_t* __restrict__ scores_out) {
    constexpr int KPT = kEaFinalKpt;
    __shared__ uint16_t skeys[kEaFinalPos];
    __shared__ uint16_t sscores[kEaFinalPos];
    __shared__ uint32_t shist[256];
    __shared__ float s_m[8], s_iz[8];
    const int chunk = blockIdx.x, row = blockIdx.y, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    shist[tid] = 0;
    pdl_launch_dependents();  // the select+compact kernel behind this one may start to take residency
    const int s0 = chunk * kEaFinalPos + tid * KPT;
    const bool in_pad = s0 < ws.S_pad;  // the padded scratch rows are readable up to S_pad (a multiple of 256)
    // 1. independent loads first: this thread's logits / norms and (warps < G) the per-CTA softmax partials
    float4 lg[8];
#pragma unroll
    for (int g = 0; g < 8; ++g)
        lg[g] = (g < G && in_pad)
                    ? __ldcg(reinterpret_cast<const float4*>(&sc.logits[((size_t)row * G + g) * ws.S_pad + s0]))
                    : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 vn4 = (use_vnorm && in_pad)
                           ? __ldcg(reinterpret_cast<const float4*>(&sc.vnorm[(size_t)row * ws.S_pad + s0]))
                           : make_float4(1.f, 1.f, 1.f, 1.f);
    float pm = -INFINITY, pz = 0.f;
    if (warp < G) {
        for (int p = lane; p < n_parts; p += 32) {
            const float2 q = sc.partial[((size_t)row * G + warp) * n_parts + p];
            const float mn = fmaxf(pm, q.x);
            pz = (mn == -INFINITY) ? 0.f : pz * __expf(pm - mn) + q.y * __expf(q.x - mn);
            pm = mn;
        }
        // 2. exact softmax normalisers of the G heads
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) {
            const float m2 = __shfl_xor_sync(0xFFFFFFFFu, pm, off);
            const float z2 = __shfl_xor_sync(0xFFFFFFFFu, pz, off);
            const float mn = fmaxf(pm, m2);
            pz = (mn == -INFINITY) ? 0.f : pz * __expf(pm - mn) + z2 * __expf(m2 - mn);
            pm = mn;
        }
        if (lane == 0) {
            s_m[warp] = pm;
            s_iz[warp] = 1.0f / pz;
        }
    }
    __syncthreads();
    const float vn[4] = {vn4.x, vn4.y, vn4.z, vn4.w};
    float fmax_valid = -INFINITY;
    score_tile_epilogue<T, KPT, false>(
        skeys, sscores, shist, row, chunk * kEaFinalPos, S, 0, n_sink, ws, scores_out, &fmax_valid, [&](int i, int) {
            float p = 0.f;
#pragma unroll
            for (int g = 0; g < 8; ++g) {
                if (g < G) {
                    const float l = (i == 0) ? lg[g].x : (i == 1) ? lg[g].y : (i == 2) ? lg[g].z : lg[g].w;
                    p += __expf(l - s_m[g]) * s_iz[g];
                }
            }
            p *= (1.0f / (float)G);
            return use_vnorm ? (p + eps) * vn[i] : p;
        });
    publish_max_valid(fmax_valid, ws);
    flush_row_hist(shist, row, ws);
}

// scores_out[..., lo:hi] = round(max_valid_score + 1) — the value the reference pads with
// (expected_attention_press.py:163, snapkv_press.py:103: `scores.max().item() + 1`).
template <typename T>
__global__ void fill_sentinel_kernel(uint16_t* __restrict__ scores_out, int R, int S, int lo, int hi,
                                     const uint32_t* __restrict__ max_slot) {
    const uint32_t ord = *max_slot;
    pdl_launch_dependents();  // the select+compact kernel behind this one may start to take residency
    const float sentinel = ordered_f32_to_float(ord) + 1.0f;
    const uint16_t bits = F16Traits<T>::from_float(sentinel);
    const int width = hi - lo;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < R * width; i += gridDim.x * blockDim.x)
        scores_out[(size_t)(i / width) * S + lo + (i % width)] = bits;
}

cudaError_t launch_fill_sentinel(int dtype, void* scores_out, int R, int S, int lo, int hi,
                                 const Workspace& ws, cudaStream_t st) {
    if (hi <= lo) return cudaSuccess;
    const uint32_t* slot = ws.counters + kCounterMaxSlot(R);
    int blocks = (R * (hi - lo) + 255) / 256;
    if (blocks > 1024) blocks = 1024;
    with_dtype(dtype, [&](auto t) {
        fill_sentinel_kernel<decltype(t)><<<blocks, 256, 0, st>>>(static_cast<uint16_t*>(scores_out), R, S, lo, hi, slot);
    });
    return cudaPeekAtLastError();
}

// ---- host launcher -----------------------------------------------------------------------------------
template <typename T, int D, int GR>
static cudaError_t launch_ea_logits_t(const Dims& d, const void* K, const void* V, const void* mu, const void* cov,
                                      int use_vnorm, int n_sink, const Workspace& ws, const EaScratch& sc,
                                      int* n_parts_out, cudaStream_t st) {
    using L = EaSmem<D, GR>;
    const int n_tiles128 = (d.S + kEaTile - 1) / kEaTile;
    const int g_total = d.Hq / d.H;
    const int n_split = (g_total + GR - 1) / GR;
    const int n_units = d.R * n_split;
    const long long total = (long long)n_units * n_tiles128;
    int n_workers = device_sm_count();
    if (n_workers > kEaMaxParts) n_workers = kEaMaxParts;
    if ((long long)n_workers > total) n_workers = (int)total;  // every CTA owns at least one item
    // slots of the per-CTA softmax partials of a unit: one per CTA that touches it
    int n_parts = 1;
    for (int u = 0; u < n_units; ++u) {
        const int first = ea2_pair_of((long long)u * n_tiles128, total, n_workers);
        const int last = ea2_pair_of((long long)(u + 1) * n_tiles128 - 1, total, n_workers);
        if (last - first + 1 > n_parts) n_parts = last - first + 1;
    }
    *n_parts_out = n_parts;

    CUtensorMap mapK, mapCov;
    cudaError_t e;
    if ((e = make_tmap_cache(&mapK, K, d, d.ks, kEaTile)) != cudaSuccess) return e;
    if ((e = make_tmap_rows(&mapCov, cov, D, D, D, (uint64_t)d.B * d.Hq, (uint64_t)D * D, D)) != cudaSuccess) return e;
    constexpr int smem = umma::smem_request(L::kTotal);
    constexpr auto kern = ea_logits_kernel<T, D, GR>;
    if ((e = ensure_dynamic_smem<kern>(smem)) != cudaSuccess) return e;
    kern<<<n_workers, umma::kTmaCtaThreads, smem, st>>>(mapK, mapCov, static_cast<const T*>(mu),
                                                        static_cast<const T*>(V), d.vs, use_vnorm, d.H, d.Hq, d.S,
                                                        n_sink, d.R, n_tiles128, n_workers, n_parts, sc, ws.S_pad,
                                                        g_total, n_split);
    return cudaPeekAtLastError();
}

template <typename T>
static cudaError_t launch_ea_t(const Dims& d, int dtype, const void* K, const void* V, const void* mu,
                               const void* cov, float eps, int n_sink, int use_vnorm,
                               const Workspace& ws, void* scores_out, cudaStream_t st) {
    const int G = d.Hq / d.H;
    if (G > 8) return cudaErrorNotSupported;
    const EaScratch sc = carve_ea(d, ws.scorer);
    int n_parts = 0;
    cudaError_t e = cudaSuccess;
    // the logits kernels also write the value norms (use_vnorm): V is not touched otherwise and may be null
    if (cov != nullptr) {
        // tensor-core path: head_dim 64 or 128; the G query heads of a kv head are cut into units of four resident
        // heads (Llama-3.1-8B: 4, Llama-3.1-70B: 8), of two for other group sizes (an odd G leaves its last unit one
        // head short: Llama-3.2-3B: 3, Qwen2-7B: 7), of one for G = 1; each unit's covariance is resident in shared
        // memory and the units of a kv head stream the same K tiles (the second reader finds them in L2).
        if (d.D != 128 && d.D != 64) return cudaErrorNotSupported;
        const bool d128 = d.D == 128;
        if (G % 4 == 0)
            e = d128 ? launch_ea_logits_t<T, 128, 4>(d, K, V, mu, cov, use_vnorm, n_sink, ws, sc, &n_parts, st)
                     : launch_ea_logits_t<T, 64, 4>(d, K, V, mu, cov, use_vnorm, n_sink, ws, sc, &n_parts, st);
        else if (G == 1)
            e = d128 ? launch_ea_logits_t<T, 128, 1>(d, K, V, mu, cov, use_vnorm, n_sink, ws, sc, &n_parts, st)
                     : launch_ea_logits_t<T, 64, 1>(d, K, V, mu, cov, use_vnorm, n_sink, ws, sc, &n_parts, st);
        else
            e = d128 ? launch_ea_logits_t<T, 128, 2>(d, K, V, mu, cov, use_vnorm, n_sink, ws, sc, &n_parts, st)
                     : launch_ea_logits_t<T, 64, 2>(d, K, V, mu, cov, use_vnorm, n_sink, ws, sc, &n_parts, st);
    } else {
        n_parts = (d.S + kScoreChunkGeneric - 1) / kScoreChunkGeneric;
        dim3 grid(n_parts, d.R);
        with_lanes_per_row(d.D, [&](auto lpr) {
            ea_mu_logits_kernel<T, lpr><<<grid, 256, 0, st>>>(static_cast<const T*>(K), d.ks, static_cast<const T*>(mu),
                                                              static_cast<const T*>(V), d.vs, use_vnorm, d.H, d.Hq, G,
                                                              d.S, d.D, n_sink, n_parts, sc, ws.S_pad);
        });
        e = cudaPeekAtLastError();
    }
    if (e != cudaSuccess) return e;
    dim3 grid2((d.S + kEaFinalPos - 1) / kEaFinalPos, d.R);
    ea_finalize_kernel<T><<<grid2, kTileThreads, 0, st>>>(G, d.S, n_sink, use_vnorm, eps, n_parts, sc, ws,
                                                          static_cast<uint16_t*>(scores_out));
    e = cudaPeekAtLastError();
    if (e != cudaSuccess) return e;
    if (scores_out != nullptr) e = launch_fill_sentinel(dtype, scores_out, d.R, d.S, 0, n_sink, ws, st);
    return e;
}

cudaError_t launch_ea_score(const Dims& d, int dtype, const void* K, const void* V, const void* mu,
                            const void* cov, float eps, int n_sink, int use_vnorm,
                            const Workspace& ws, void* scores_out, cudaStream_t st) {
    // keys + histogram are always produced; a score-only call skips the select stage
    return with_dtype(dtype, [&](auto t) {
        return launch_ea_t<decltype(t)>(d, dtype, K, V, mu, cov, eps, n_sink, use_vnorm, ws, scores_out, st);
    });
}

}  // namespace kvp
