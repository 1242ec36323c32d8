// non_causal_attention.cu — stage S for NonCausalAttnPress (sm_90a: TMA + wgmma), the attention half of Compactor.
//
// Reference semantics (kvpress/presses/non_causal_attention_press.py), with G = Hq / Hkv, the query heads h = j G + g of
// kv head j and chunks [c cs, (c+1) cs) of the sequence's own positions:
//     y[h, i, s]  = q[h, i] . k[j, s]                     (no 1/sqrt(D) scaling), i and s in the same chunk
//     A[h, s]     = sum_i softmax_s(y[h, i, :])[s]        (non-causal, over the chunk's keys only)
//     x[j, s]     = (1/G) sum_g A[j G + g, s] * ||v[j, s]||_2
//     pooled      = avg_pool1d(x, 3, padding 1, stride 1) (zeros outside [0, S), always / 3)
//     z           = (pooled - mean) / max(std, 1e-6)      (mean, unbiased std over ALL B Hkv S entries)
// The last chunk, when S is not a multiple of cs, is zero-padded to cs rows by the reference and its pad = n_chunks cs
// - S padded keys are NOT masked out: they sit at logit -1e-9, which is 0 to fp32 resolution. Here the K rows past S
// read as zero through the TMA map, so their logits are exactly 0 and they take their share of every valid row's
// normaliser as in the reference. Each of the pad padded query rows spreads a uniform 1/cs over the chunk's keys; those
// rows are not multiplied, their pad / cs is added to every valid key in closed form.
//   nca_colsum_kernel   item = (b, j, chunk c): the K chunk resident, the G heads' Q chunks stream through a TMA ring.
//                       Per head, pass A (Q K^T, 64 query rows x 128 keys per MMA) forms every valid query row's exact
//                       normaliser cb = -(m + log2 Z) in shared memory; pass B recomputes the product transposed (K Q^T,
//                       64 keys x 128 query rows) and each key sums exp2(log2e y + cb) = P over the rows in registers,
//                       over the G heads in order. No atomics. The producer warpgroup's three idle warps compute ||v||.
//   nca_partials_kernel per 256-position tile: pooled, and the fp64 sums of (pooled - p0) and its square (p0 = pooled at
//                       b = j = s = 0: the shift keeps the one-pass variance free of cancellation).
//   nca_stats_kernel    one CTA: the partials in a fixed order -> mean, std.
//   nca_z_kernel        z in fp64, ONE rounding to the cache dtype, keys + histogram for selection.
// The MMA kernel is persistent (one CTA per SM) with one TMA producer thread and two wgmma consumer warpgroups. Items
// are enumerated chunk-major (u = c R + row): every item carries the same work except the last chunk of each row, which
// comes last, so the round-robin deal bounds every CTA's load by the mean plus one item. One CTA owns each item and
// every reduction runs in a fixed order, so two calls give bitwise-equal scores.
#include <algorithm>
#include <type_traits>

#include "knorm_chunk.cuh"
#include "qk_tiles.cuh"

namespace kvp {

constexpr int kNcaVnormLoads = 8;  // 16-byte V loads in flight per lane of a value-norm warp

struct NcaScratch {
    float* colsum;     // [R][S_pad]  (1/G) sum_g A[b, j G + g, s], the padded query rows' pad / cs included
    float* vnorm;      // [R][S_pad]  ||v[b, j, s]||_2
    double* partials;  // [R n_tiles][2] per finalize tile: sum of (pooled - p0) and of its square
    double* stats;     // [2] mean and max(std, 1e-6) of pooled over all R S entries
};

// The scratch in ws.scorer; with a null base only its size (*bytes).
static NcaScratch carve_nca(const Dims& d, void* base, size_t* bytes = nullptr) {
    const size_t n_tiles = (size_t)(d.S + kTile - 1) / kTile, S_pad = n_tiles * kTile;
    Carve c(base);
    NcaScratch s;
    s.colsum = c.take<float>((size_t)d.R * S_pad);
    s.vnorm = c.take<float>((size_t)d.R * S_pad);
    s.partials = c.take<double>((size_t)d.R * n_tiles * 2);
    s.stats = c.take<double>(2);
    if (bytes) *bytes = c.bytes;
    return s;
}

size_t non_causal_attention_scratch_bytes(const Dims& d) {
    size_t bytes;
    carve_nca(d, nullptr, &bytes);
    return bytes;
}

bool non_causal_attention_supported(const Dims& d, int chunk_size) {
    const int G = d.Hq / d.H;
    return (d.D == 64 || d.D == 128) && (chunk_size == 128 || chunk_size == 256) && G >= 1 && G <= 8;
}

// One resident K chunk [CS x D] and a ring of Q chunks, K-major SW128 panels of 64 columns; two buffers of the per-row
// normalisers (consecutive heads alternate, so one consumer may start a head while the other finishes the last one).
template <int D, int CS>
struct NcaSmem {
    static constexpr int kPanels = D / 64;
    static constexpr int kPanel = CS * 128;  // bytes of one 64-column panel of a chunk
    static constexpr int kChunkBytes = kPanels * kPanel;
    static constexpr int kCbBytes = 2 * CS * 4;
    static constexpr int kStages = umma::ring_stages(kChunkBytes + kCbBytes + 256, kChunkBytes);
    static_assert(kStages >= 2, "Q ring needs two stages");
    static constexpr int kKOff = 0;
    static constexpr int kStageOff = kChunkBytes;
    static constexpr int kCbOff = kStageOff + kStages * kChunkBytes;
    static constexpr int kBarOff = kCbOff + kCbBytes;
    static constexpr int kTotal = kBarOff + 256;
    static_assert(umma::smem_request(kTotal) <= umma::kSmemBudget, "shared memory budget");
};

// ---- the column sums -------------------------------------------------------------------------------------------------
// Consumer warpgroup cw owns the 64-row blocks cw, cw + 2, ... of the chunk: as query rows in pass A, as keys in pass B.
// A thread holds rows (16 w + l/4, +8) of a block and 32 of the 128 columns of each product.
template <typename T, int D, int CS>
__global__ void __launch_bounds__(umma::kTmaCtaThreads, 1)
nca_colsum_kernel(const __grid_constant__ CUtensorMap mapK, const __grid_constant__ CUtensorMap mapQ,
                  const T* __restrict__ V, Strides3 vs, int H, int G, int S, int R, int n_chunks, NcaScratch sc,
                  int S_pad) {
    using L = NcaSmem<D, CS>;
    constexpr int kTiles = CS / kSnTile;  // 128-row tiles of a chunk
    constexpr int kMyBlocks = CS / 128;   // 64-row blocks of a chunk per consumer warpgroup
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* smem = umma::smem_align_1024(smem_raw);
    unsigned char* s_k = smem + L::kKOff;
    unsigned char* s_stage = smem + L::kStageOff;
    float* s_cb = reinterpret_cast<float*>(smem + L::kCbOff);
    auto* q_ring = reinterpret_cast<umma::TmaRing<L::kStages>*>(smem + L::kBarOff);
    auto* k_ring = reinterpret_cast<umma::TmaRing<1>*>(q_ring + 1);  // the resident K chunk

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
    if (tid == 0) {
        umma::prefetch_tmap(&mapK);
        umma::prefetch_tmap(&mapQ);
        q_ring->init(umma::kTmaConsumerWarps);
        k_ring->init(umma::kTmaConsumerWarps);
        umma::mbar_fence_init();
    }
    __syncthreads();

    const int n_items = R * n_chunks;
    if (wg == 0) {
        if (tid == 0) {
            // ===== TMA producer =====
            uint32_t q_it = 0, k_it = 0;
            for (int u = blockIdx.x; u < n_items; u += gridDim.x, ++k_it) {
                const int c = u / R, row = u % R;
                const int b = row / H, j = row % H;
                const int n_qt = (min(CS, S - c * CS) + kSnTile - 1) / kSnTile;  // Q tiles holding valid rows
                k_ring->acquire(k_it, L::kChunkBytes);  // key rows past S read as zero
                for (int t = 0; t < kTiles; ++t)
                    for (int kp = 0; kp < L::kPanels; ++kp)
                        umma::tma_load_4d(s_k + kp * L::kPanel + t * kSnTile * 128, &mapK, k_ring->full(0), kp * 64,
                                          c * CS + t * kSnTile, j, b);
                for (int g = 0; g < G; ++g, ++q_it) {
                    const int stage = q_ring->acquire(q_it, (uint32_t)(n_qt * L::kPanels * kSnTile * 128));
                    for (int t = 0; t < n_qt; ++t)
                        for (int kp = 0; kp < L::kPanels; ++kp)
                            umma::tma_load_3d(s_stage + stage * L::kChunkBytes + kp * L::kPanel + t * kSnTile * 128,
                                              &mapQ, q_ring->full(stage), kp * 64, c * CS + t * kSnTile,
                                              (b * H + j) * G + g);
                }
            }
        } else if (warp > 0) {
            // ===== value norms of the items' positions, next to the MMAs =====
            for (int u = blockIdx.x; u < n_items; u += gridDim.x) {
                const int c = u / R, row = u % R;
                row_norm_span<T, D / 8, kNcaVnormLoads>(V, vs, row / H, row % H, c * CS, min(S, (c + 1) * CS), D,
                                                        sc.vnorm + (size_t)row * S_pad, warp - 1, 3);
            }
        }
    } else {
        // ===== consumers =====
        const int cw = wg - 1, w4 = warp & 3, qd = lane & 3;
        const float c2 = kLog2e;  // logits -> log2 domain (the reference does not scale them)
        uint32_t q_it = 0, k_it = 0;
        for (int u = blockIdx.x; u < n_items; u += gridDim.x, ++k_it) {
            const int c = u / R, row = u % R;
            const int n_valid = min(CS, S - c * CS);  // valid rows (queries and keys) of the chunk
            const int n_qt = (n_valid + kSnTile - 1) / kSnTile;
            const uint32_t kbase = umma::smem_u32(s_k);
            k_ring->wait(k_it);
            float tot[kMyBlocks][2];
#pragma unroll
            for (int i = 0; i < kMyBlocks; ++i) tot[i][0] = tot[i][1] = 0.f;
            for (int g = 0; g < G; ++g, ++q_it) {
                float* cb = s_cb + (q_it & 1) * CS;
                const int stage = q_ring->wait(q_it);
                const uint32_t qbase = umma::smem_u32(s_stage + stage * L::kChunkBytes);
                // ---- pass A: every valid query row's max and sum exp2 over all CS keys of the chunk ----
                // Both passes keep their own epilogues rather than qk_tiles.cuh's (no key is masked here): built on
                // those, this kernel measured about 1 % slower at cs = 256 (H100 80GB HBM3, 700 W).
#pragma unroll 1
                for (int i = 0; i < kMyBlocks; ++i) {
                    const int mb = 2 * i + cw;
                    float m[2] = {-INFINITY, -INFINITY}, z[2] = {0.f, 0.f};
                    if (mb * 64 < n_valid) {  // warpgroup-uniform
#pragma unroll 1
                        for (int t = 0; t < kTiles; ++t) {
                            float acc[64];
                            snap_mma<T, D>(acc, qbase + mb * 64 * 128, L::kPanel, kbase + t * kSnTile * 128,
                                           L::kPanel);
#pragma unroll
                            for (int hh = 0; hh < 2; ++hh) {
                                float m16[16];
#pragma unroll
                                for (int jj = 0; jj < 16; ++jj)
                                    m16[jj] = fmaxf(acc[4 * jj + 2 * hh], acc[4 * jj + 2 * hh + 1]);
#pragma unroll
                                for (int jj = 0; jj < 8; ++jj) m16[jj] = fmaxf(m16[jj], m16[jj + 8]);
#pragma unroll
                                for (int jj = 0; jj < 4; ++jj) m16[jj] = fmaxf(m16[jj], m16[jj + 4]);
                                const float m_new =
                                    fmaxf(m[hh], fmaxf(fmaxf(m16[0], m16[2]), fmaxf(m16[1], m16[3])));
                                const float neg = -m_new * c2;
                                float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;  // four independent sum chains
#pragma unroll
                                for (int jj = 0; jj < 16; jj += 2) {
                                    a0 += fast_exp2(fmaf(acc[4 * jj + 2 * hh], c2, neg));
                                    a1 += fast_exp2(fmaf(acc[4 * jj + 2 * hh + 1], c2, neg));
                                    a2 += fast_exp2(fmaf(acc[4 * jj + 4 + 2 * hh], c2, neg));
                                    a3 += fast_exp2(fmaf(acc[4 * jj + 4 + 2 * hh + 1], c2, neg));
                                }
                                z[hh] = z[hh] * fast_exp2((m[hh] - m_new) * c2) + ((a0 + a1) + (a2 + a3));
                                m[hh] = m_new;
                            }
                        }
                    }
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        float mm = m[hh], zz = z[hh];
#pragma unroll
                        for (int o = 1; o <= 2; o <<= 1) {  // the four threads of a row
                            const float m2 = __shfl_xor_sync(0xFFFFFFFFu, mm, o);
                            const float z2 = __shfl_xor_sync(0xFFFFFFFFu, zz, o);
                            const float mn = fmaxf(mm, m2);
                            zz = (mn == -INFINITY) ? 0.f
                                                   : zz * fast_exp2((mm - mn) * c2) + z2 * fast_exp2((m2 - mn) * c2);
                            mm = mn;
                        }
                        const int r = mb * 64 + w4 * 16 + (lane >> 2) + 8 * hh;
                        // padded query rows get -inf: pass B adds nothing for them
                        if (qd == 0) cb[r] = r < n_valid ? -mm * c2 - log2f(zz) : -INFINITY;
                    }
                }
                asm volatile("bar.sync 1, 256;" ::: "memory");  // both consumers' normalisers of this head written
                // ---- pass B: P summed over the valid query rows, per key, transposed product ----
#pragma unroll
                for (int i = 0; i < kMyBlocks; ++i) {
                    const int kb = 2 * i + cw;
                    if (kb * 64 >= n_valid) continue;  // warpgroup-uniform
#pragma unroll 1
                    for (int t = 0; t < n_qt; ++t) {
                        float acc[64];
                        snap_mma<T, D>(acc, kbase + kb * 64 * 128, L::kPanel, qbase + t * kSnTile * 128, L::kPanel);
                        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
                        for (int jj = 0; jj < 16; ++jj) {
                            const float2 cbv = *reinterpret_cast<const float2*>(cb + t * kSnTile + 8 * jj + 2 * qd);
                            a0 += fast_exp2(fmaf(acc[4 * jj], c2, cbv.x));
                            a1 += fast_exp2(fmaf(acc[4 * jj + 1], c2, cbv.y));
                            a2 += fast_exp2(fmaf(acc[4 * jj + 2], c2, cbv.x));
                            a3 += fast_exp2(fmaf(acc[4 * jj + 3], c2, cbv.y));
                        }
                        tot[i][0] += a0 + a1;
                        tot[i][1] += a2 + a3;
                    }
                }
                q_ring->release(stage);
            }
            k_ring->release(0);  // every MMA on the K chunk has completed
            // the padded query rows of a last chunk: pad of them, each 1/CS on every key (exact: CS is a power of 2)
            const float pad_share = (float)max(0, (c + 1) * CS - S) / CS;
#pragma unroll
            for (int i = 0; i < kMyBlocks; ++i) {
                const int kb = 2 * i + cw;
                if (kb * 64 >= n_valid) continue;  // warpgroup-uniform
                float t0 = tot[i][0], t1 = tot[i][1];
#pragma unroll
                for (int o = 1; o <= 2; o <<= 1) {
                    t0 += __shfl_xor_sync(0xFFFFFFFFu, t0, o);
                    t1 += __shfl_xor_sync(0xFFFFFFFFu, t1, o);
                }
                const int r = kb * 64 + w4 * 16 + (lane >> 2);
                float* out = sc.colsum + (size_t)row * S_pad + c * CS;
                if (qd == 0 && r < n_valid) out[r] = t0 / (float)G + pad_share;
                if (qd == 0 && r + 8 < n_valid) out[r + 8] = t1 / (float)G + pad_share;
            }
        }
    }
}

// ---- finalize: pool, global mean / std, z, ONE rounding --------------------------------------------------------------
// pooled[s] = (x[s-1] + x[s] + x[s+1]) / 3 with x = colsum * vnorm and zeros outside [0, S); the same expression in
// both kernels that need it, so they see the same value.
__device__ __forceinline__ float nca_pooled(const NcaScratch& sc, size_t base, int s, int S) {
    const float xm = s > 0 ? sc.colsum[base + s - 1] * sc.vnorm[base + s - 1] : 0.f;
    const float x0 = sc.colsum[base + s] * sc.vnorm[base + s];
    const float xp = s + 1 < S ? sc.colsum[base + s + 1] * sc.vnorm[base + s + 1] : 0.f;
    return ((xm + x0) + xp) / 3.f;
}

// A fixed-order sum over the 256 threads of a CTA (xor tree in each warp, then the eight warp sums in order);
// thread 0 gets the result.
__device__ __forceinline__ double nca_block_sum(double v, double* s_warp) {
    const int tid = threadIdx.x, lane = tid & 31;
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
    __syncthreads();  // s_warp reusable
    if (lane == 0) s_warp[tid >> 5] = v;
    __syncthreads();
    double t = 0.0;
    if (tid == 0)
        for (int w = 0; w < kTileThreads / 32; ++w) t += s_warp[w];
    return t;
}

__global__ void __launch_bounds__(kTileThreads)
nca_partials_kernel(int S, int S_pad, NcaScratch sc) {
    __shared__ double s_warp[kTileThreads / 32];
    const int tile = blockIdx.x, row = blockIdx.y, s = tile * kTile + threadIdx.x;
    const double p0 = nca_pooled(sc, 0, 0, S);
    const double dv = s < S ? (double)nca_pooled(sc, (size_t)row * S_pad, s, S) - p0 : 0.0;
    const double sum = nca_block_sum(dv, s_warp);
    const double sq = nca_block_sum(dv * dv, s_warp);
    if (threadIdx.x == 0) {
        double* part = sc.partials + ((size_t)row * gridDim.x + tile) * 2;
        part[0] = sum;
        part[1] = sq;
    }
}

__global__ void __launch_bounds__(kTileThreads)
nca_stats_kernel(int S, int R, int n_parts, NcaScratch sc) {
    __shared__ double s_warp[kTileThreads / 32];
    double a = 0.0, q = 0.0;
    for (int i = threadIdx.x; i < n_parts; i += kTileThreads) {
        a += sc.partials[2 * (size_t)i];
        q += sc.partials[2 * (size_t)i + 1];
    }
    const double sum = nca_block_sum(a, s_warp);
    const double sq = nca_block_sum(q, s_warp);
    if (threadIdx.x == 0) {
        const double n = (double)R * (double)S;
        const double mean_d = sum / n;
        const double m2 = fmax(sq - sum * mean_d, 0.0);
        double sd = sqrt(m2 / (n - 1.0));  // n == 1: 0 / 0 = NaN, as torch's unbiased std
        if (!isnan(sd)) sd = fmax(sd, 1e-6);
        sc.stats[0] = (double)nca_pooled(sc, 0, 0, S) + mean_d;
        sc.stats[1] = sd;
    }
}

template <typename T>
__global__ void __launch_bounds__(kTileThreads)
nca_z_kernel(int S, NcaScratch sc, Workspace ws, uint16_t* __restrict__ scores_out) {
    __shared__ uint16_t skeys[kTile];
    __shared__ uint16_t sscores[kTile];
    __shared__ uint32_t shist[256];
    const int tile = blockIdx.x, row = blockIdx.y, tid = threadIdx.x;
    shist[tid] = 0;
    pdl_launch_dependents();  // the select+compact kernel behind this one may start to take residency
    score_tile_epilogue<T, 1>(skeys, sscores, shist, row, tile * kTile, S, 0, 0, ws, scores_out, nullptr, [&](int, int s) {
        return (nca_pooled(sc, (size_t)row * ws.S_pad, s, S) - sc.stats[0]) / sc.stats[1];
    });
}

// ---- host launcher ------------------------------------------------------------------------------------------------
template <typename T, int D, int CS>
static cudaError_t launch_nca_t(const Dims& d, const void* K, const void* V, const void* q, const Workspace& ws,
                                void* scores_out, cudaStream_t st) {
    using L = NcaSmem<D, CS>;
    const int sm_count = device_sm_count();
    const int G = d.Hq / d.H;
    const NcaScratch sc = carve_nca(d, ws.scorer);
    const int n_chunks = (d.S + CS - 1) / CS;
    const int grid = (int)std::min<long long>(sm_count, (long long)d.R * n_chunks);

    CUtensorMap mapK, mapQ;
    cudaError_t e;
    if ((e = make_tmap_cache(&mapK, K, d, d.ks, kSnTile)) != cudaSuccess) return e;
    // q [B Hq, S, D] contiguous
    if ((e = make_tmap_rows(&mapQ, q, D, d.S, D, (uint64_t)d.B * d.Hq, (uint64_t)d.S * D, kSnTile)) != cudaSuccess)
        return e;
    constexpr int smem = umma::smem_request(L::kTotal);
    constexpr auto k1 = nca_colsum_kernel<T, D, CS>;
    if ((e = ensure_dynamic_smem<k1>(smem)) != cudaSuccess) return e;

    k1<<<grid, umma::kTmaCtaThreads, smem, st>>>(mapK, mapQ, static_cast<const T*>(V), d.vs, d.H, G, d.S, d.R, n_chunks,
                                                 sc, ws.S_pad);
    if ((e = cudaPeekAtLastError()) != cudaSuccess) return e;
    nca_partials_kernel<<<dim3(ws.n_tiles, d.R), kTileThreads, 0, st>>>(d.S, ws.S_pad, sc);
    if ((e = cudaPeekAtLastError()) != cudaSuccess) return e;
    nca_stats_kernel<<<1, kTileThreads, 0, st>>>(d.S, d.R, ws.n_tiles * d.R, sc);
    if ((e = cudaPeekAtLastError()) != cudaSuccess) return e;
    nca_z_kernel<T><<<dim3(ws.n_tiles, d.R), kTileThreads, 0, st>>>(d.S, sc, ws, static_cast<uint16_t*>(scores_out));
    return cudaPeekAtLastError();
}

template <typename T>
static cudaError_t launch_nca_d(const Dims& d, const void* K, const void* V, const void* q, int chunk_size,
                                const Workspace& ws, void* scores_out, cudaStream_t st) {
    if (!non_causal_attention_supported(d, chunk_size)) return cudaErrorNotSupported;
#define KVP_NCA(DD, CC) \
    if (d.D == DD && chunk_size == CC) return launch_nca_t<T, DD, CC>(d, K, V, q, ws, scores_out, st)
    KVP_NCA(128, 256);
    KVP_NCA(128, 128);
    KVP_NCA(64, 256);
    KVP_NCA(64, 128);
#undef KVP_NCA
    return cudaErrorNotSupported;
}

cudaError_t launch_non_causal_attention_score(const Dims& d, int dtype, const void* K, const void* V, const void* q,
                                              int chunk_size, const Workspace& ws, void* scores_out, cudaStream_t st) {
    return with_dtype(dtype, [&](auto t) { return launch_nca_d<decltype(t)>(d, K, V, q, chunk_size, ws, scores_out, st); });
}

}  // namespace kvp
