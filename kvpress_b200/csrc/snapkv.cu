// snapkv.cu — stage S for SnapKVPress (sm_90a: TMA + wgmma).
//
// Reference semantics (kvpress/presses/snapkv_press.py:41-105), per kv head h with its G = Hq/Hkv
// query heads and the w = window_size last (RoPE'd) queries of each:
//     logit[r, j] = q_r . k_j / sqrt(d)          r = g*w + i (NQ = G*w query rows), j in [0, S)   (:62)
//     masked where j > S - w + i                  (causal inside the window)                        (:63-65)
//     p[r, :]     = softmax_j(logit[r, :])        (normaliser over ALL S keys)                      (:66)
//     s[j]        = mean_i, then avg_pool1d(kernel, pad=kernel/2, stride 1, /kernel), then mean_g
//                   of p[:, j] for j < S - w                                                         (:95-100)
//   and the last w positions are forced to be kept (:103). mean/pool/mean are linear and commute.
// The reference materialises repeat_kv(K), a [B,Hq,w,S] logit tensor, a mask and an fp32 softmax copy.
// Here K is streamed twice through TMA (second time mostly from L2) and never expanded:
//   pass 1 (snap_stats_kernel)  D[qrow, key] = Q_block[64 x d] * K_tile^T : each query row keeps an
//          online (max, sum exp2) -> per-CTA partials;
//   (each pass-2 CTA first merges the partials into the exact normalisers: cb_r = -m_r - log2 Z_r)
//   pass 2 (snap_colsum_kernel) D[key, qrow] = K_half[64 x d] * Q_chunk^T : each key sums exp2(c * D + cb)
//          over the NQ query rows = sum_r p[r, j] -> fp32 pre-pool scores;
//   finalize (snap_finalize_kernel): 1/(G w) scaling, the 1-D box filter, ONE rounding to the cache
//          dtype, keys + histogram for the select stage.
// Both MMA kernels are persistent (one CTA per SM), warp-specialised: one TMA producer thread and two consumer
// warpgroups that issue wgmma and reduce their register accumulators; while one warpgroup reduces, the other's
// MMAs run.
#include <algorithm>
#include <type_traits>

#include "qk_tiles.cuh"

namespace kvp {

constexpr int kSnMaxParts = 640;

struct SnapScratch {
    float2* partial;  // [R][NQ][n_parts]  (max, sum) in the log2 domain
    float* colsum;    // [R][S_pad]        sum_r p[r, j]
};

// The parts of a row: launch_snap_t splits a row over at most one CTA per 128-key tile, and at most kSnMaxParts.
static int snap_max_parts(const Dims& d) { return std::min(kSnMaxParts, (d.S + kSnTile - 1) / kSnTile); }

// The scratch in ws.scorer; with a null base only its size (*bytes).
static SnapScratch carve_snap(const Dims& d, int window, void* base, size_t* bytes = nullptr) {
    const size_t NQ = (size_t)(d.Hq / d.H) * window;
    const size_t S_pad = (size_t)((d.S + kTile - 1) / kTile) * kTile;
    Carve c(base);
    SnapScratch s;
    s.partial = c.take<float2>((size_t)d.R * NQ * snap_max_parts(d));
    s.colsum = c.take<float>((size_t)d.R * S_pad);
    if (bytes) *bytes = c.bytes;
    return s;
}

size_t snapkv_scratch_bytes(const Dims& d, int window) {
    size_t bytes;
    carve_snap(d, window, nullptr, &bytes);
    return bytes;
}

// Producer of both passes (one thread): the resident Q block of this row, then the K tiles [t_begin, t_end).
template <int D, int NQP>
__device__ __forceinline__ void snap_produce(const CUtensorMap* mapK, const CUtensorMap* mapQ, unsigned char* s_q,
                                             unsigned char* s_stage, umma::TmaRing<SnSmem<D, NQP>::kStages>* k_ring,
                                             uint64_t* q_full, int q_row0, int b, int h, int t_begin, int t_end,
                                             uint32_t& k_it) {
    using L = SnSmem<D, NQP>;
    // all NQP resident rows are loaded (boxes of min(NQP, 256) rows): rows >= NQ belong to the next kv head or lie
    // past the tensor (zero fill); their outputs are never used
    umma::mbar_arrive_expect_tx(q_full, (uint32_t)(L::kPanels * NQP * 128));
    for (int kp = 0; kp < L::kPanels; ++kp)
        for (int r0 = 0; r0 < NQP; r0 += 256)
            umma::tma_load_3d(s_q + kp * L::kQPanel + r0 * 128, mapQ, q_full, kp * 64, q_row0 + r0, 0);
    for (int t = t_begin; t < t_end; ++t, ++k_it) {
        const int stage = k_ring->acquire(k_it, L::kStageBytes);
        for (int kp = 0; kp < L::kPanels; ++kp)
            umma::tma_load_4d(s_stage + stage * L::kStageBytes + kp * (kSnTile * 128), mapK, k_ring->full(stage),
                              kp * 64, t * kSnTile, h, b);
    }
}

// ---- pass 1: per-query-row softmax statistics ---------------------------------------------------------
// Consumer warpgroup cw computes D[qrow, key] for the 64-row blocks mb = cw, cw + 2, ... of Q against every K tile;
// a thread holds rows (16 w + l/4, +8) of a block and 32 of the 128 keys, keeps an online (max, sum exp2) per row,
// and the four threads that share a row merge theirs at the end of the row.
template <typename T, int D, int NQP>
__global__ void __launch_bounds__(umma::kTmaCtaThreads, 1)
snap_stats_kernel(const __grid_constant__ CUtensorMap mapK, const __grid_constant__ CUtensorMap mapQ, int H,
                  int G, int S, int window, int R, int n_tiles128, int ctas_per_row, int n_parts,
                  SnapScratch sc) {
    using L = SnSmem<D, NQP>;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* smem = umma::smem_align_1024(smem_raw);
    unsigned char* s_q = smem + L::kQOff;
    unsigned char* s_stage = smem + L::kStageOff;
    auto* k_ring = reinterpret_cast<umma::TmaRing<L::kStages>*>(smem + L::kBarOff);
    uint64_t* q_full = reinterpret_cast<uint64_t*>(k_ring + 1);

    constexpr int kMyBlocks = NQP / 128;  // 64-row blocks of Q per consumer warpgroup
    const int NQ = G * window;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
    const int n_groups = gridDim.x / ctas_per_row;
    const int group = blockIdx.x / ctas_per_row;
    const int part = blockIdx.x % ctas_per_row;

    if (tid == 0) {
        umma::prefetch_tmap(&mapK);
        umma::prefetch_tmap(&mapQ);
        k_ring->init(umma::kTmaConsumerWarps);
        umma::mbar_init(q_full, 1);
        umma::mbar_fence_init();
    }
    __syncthreads();

    const int tiles_per_part = (n_tiles128 + ctas_per_row - 1) / ctas_per_row;
    const int t_begin = part * tiles_per_part;
    const int t_end = min(n_tiles128, t_begin + tiles_per_part);
    const float c = kLog2e * rsqrtf((float)D);  // logits -> log2 domain

    uint32_t k_it = 0, q_it = 0;
    for (int row = group; row < R; row += n_groups) {
        const int b = row / H, h = row % H;
        const int q_row0 = (b * (H * G) + h * G) * window;  // first of this kv head's NQ rows in q_window
        __syncthreads();  // previous row fully consumed: s_q reusable

        if (wg == 0) {
            if (tid == 0)
                snap_produce<D, NQP>(&mapK, &mapQ, s_q, s_stage, k_ring, q_full, q_row0, b, h, t_begin, t_end, k_it);
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
            for (int t = t_begin; t < t_end; ++t, ++k_it) {
                const int stage = k_ring->wait(k_it);
                const uint32_t kb = umma::smem_u32(s_stage + stage * L::kStageBytes);
                const int key0 = t * kSnTile + 2 * qd;
                const bool interior = (t + 1) * kSnTile <= S - window;  // no masking, all keys valid
#pragma unroll
                for (int i = 0; i < kMyBlocks; ++i) {
                    const int mb = 2 * i + cw;
                    if (mb * 64 >= NQ) continue;  // warpgroup-uniform
                    float acc[64];
                    snap_mma<T, D>(acc, umma::smem_u32(s_q + mb * 64 * 128), L::kQPanel, kb, kSnTile * 128);
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        const int r = mb * 64 + w4 * 16 + (lane >> 2) + 8 * hh;  // query row
                        const int limit = (S - window) + (r % window);          // last visible key position
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
                    if (qd == 0 && r < NQ)
                        sc.partial[((size_t)row * NQ + r) * n_parts + part] = make_float2(m * c, z);  // (max in log2 units, sum)
                }
            }
        }
    }
}

// ---- pass 2: normalised column sums --------------------------------------------------------------------
// Consumer warpgroup cw computes D[key, qrow] for keys [64 cw, 64 cw + 64) of every tile against 128-row chunks of
// Q; a thread holds keys (16 w + l/4, +8) and sums exp2(c y - m_r - log2 Z_r) = p[r, key] over its columns. The four
// threads that share a key add their sums; every key of a tile belongs to exactly one thread.
template <typename T, int D, int NQP>
__global__ void __launch_bounds__(umma::kTmaCtaThreads, 1)
snap_colsum_kernel(const __grid_constant__ CUtensorMap mapK, const __grid_constant__ CUtensorMap mapQ, int H,
                   int G, int S, int window, int R, int n_tiles128, int ctas_per_row, int n_parts,
                   SnapScratch sc, int S_pad) {
    using L = SnSmem<D, NQP>;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* smem = umma::smem_align_1024(smem_raw);
    unsigned char* s_q = smem + L::kQOff;
    unsigned char* s_stage = smem + L::kStageOff;
    float* s_cb = reinterpret_cast<float*>(smem + L::kCbOff);
    auto* k_ring = reinterpret_cast<umma::TmaRing<L::kStages>*>(smem + L::kBarOff);
    uint64_t* q_full = reinterpret_cast<uint64_t*>(k_ring + 1);

    constexpr int kNChunks = NQP / 128;  // 128-column MMAs per tile
    const int NQ = G * window;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
    const int n_groups = gridDim.x / ctas_per_row;
    const int group = blockIdx.x / ctas_per_row;
    const int part = blockIdx.x % ctas_per_row;

    if (tid == 0) {
        umma::prefetch_tmap(&mapK);
        umma::prefetch_tmap(&mapQ);
        k_ring->init(umma::kTmaConsumerWarps);
        umma::mbar_init(q_full, 1);
        umma::mbar_fence_init();
    }
    __syncthreads();

    // only positions < S - window receive a score: tiles beyond are skipped entirely
    const int n_tiles_scored = min(n_tiles128, (S - window + kSnTile - 1) / kSnTile);
    const int tiles_per_part = (n_tiles_scored + ctas_per_row - 1) / ctas_per_row;
    const int t_begin = part * tiles_per_part;
    const int t_end = min(n_tiles_scored, t_begin + tiles_per_part);
    const float c = kLog2e * rsqrtf((float)D);

    uint32_t k_it = 0, q_it = 0;
    for (int row = group; row < R; row += n_groups) {
        const int b = row / H, h = row % H;
        const int q_row0 = (b * (H * G) + h * G) * window;
        __syncthreads();
        for (int n = tid; n < NQP; n += umma::kTmaCtaThreads) {
            // exact normaliser of query row n from the per-CTA partials of pass 1:
            // p[n, j] = exp2(c*y - m) / Z = exp2(c*y + cb),  cb = -m - log2 Z; padding rows (n >= NQ) add exactly 0
            float cb = -INFINITY;
            if (n < NQ) {
                float m = -INFINITY, z = 0.f;
                const float2* part_n = sc.partial + ((size_t)row * NQ + n) * n_parts;
                for (int pp = 0; pp < n_parts; ++pp) {
                    const float2 pz = part_n[pp];
                    const float mn = fmaxf(m, pz.x);
                    z = (mn == -INFINITY) ? 0.f : z * fast_exp2(m - mn) + pz.y * fast_exp2(pz.x - mn);
                    m = mn;
                }
                cb = -m - log2f(z);
            }
            s_cb[n] = cb;
        }
        __syncthreads();

        if (wg == 0) {
            if (tid == 0)
                snap_produce<D, NQP>(&mapK, &mapQ, s_q, s_stage, k_ring, q_full, q_row0, b, h, t_begin, t_end, k_it);
        } else {
            const int cw = wg - 1, w4 = warp & 3, qd = lane & 3;
            umma::mbar_wait(q_full, q_it & 1);
            for (int t = t_begin; t < t_end; ++t, ++k_it) {
                const int stage = k_ring->wait(k_it);
                const uint32_t kb = umma::smem_u32(s_stage + stage * L::kStageBytes) + cw * 64 * 128;
                float tot0 = 0.f, tot1 = 0.f;
#pragma unroll 1
                for (int nc = 0; nc < kNChunks; ++nc) {
                    if (nc * 128 >= NQ) break;  // warpgroup-uniform
                    float acc[64];
                    snap_mma<T, D>(acc, kb, kSnTile * 128, umma::smem_u32(s_q + nc * 128 * 128), L::kQPanel);
                    colsum_tile(acc, s_cb + nc * 128, qd, c, tot0, tot1);
                }
                k_ring->release(stage);
                quad_sum(tot0, tot1);
                const int pos = t * kSnTile + cw * 64 + w4 * 16 + (lane >> 2);
                if (qd == 0 && pos < S - window) sc.colsum[(size_t)row * S_pad + pos] = tot0;
                if (qd == 0 && pos + 8 < S - window) sc.colsum[(size_t)row * S_pad + pos + 8] = tot1;
            }
            ++q_it;
        }
    }
}

// ---- finalize: scaling, box filter, ONE rounding, keys + histogram -------------------------------------
template <typename T>
__global__ void __launch_bounds__(kTileThreads)
snap_finalize_kernel(int S, int window, int kernel_size, float inv_gw, SnapScratch sc, Workspace ws,
                     uint16_t* __restrict__ scores_out) {
    __shared__ uint16_t skeys[kTile];
    __shared__ uint16_t sscores[kTile];
    __shared__ uint32_t shist[256];
    const int tile = blockIdx.x, row = blockIdx.y, tid = threadIdx.x;
    shist[tid] = 0;
    pdl_launch_dependents();  // the select+compact kernel behind this one may start to take residency
    const int n_scored = S - window;
    float fmax_valid = -INFINITY;
    for (int sub = 0; sub < kFinalizeTiles; ++sub) {
        const int t = tile * kFinalizeTiles + sub;
        if (t >= ws.n_tiles) break;
        if (sub > 0) __syncthreads();  // the previous tile's keys and scores are out of skeys / sscores
        score_tile_epilogue<T, 1, false>(skeys, sscores, shist, row, t * kTile, S, n_scored, S, ws, scores_out,
                                         &fmax_valid, [&](int, int s) {
            const int half = kernel_size >> 1;
            float acc = 0.f;
            for (int o = -half; o <= half; ++o) {
                const int j = s + o;
                if (j >= 0 && j < n_scored) acc += sc.colsum[(size_t)row * ws.S_pad + j];
            }
            return acc * inv_gw / (float)kernel_size;  // count_include_pad: always / kernel
        });
    }
    publish_max_valid(fmax_valid, ws);
    flush_row_hist(shist, row, ws);
}

// ---- host launcher -----------------------------------------------------------------------------------------
template <typename T, int D, int NQP>
static cudaError_t launch_snap_t(const Dims& d, int dtype, const void* K, const void* q_window, int window,
                                 int kernel_size, const Workspace& ws, void* scores_out, cudaStream_t st) {
    using L = SnSmem<D, NQP>;
    const int sm_count = device_sm_count();
    const int G = d.Hq / d.H;
    const int NQ = G * window;
    const SnapScratch sc = carve_snap(d, window, ws.scorer);
    const int n_tiles128 = (d.S + kSnTile - 1) / kSnTile;
    int ctas_per_row = sm_count / d.R;
    if (ctas_per_row < 1) ctas_per_row = 1;
    if (ctas_per_row > snap_max_parts(d)) ctas_per_row = snap_max_parts(d);  // the parts carve_snap sized
    int n_groups = sm_count / ctas_per_row;
    if (n_groups > d.R) n_groups = d.R;
    const int grid = n_groups * ctas_per_row;
    const int n_parts = ctas_per_row;  // one (max, sum) per query row and CTA of the row

    CUtensorMap mapK, mapQ;
    cudaError_t e;
    if ((e = make_tmap_cache(&mapK, K, d, d.ks, kSnTile)) != cudaSuccess) return e;
    const uint64_t rows = (uint64_t)d.B * d.Hq * window;
    if ((e = make_tmap_rows(&mapQ, q_window, D, rows, D, 1, rows * D, NQP < 256 ? NQP : 256)) != cudaSuccess) return e;
    constexpr int smem = umma::smem_request(L::kTotal);
    constexpr auto k1 = snap_stats_kernel<T, D, NQP>;
    constexpr auto k2 = snap_colsum_kernel<T, D, NQP>;
    if ((e = ensure_dynamic_smem<k1>(smem)) != cudaSuccess) return e;
    if ((e = ensure_dynamic_smem<k2>(smem)) != cudaSuccess) return e;

    k1<<<grid, umma::kTmaCtaThreads, smem, st>>>(mapK, mapQ, d.H, G, d.S, window, d.R, n_tiles128, ctas_per_row,
                                                 n_parts, sc);
    if ((e = cudaPeekAtLastError()) != cudaSuccess) return e;
    k2<<<grid, umma::kTmaCtaThreads, smem, st>>>(mapK, mapQ, d.H, G, d.S, window, d.R, n_tiles128, ctas_per_row,
                                                 n_parts, sc, ws.S_pad);
    if ((e = cudaPeekAtLastError()) != cudaSuccess) return e;
    dim3 grid3((ws.n_tiles + kFinalizeTiles - 1) / kFinalizeTiles, d.R);
    snap_finalize_kernel<T><<<grid3, kTileThreads, 0, st>>>(d.S, window, kernel_size, 1.0f / (float)NQ, sc, ws,
                                                            static_cast<uint16_t*>(scores_out));
    if ((e = cudaPeekAtLastError()) != cudaSuccess) return e;
    if (scores_out != nullptr)
        e = launch_fill_sentinel(dtype, scores_out, d.R, d.S, d.S - window, d.S, ws, st);
    return e;
}

template <typename T>
static cudaError_t launch_snap_d(const Dims& d, int dtype, const void* K, const void* q_window, int window,
                                 int kernel_size, const Workspace& ws, void* scores_out, cudaStream_t st) {
    const int G = d.Hq / d.H;
    const int NQ = G * window;
    // any group size / window with G * window <= 512 query rows per kv head: the resident Q block is padded to
    // 128 / 256 / 512 rows, padding rows are computed and ignored (Llama-3.2-3B: G = 3, Qwen2-7B: G = 7, ...)
    if (NQ < 1 || NQ > kSnapMaxRows) return cudaErrorNotSupported;
    const int NQP = NQ <= 128 ? 128 : (NQ <= 256 ? 256 : 512);
#define KVP_SNAP(DD, NN) \
    if (d.D == DD && NQP == NN) return launch_snap_t<T, DD, NN>(d, dtype, K, q_window, window, kernel_size, ws, scores_out, st)
    KVP_SNAP(128, 128);
    KVP_SNAP(128, 256);
    KVP_SNAP(128, 512);
    KVP_SNAP(64, 128);
    KVP_SNAP(64, 256);
    KVP_SNAP(64, 512);
#undef KVP_SNAP
    return cudaErrorNotSupported;
}

cudaError_t launch_snapkv_score(const Dims& d, int dtype, const void* K, const void* q_window, int window,
                                int kernel_size, const Workspace& ws, void* scores_out, cudaStream_t st) {
    return with_dtype(dtype, [&](auto t) {
        return launch_snap_d<decltype(t)>(d, dtype, K, q_window, window, kernel_size, ws, scores_out, st);
    });
}

}  // namespace kvp
