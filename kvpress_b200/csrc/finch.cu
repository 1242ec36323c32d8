// finch.cu — stage S for FinchPress (sm_90a: TMA + wgmma).
//
// Reference semantics (kvpress/presses/finch_press.py, FinchPress.score), per (b, kv head j, key s), with G = Hq / Hkv
// and the w window queries (the question after the delimiter) at positions S - w + i, i in [0, w):
//     P[h, i, :]  = softmax over all S keys of q[h, i] . k[j, :] / sqrt(D), causal inside the window
//     c_i         = S - w + i if normalize, else 1
//     score(s)    = (1 / (G w)) sum_g sum_i c_i P[j G + g, i, s]        for the context keys s < S - w
// and the window is forced to be kept (the reference pads it with max + 1). The reference materialises repeat_kv(K),
// a [B, Hq, w, S] logit tensor, a mask and an fp32 softmax copy; here the logits never leave the SMs:
//   pass 1 (finch_stats_kernel)  item = (b, j, block of qpos window positions, part of the block's key tiles), the G
//          heads' rows resident in shared memory; the block's K tiles are split into n_parts ranges so that a short
//          window still spreads over many CTAs; every row keeps an online (max, sum exp2) -> one partial per part.
//   merge (finch_cb_kernel) per window row: the partials in part order -> cb = -(m + log2 Z) + log2 c_i, so that
//          exp2(c y + cb) = c_i P: the weight costs nothing in pass 2.
//   pass 2 (ObservedAttention's column-sum kernel, launch_attention_colsum) over the context key tiles only: every
//          context key is visible to every window row, so no mask applies to the positions that are scored.
//   finalize (finch_finalize_kernel): / (G w), ONE rounding to the cache dtype, keys + histogram for the selection,
//          the window forced; the max + 1 sentinel of scores_out follows (launch_fill_sentinel).
// Every sum has a fixed order that depends only on (S, w, G, D): two calls give bitwise-equal scores, and a row's
// scores do not depend on the batch, the other rows or the SM count.
#include <algorithm>

#include "qk_tiles.cuh"

namespace kvp {

constexpr int kFinchParts = 64;  // target (block, part) items per row of pass 1

struct FinchScratch {
    int32_t* kept;    // [R][S]          chunked selection: the kept positions of a row, in output order
    float2* partial;  // [B Hq][w][P]    (max, sum) per window row and part, log2 units
    float* cb;        // [B Hq][w]       -(max + log2 sum) + log2 c_i
    float* colsum;    // [R][S_pad]      sum_g sum_i c_i P[., s]
};

// Parts of each query block: enough (block, part) items per row to fill the GPU at a short window, never more parts
// than the block has K tiles.
static int finch_parts(int S, int window, int qpos) {
    const int n_blocks = (window + qpos - 1) / qpos;
    const int n_tiles = (S + kSnTile - 1) / kSnTile;
    return std::max(1, std::min(n_tiles, (kFinchParts + n_blocks - 1) / n_blocks));
}

// The scratch in ws.scorer for a window of w rows; with a null base only its size (*bytes). The partials take
// w P <= qpos kFinchParts + w slots per head (P <= kFinchParts / n_blocks + 1, n_blocks >= w / qpos), so the layout
// only grows with w and the largest window, w = S - 1, sizes it for every call.
static FinchScratch carve_finch(const Dims& d, int window, void* base, size_t* bytes = nullptr) {
    const size_t heads = (size_t)d.B * d.Hq;
    const size_t S_pad = (size_t)((d.S + kTile - 1) / kTile) * kTile;
    const int qpos = obs_qpos(d.Hq / d.H);
    Carve c(base);
    FinchScratch s;
    s.kept = c.take<int32_t>((size_t)d.R * d.S);
    s.partial = c.take<float2>(heads * ((size_t)qpos * kFinchParts + window));
    s.cb = c.take<float>(heads * window);
    s.colsum = c.take<float>((size_t)d.R * S_pad);
    if (bytes) *bytes = c.bytes;
    return s;
}

size_t finch_scratch_bytes(const Dims& d, int window) {
    size_t bytes;
    carve_finch(d, window, nullptr, &bytes);
    return bytes;
}

int32_t* finch_scratch_kept(const Dims& d, const Workspace& ws) { return carve_finch(d, 1, ws.scorer).kept; }

// ---- pass 1: per-window-row softmax partials ---------------------------------------------------------------------
// Item u: block qb = n_blocks - 1 - u / (R P) (later blocks see more keys: work never increases with u), then part
// and row. Resident row r = g qpos + i is window row p0 + i of head j G + g (rows of padding heads, g >= G, and rows
// past w are computed and ignored). Consumer warpgroup cw computes D[qrow, key] for the 64-row blocks mb = cw, cw + 2,
// ... against the part's K tiles; the four threads that share a row merge their online (max, sum) at the end.
template <typename T, int D, int NQP>
__global__ void __launch_bounds__(umma::kTmaCtaThreads, 1)
finch_stats_kernel(const __grid_constant__ CUtensorMap mapK, const __grid_constant__ CUtensorMap mapQ, int H, int G,
                   int S, int window, int qpos, int R, int n_blocks, int n_parts, float c, float2* __restrict__ partial) {
    using L = SnSmem<D, NQP>;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* smem = umma::smem_align_1024(smem_raw);
    unsigned char* s_q = smem + L::kQOff;
    unsigned char* s_stage = smem + L::kStageOff;
    auto* k_ring = reinterpret_cast<umma::TmaRing<L::kStages>*>(smem + L::kBarOff);
    uint64_t* q_full = reinterpret_cast<uint64_t*>(k_ring + 1);

    constexpr int kMyBlocks = NQP / 128;
    const int NQ = G * qpos;
    const int off = S - window;  // position of window row 0
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;

    if (tid == 0) {
        umma::prefetch_tmap(&mapK);
        umma::prefetch_tmap(&mapQ);
        k_ring->init(umma::kTmaConsumerWarps);
        umma::mbar_init(q_full, 1);
        umma::mbar_fence_init();
    }
    __syncthreads();

    const long long n_items = (long long)R * n_blocks * n_parts;
    uint32_t k_it = 0, q_it = 0;
    for (long long u = blockIdx.x; u < n_items; u += gridDim.x) {
        const int qb = n_blocks - 1 - (int)(u / ((long long)R * n_parts));
        const int rem = (int)(u % ((long long)R * n_parts));
        const int part = rem / R, row = rem % R;
        const int b = row / H, j = row % H;
        const int p0 = qb * qpos;
        const int n_tiles = obs_stats_tiles(S, window, p0, qpos);
        const int per_part = (n_tiles + n_parts - 1) / n_parts;
        const int t_begin = part * per_part, t_end = min(n_tiles, t_begin + per_part);
        const bool empty = t_begin >= t_end;  // CTA-uniform: no Q load, the partial is (-inf, 0)
        __syncthreads();  // previous item fully consumed: s_q reusable

        if (wg == 0) {
            if (tid == 0 && !empty) {
                // rows past the window read as zero; rows of padding heads are not loaded
                umma::mbar_arrive_expect_tx(q_full, (uint32_t)(G * L::kPanels * qpos * 128));
                for (int g = 0; g < G; ++g)
                    for (int kp = 0; kp < L::kPanels; ++kp)
                        umma::tma_load_3d(s_q + kp * L::kQPanel + g * qpos * 128, &mapQ, q_full, kp * 64, p0,
                                          (b * H + j) * G + g);
                for (int t = t_begin; t < t_end; ++t, ++k_it) {
                    const int stage = k_ring->acquire(k_it, L::kStageBytes);
                    for (int kp = 0; kp < L::kPanels; ++kp)
                        umma::tma_load_4d(s_stage + stage * L::kStageBytes + kp * (kSnTile * 128), &mapK,
                                          k_ring->full(stage), kp * 64, t * kSnTile, j, b);
                }
            }
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
            if (!empty) {
                umma::mbar_wait(q_full, q_it & 1);
                for (int t = t_begin; t < t_end; ++t, ++k_it) {
                    const int stage = k_ring->wait(k_it);
                    const uint32_t kb = umma::smem_u32(s_stage + stage * L::kStageBytes);
                    const int key0 = t * kSnTile + 2 * qd;
                    const bool interior = (t + 1) * kSnTile <= off + p0 + 1;  // every key visible to every row
#pragma unroll
                    for (int i = 0; i < kMyBlocks; ++i) {
                        const int mb = 2 * i + cw;
                        if (mb * 64 >= NQ) continue;  // warpgroup-uniform
                        float acc[64];
                        snap_mma<T, D>(acc, umma::smem_u32(s_q + mb * 64 * 128), L::kQPanel, kb, kSnTile * 128);
#pragma unroll
                        for (int hh = 0; hh < 2; ++hh) {
                            const int r = mb * 64 + w4 * 16 + (lane >> 2) + 8 * hh;  // resident row
                            const int limit = off + p0 + r % qpos;                  // last visible key position
                            online_row_update(acc, hh, c, interior, key0, limit, S, run_m[i][hh], run_z[i][hh]);
                        }
                    }
                    k_ring->release(stage);
                }
                ++q_it;
            }
#pragma unroll
            for (int i = 0; i < kMyBlocks; ++i) {
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    float m = run_m[i][hh], z = run_z[i][hh];
                    quad_merge(m, z, c);
                    const int r = (2 * i + cw) * 64 + w4 * 16 + (lane >> 2) + 8 * hh;
                    const int g = r / qpos, pos = p0 + r % qpos;
                    if (qd == 0 && g < G && pos < window)
                        partial[((size_t)((b * H + j) * G + g) * window + pos) * n_parts + part] =
                            make_float2(m * c, z);  // (max in log2 units, sum)
                }
            }
        }
    }
}

// ---- merge: the exact normaliser of each window row, with its weight log2 c_i folded in ------------------------------
__global__ void __launch_bounds__(256)
finch_cb_kernel(int S, int window, int n_parts, int normalize, long long n_rows, const float2* __restrict__ partial,
                float* __restrict__ cb) {
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n_rows) return;
    const int i = (int)(q % window);
    const float2* part_q = partial + q * n_parts;
    float m = -INFINITY, z = 0.f;
    for (int pp = 0; pp < n_parts; ++pp) {  // fixed order: part 0 first
        const float2 pz = part_q[pp];
        const float mn = fmaxf(m, pz.x);
        z = (mn == -INFINITY) ? 0.f : z * fast_exp2(m - mn) + pz.y * fast_exp2(pz.x - mn);
        m = mn;
    }
    // c_i = S - w + i is an integer below 2^24: exact in fp32
    const float log2_ci = normalize ? log2f((float)(S - window + i)) : 0.f;
    cb[q] = -m - log2f(z) + log2_ci;
}

// ---- finalize: / (G w), ONE rounding, keys + histogram -----------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kTileThreads)
finch_finalize_kernel(int S, int window, float gw, const float* __restrict__ colsum, Workspace ws,
                      uint16_t* __restrict__ scores_out) {
    __shared__ uint16_t skeys[kTile];
    __shared__ uint16_t sscores[kTile];
    __shared__ uint32_t shist[256];
    const int tile = blockIdx.x, row = blockIdx.y, tid = threadIdx.x;
    shist[tid] = 0;
    pdl_launch_dependents();  // the select+compact kernel behind this one may start to take residency
    float fmax_valid = -INFINITY;
    score_tile_epilogue<T, 1, false>(skeys, sscores, shist, row, tile * kTile, S, S - window, S, ws, scores_out,
                                     &fmax_valid,
                                     [&](int, int s) { return colsum[(size_t)row * ws.S_pad + s] / gw; });
    publish_max_valid(fmax_valid, ws);
    flush_row_hist(shist, row, ws);
}

// ---- host launcher -------------------------------------------------------------------------------------------------
template <typename T, int D, int NQP>
static cudaError_t launch_finch_t(const Dims& d, int dtype, const void* K, const void* q, int window, int normalize,
                                  const Workspace& ws, void* scores_out, cudaStream_t st) {
    using L = SnSmem<D, NQP>;
    const int G = d.Hq / d.H, qpos = obs_qpos(G);
    const FinchScratch sc = carve_finch(d, window, ws.scorer);
    const int n_blocks = (window + qpos - 1) / qpos;
    const int n_parts = finch_parts(d.S, window, qpos);
    const long long n_items = (long long)d.R * n_blocks * n_parts;
    const int grid1 = (int)std::min<long long>(device_sm_count(), n_items);
    const float c = kLog2e * rsqrtf((float)D);  // 1 / sqrt(head_dim), logits -> log2 domain

    CUtensorMap mapK, mapQ;
    cudaError_t e;
    if ((e = make_tmap_cache(&mapK, K, d, d.ks, kSnTile)) != cudaSuccess) return e;
    // q_window [B Hq, w, D] contiguous: rows past w of a head read as zero
    const uint64_t n_heads = (uint64_t)d.B * d.Hq, head_stride = (uint64_t)window * D;
    if ((e = make_tmap_rows(&mapQ, q, D, window, D, n_heads, head_stride, qpos)) != cudaSuccess) return e;
    constexpr int smem = umma::smem_request(L::kTotal);
    constexpr auto k1 = finch_stats_kernel<T, D, NQP>;
    if ((e = ensure_dynamic_smem<k1>(smem)) != cudaSuccess) return e;

    k1<<<grid1, umma::kTmaCtaThreads, smem, st>>>(mapK, mapQ, d.H, G, d.S, window, qpos, d.R, n_blocks, n_parts, c,
                                                  sc.partial);
    if ((e = cudaPeekAtLastError()) != cudaSuccess) return e;
    const long long n_rows = (long long)n_heads * window;
    finch_cb_kernel<<<(unsigned)((n_rows + 255) / 256), 256, 0, st>>>(d.S, window, n_parts, normalize, n_rows,
                                                                       sc.partial, sc.cb);
    if ((e = cudaPeekAtLastError()) != cudaSuccess) return e;
    const int n_ctx_tiles = (d.S - window + kSnTile - 1) / kSnTile;  // key tiles holding a context position
    if ((e = launch_attention_colsum(d, dtype, K, q, window, n_ctx_tiles, c, sc.cb, sc.colsum, ws.S_pad, st)) !=
        cudaSuccess)
        return e;
    finch_finalize_kernel<T><<<dim3(ws.n_tiles, d.R), kTileThreads, 0, st>>>(
        d.S, window, (float)(G * window), sc.colsum, ws, static_cast<uint16_t*>(scores_out));
    if ((e = cudaPeekAtLastError()) != cudaSuccess) return e;
    if (scores_out != nullptr) e = launch_fill_sentinel(dtype, scores_out, d.R, d.S, d.S - window, d.S, ws, st);
    return e;
}

template <typename T>
static cudaError_t launch_finch_d(const Dims& d, int dtype, const void* K, const void* q, int window, int normalize,
                                  const Workspace& ws, void* scores_out, cudaStream_t st) {
    const int G = d.Hq / d.H;
    // 1 <= G <= 8: the G heads' query blocks (G qpos rows) are padded to 128 / 256 / 512 resident rows
    if (G < 1 || G > 8) return cudaErrorNotSupported;
    const int NQ = G * obs_qpos(G);
    const int NQP = NQ <= 128 ? 128 : (NQ <= 256 ? 256 : 512);
#define KVP_FINCH(DD, NN) \
    if (d.D == DD && NQP == NN) return launch_finch_t<T, DD, NN>(d, dtype, K, q, window, normalize, ws, scores_out, st)
    KVP_FINCH(128, 128);
    KVP_FINCH(128, 256);
    KVP_FINCH(128, 512);
    KVP_FINCH(64, 128);
    KVP_FINCH(64, 256);
    KVP_FINCH(64, 512);
#undef KVP_FINCH
    return cudaErrorNotSupported;
}

cudaError_t launch_finch_score(const Dims& d, int dtype, const void* K, const void* q_window, int window,
                               int normalize, const Workspace& ws, void* scores_out, cudaStream_t st) {
    return with_dtype(dtype, [&](auto t) {
        return launch_finch_d<decltype(t)>(d, dtype, K, q_window, window, normalize, ws, scores_out, st);
    });
}

}  // namespace kvp
