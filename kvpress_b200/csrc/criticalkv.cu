// criticalkv.cu — stage S for CriticalKVPress (sm_90a: TMA + wgmma).
//
// Reference semantics (kvpress/presses/criticalkv_press.py:57-92), per (b, kv head j, position s), with G = Hq / Hkv
// and the query heads h = j G + g of kv head j (repeat_kv order):
//     norm(s)  = (1/G) sum_g sum_{n < hidden} | sum_d V[b,j,s,d] Wo[n, h D + d] |        (vwl1norm, :57-76)
//     score(s) = (base(s) + epsilon) * norm(s)                                             (:87)
//   and the n_first positions with the largest base score get finfo(dtype).max            (:82-90).
// The reference materialises V_h @ Wo_h^T, a [B, S, hidden] tensor per query head, only to take its row L1 norms.
// Here one persistent kernel (criticalkv_kernel, one CTA per SM, warp-specialised) keeps every product tile in
// registers: TMA loads a kCkvRows-position V tile (SWIZZLE_128B, strided caches in place) into one of two V buffers
// and streams 128-row chunks of Wo through a ring, K-major as stored (the rows of o_proj.weight are contiguous along
// d: no transpose, no copy); each consumer warpgroup multiplies its 64-row slices of the V tile with the chunk
// (wgmma, both operands from shared memory) and adds the magnitudes of the [64 x 128] product to per-row fp32 sums
// right away. Nothing of size S x hidden touches memory.
// The score is formed in fp32 and rounded once to the cache dtype. Stage 1 (the forced n_first) reuses the selection
// kernels: keys of the base scores, a select-only pass into workspace scratch, then criticalkv_force_kernel.
#include "common.cuh"
#include "umma.cuh"

namespace kvp {

constexpr int kCkvN = 128;        // Wo rows (output features) per chunk: the wgmma N
constexpr int kCkvMt = 2;         // 64-row m-tiles per consumer warpgroup (DESIGN.md §3, CriticalKV)
constexpr int kCkvRows = 2 * 64 * kCkvMt;  // positions per item

struct CkvScratch {
    int32_t* first;    // [R][n_first] positions forced by stage 1
    uint16_t* scores;  // [R][S] final scores of a compress call that returns none
};

// The scratch in ws.scorer; with a null base only its size (*bytes).
static CkvScratch carve_ckv(const Dims& d, void* base, size_t* bytes = nullptr) {
    Carve c(base);
    CkvScratch s;
    s.first = c.take<int32_t>((size_t)d.R * d.S);
    s.scores = c.take<uint16_t>((size_t)d.R * d.S);
    if (bytes) *bytes = c.bytes;
    return s;
}

size_t criticalkv_scratch_bytes(const Dims& d) {
    size_t bytes;
    carve_ckv(d, nullptr, &bytes);
    return bytes;
}

void* criticalkv_scratch_scores(const Dims& d, const Workspace& ws) { return carve_ckv(d, ws.scorer).scores; }

template <int D>
struct CkvSmem {
    static constexpr int kPanels = D / 64;                    // 64-element (128 B) panels along d
    static constexpr int kVBytes = kPanels * kCkvRows * 128;  // one V tile
    static constexpr int kWBytes = kPanels * kCkvN * 128;     // one Wo chunk
    static constexpr int kStages = umma::ring_stages(2 * kVBytes + 256, kWBytes);  // Wo ring next to two V buffers
    static_assert(kStages >= 2, "Wo ring needs two stages");
    static constexpr int kVOff = 0;
    static constexpr int kWOff = 2 * kVBytes;
    static constexpr int kBarOff = kWOff + kStages * kWBytes;
    static constexpr int kTotal = kBarOff + 256;
    static_assert(umma::smem_request(kTotal) <= umma::kSmemBudget, "shared memory budget");
};

// CTA p of n_workers owns the items [ckv_start(p), ckv_start(p + 1)): equal contiguous ranges.
__host__ __device__ inline long long ckv_start(int p, long long total, int n_workers) {
    return ((long long)p * total) / n_workers;
}

// Work: item = (row = b Hkv + j, kCkvRows-position tile). Per item the producer loads the V tile once, then the
// G * n_chunks Wo chunks of the row's query heads in (g, chunk) order. Consumer warpgroup cw owns the rows
// [64 (cw kCkvMt + mt), +64) of the tile. Summation order: a thread holds rows r0 and r0 + 8 of each of its m-tiles
// and adds the magnitudes of its accumulator columns into two fp32 sums per row (column pairs 8i + 2qd and
// 8i + 2qd + 1), register by register, chunk after chunk; at the end of the item it adds its two sums and the four
// threads of a row add theirs (xor 1, then xor 2). The order depends only on the shape.
template <typename T, int D>
__global__ void __launch_bounds__(umma::kTmaCtaThreads, 1)
criticalkv_kernel(const __grid_constant__ CUtensorMap mapV, const __grid_constant__ CUtensorMap mapW,
                  const uint16_t* __restrict__ base, int64_t sb, int64_t sh, uint16_t* __restrict__ scores_out, int H,
                  int G, int S, int R, int n_tiles, int n_chunks, int n_workers, float eps) {
    using L = CkvSmem<D>;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* smem = umma::smem_align_1024(smem_raw);
    unsigned char* s_v = smem + L::kVOff;
    unsigned char* s_w = smem + L::kWOff;
    auto* w_ring = reinterpret_cast<umma::TmaRing<L::kStages>*>(smem + L::kBarOff);
    auto* v_ring = reinterpret_cast<umma::TmaRing<2>*>(w_ring + 1);  // the two V buffers

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
    if (tid == 0) {
        umma::prefetch_tmap(&mapV);
        umma::prefetch_tmap(&mapW);
        w_ring->init(umma::kTmaConsumerWarps);
        v_ring->init(umma::kTmaConsumerWarps);
        umma::mbar_fence_init();
    }
    __syncthreads();

    const long long total = (long long)R * n_tiles;
    const long long i_begin = ckv_start(blockIdx.x, total, n_workers);
    const long long i_end = ckv_start(blockIdx.x + 1, total, n_workers);
    const int n_gc = G * n_chunks;

    if (wg == 0) {
        if (tid == 0) {
            // ===== TMA producer =====
            uint32_t w_it = 0, v_it = 0;
            for (long long it = i_begin; it < i_end; ++it, ++v_it) {
                const int row = (int)(it / n_tiles), tile = (int)(it - (long long)row * n_tiles);
                const int b = row / H, j = row % H;
                const int vb = v_ring->acquire(v_it, L::kVBytes);
                for (int kp = 0; kp < L::kPanels; ++kp)
                    umma::tma_load_4d(s_v + vb * L::kVBytes + kp * (kCkvRows * 128), &mapV, v_ring->full(vb), kp * 64,
                                      tile * kCkvRows, j, b);
                for (int gc = 0; gc < n_gc; ++gc, ++w_it) {
                    const int g = gc / n_chunks, c = gc - g * n_chunks;
                    const int stage = w_ring->acquire(w_it, L::kWBytes);
                    for (int kp = 0; kp < L::kPanels; ++kp)
                        umma::tma_load_3d(s_w + stage * L::kWBytes + kp * (kCkvN * 128), &mapW, w_ring->full(stage),
                                          (j * G + g) * D + kp * 64, c * kCkvN, 0);
                }
            }
        }
    } else {
        // ===== consumers: wgmma + |.| sums; thread = rows r0, r0 + 8 of each m-tile =====
        const int cw = wg - 1, qd = lane & 3;
        const float inv_g = 1.0f / (float)G;
        uint32_t w_it = 0, v_it = 0;
        for (long long it = i_begin; it < i_end; ++it, ++v_it) {
            const int row = (int)(it / n_tiles), tile = (int)(it - (long long)row * n_tiles);
            const int vb = v_ring->wait(v_it);
            const uint32_t v_base = umma::smem_u32(s_v + vb * L::kVBytes);
            float sum[kCkvMt][4];
#pragma unroll
            for (int mt = 0; mt < kCkvMt; ++mt) sum[mt][0] = sum[mt][1] = sum[mt][2] = sum[mt][3] = 0.f;
            for (int gc = 0; gc < n_gc; ++gc, ++w_it) {
                const int stage = w_ring->wait(w_it);
                const uint32_t w_base = umma::smem_u32(s_w + stage * L::kWBytes);
#pragma unroll
                for (int mt = 0; mt < kCkvMt; ++mt) {
                    float acc[kCkvN / 2];
                    umma::wgmma_fence();
#pragma unroll
                    for (int kk = 0; kk < D / 16; ++kk) {
                        const int kp = kk >> 2, ks = kk & 3;
                        umma::wgmma_ss<kCkvN, F16Traits<T>::kMmaFormat>(
                            acc,
                            umma::smem_desc_sw128(v_base + kp * (kCkvRows * 128) + (cw * kCkvMt + mt) * (64 * 128) +
                                                  ks * 32),
                            umma::smem_desc_sw128(w_base + kp * (kCkvN * 128) + ks * 32), kk > 0);
                    }
                    umma::wgmma_commit();
                    umma::wgmma_wait_all();
                    // register i: row r0 + 8 ((i / 2) & 1), column 8 (i / 4) + 2 qd + (i & 1)
#pragma unroll
                    for (int i = 0; i < kCkvN / 2; ++i) sum[mt][i & 3] += fabsf(acc[i]);
                }
                w_ring->release(stage);  // the chunk's MMAs have completed
            }
            v_ring->release(vb);
            const int b = row / H, j = row % H;
#pragma unroll
            for (int mt = 0; mt < kCkvMt; ++mt) {
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    float l1 = sum[mt][2 * hh] + sum[mt][2 * hh + 1];
                    l1 += __shfl_xor_sync(0xFFFFFFFFu, l1, 1);
                    l1 += __shfl_xor_sync(0xFFFFFFFFu, l1, 2);
                    const int s = tile * kCkvRows + (cw * kCkvMt + mt) * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * hh;
                    if (qd == 0 && s < S) {
                        const float bs = F16Traits<T>::to_float(base[(int64_t)b * sb + (int64_t)j * sh + s]);
                        scores_out[(size_t)row * S + s] = F16Traits<T>::from_float((bs + eps) * (l1 * inv_g));
                    }
                }
            }
        }
    }
}

// Stage 1: scores[row][first[row][i]] = finfo(dtype).max for i < n_first.
__global__ void criticalkv_force_kernel(uint16_t* __restrict__ scores, int S, const int32_t* __restrict__ first,
                                        int n_first, int R, uint16_t max_bits) {
    const long long n = (long long)R * n_first;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        scores[(i / n_first) * S + first[i]] = max_bits;
}

// ---- host launcher -----------------------------------------------------------------------------------
template <typename T, int D>
static cudaError_t launch_criticalkv_t(const Dims& d, const void* V, const void* base, int64_t sb, int64_t sh,
                                       const void* wo, int hidden, int64_t wo_stride, float eps, void* scores_out,
                                       cudaStream_t st) {
    using L = CkvSmem<D>;
    const int n_tiles = (d.S + kCkvRows - 1) / kCkvRows;
    const int n_chunks = (hidden + kCkvN - 1) / kCkvN;
    const long long total = (long long)d.R * n_tiles;
    int n_workers = device_sm_count();
    if ((long long)n_workers > total) n_workers = (int)total;  // every CTA owns at least one item

    constexpr int smem = umma::smem_request(L::kTotal);
    constexpr auto kern = criticalkv_kernel<T, D>;
    cudaError_t e = ensure_dynamic_smem<kern>(smem);
    if (e != cudaSuccess) return e;
    CUtensorMap mapV, mapW;
    if ((e = make_tmap_cache(&mapV, V, d, d.vs, kCkvRows)) != cudaSuccess) return e;
    // Wo [hidden, wo_stride] as stored; rows past `hidden` read as zero and add nothing
    if ((e = make_tmap_rows(&mapW, wo, (uint64_t)d.Hq * D, hidden, wo_stride, 1, (uint64_t)wo_stride * hidden,
                            kCkvN)) != cudaSuccess)
        return e;
    kern<<<n_workers, umma::kTmaCtaThreads, smem, st>>>(mapV, mapW, static_cast<const uint16_t*>(base), sb, sh,
                                                        static_cast<uint16_t*>(scores_out), d.H, d.Hq / d.H, d.S, d.R,
                                                        n_tiles, n_chunks, n_workers, eps);
    return cudaPeekAtLastError();
}

cudaError_t launch_criticalkv_score(const Dims& d, int dtype, const void* V, const void* base, int64_t sb,
                                    int64_t sh, const void* wo, int hidden, int64_t wo_stride, float eps, int n_first,
                                    const Workspace& ws, void* scores_out, cudaStream_t st) {
    if (d.D != 64 && d.D != 128) return cudaErrorNotSupported;
    const CkvScratch sc = carve_ckv(d, ws.scorer);
    cudaError_t e;
    if (n_first > 0) {
        // the n_first best base scores of every row (ties to the lowest positions) into sc.first; ws is zeroed
        if ((e = launch_keys_from_scores(d, dtype, base, sb, sh, ws, st)) != cudaSuccess) return e;
        Dims ds = d;
        ds.n_kept = n_first;
        ds.ks = ds.vs = {0, 0, 0};
        if ((e = launch_select_compact(ds, nullptr, nullptr, nullptr, nullptr, sc.first, ws, st)) != cudaSuccess)
            return e;
    }
    e = with_dtype(dtype, [&](auto t) {
        using T = decltype(t);
        if (d.D == 128) return launch_criticalkv_t<T, 128>(d, V, base, sb, sh, wo, hidden, wo_stride, eps, scores_out, st);
        return launch_criticalkv_t<T, 64>(d, V, base, sb, sh, wo, hidden, wo_stride, eps, scores_out, st);
    });
    if (e != cudaSuccess || n_first == 0) return e;
    const long long n = (long long)d.R * n_first;
    const int blocks = (int)(n < 256 * 1024 ? (n + 255) / 256 : 1024);
    criticalkv_force_kernel<<<blocks, 256, 0, st>>>(static_cast<uint16_t*>(scores_out), d.S, sc.first, n_first, d.R,
                                                    dtype == KVP_BF16 ? (uint16_t)0x7F7Fu : (uint16_t)0x7BFFu);
    return cudaPeekAtLastError();
}

}  // namespace kvp
