// kvzap.cu — KVzapPress's surrogate scores and DMSPress's threshold eviction (sm_90a).
//
// Reference semantics (kvpress/presses/kvzap_press.py:56-80): per layer, a surrogate model applied to the attention
// module's input hidden states x [B, S, hidden] gives one score per (b, kv head j, s):
//     MLP    score = b2[j] + sum_c W2[j, c] gelu(b1[c] + sum_k W1[c, k] x[b, s, k])   (W1 [hd, hidden], W2 [Hkv, hd])
//     linear score = b[j] + sum_k W[j, k] x[b, s, k]                                     (W [Hkv, hidden])
// with nn.GELU's exact erf form. The reference evaluates Linear -> GELU -> Linear in the cache dtype, writing and
// re-reading a [B, S, hd] intermediate, then transposes. Here:
//   * kvzap_mlp_kernel (B S > kZapGemvRows): one persistent, warp-specialised CTA per SM. TMA streams 64-column panels
//     of a 128-position x tile (strided views in place) and of a 128-row chunk of W1, K-major as stored, through one
//     ring; each consumer warpgroup multiplies its 64 rows with the chunk (wgmma), applies bias + GELU to the fp32
//     accumulators and folds them into one fp32 partial sum per (row, kv head) with W2 and b1 held in shared memory.
//     Items are (tile, chunk) with the chunk inner and dealt round-robin, so the chunks of one tile run side by side and
//     the tile is read from HBM about once. Nothing of size S x hd touches memory: the partials are
//     [ceil(hd / 128)][Hkv][B S] fp32.
//   * kvzap_gemv_kernel (B S <= kZapGemvRows, decoding): W1 is spread over ceil(hd / 8) CTAs, one hidden unit per
//     warp, so one call reads W1 once across the SMs; partials [ceil(hd / 8)][Hkv][B S].
//   * kvzap_reduce_kernel adds each row's partials in part order, then b2, and rounds once into [B, Hkv, S].
//   * kvzap_linear_kernel (hd == 0): CUDA cores, four rows per warp, 16-byte loads; the model is bound by reading x.
// Every sum is fp32 in an order fixed by the shape; the score is rounded once to the cache dtype.
//
// kvp_threshold_evict (DMSPress, kvpress/presses/dms_press.py:92-107): every (b, h, s < n_evict) whose score is below
// the threshold rounded to the score dtype, in torch.where order, by per-(row, 4096-position tile) counts, one scan
// and an ordered write.
#include "common.cuh"
#include "umma.cuh"

namespace kvp {

constexpr int kZapRows = 128;                       // positions per tile: two consumer warpgroups x 64
constexpr int kZapN = 128;                          // hidden units (W1 rows) per chunk: the wgmma N
constexpr int kZapStageBytes = 2 * kZapRows * 128;  // one 64-column panel of the x tile and one of the W1 chunk
constexpr int kZapLinRows = 4;                      // rows per warp of the linear kernel

template <int kStages>
struct ZapSmem {
    static constexpr int kBarOff = kStages * kZapStageBytes;
    static constexpr int kParamOff = kBarOff + 256;  // b1 [hd], then W2 [Hkv][hd], 16-bit
    static constexpr int kParamMax = umma::kSmemBudget - umma::kSmemAlignSlack - kParamOff;
};
static_assert(ZapSmem<2>::kParamMax >= 2 * kZapMaxHd * (kZapMaxHeads + 1), "b1 + W2 of the largest model fit");

size_t kvzap_scratch_bytes(const Dims& d) {
    const size_t rows = (size_t)d.B * d.S;
    const size_t parts = rows <= (size_t)kZapGemvRows ? (kZapMaxHd + kZapGemvUnits - 1) / kZapGemvUnits
                                                      : (kZapMaxHd + kZapN - 1) / kZapN;
    return align256(parts * d.H * rows * sizeof(float)) + align256((size_t)d.R * d.S * sizeof(uint16_t));
}

void* kvzap_scratch_scores(const Dims& d, const Workspace& ws) {
    return static_cast<char*>(ws.scorer) + (kvzap_scratch_bytes(d) - align256((size_t)d.R * d.S * sizeof(uint16_t)));
}

__device__ __forceinline__ float gelu_erf(float v) { return 0.5f * v * (1.f + erff(v * 0.70710678118654752f)); }

__device__ __forceinline__ void wgmma_wait_1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
    return v;
}

// acc + sum_e w[e] x[e] over the 8 elements of two 16-byte vectors, in element order
template <typename T>
__device__ __forceinline__ float dot8(uint4 w, uint4 x, float acc) {
    const uint32_t wv[4] = {w.x, w.y, w.z, w.w}, xv[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 a = F16Traits<T>::unpack2(wv[i]), b = F16Traits<T>::unpack2(xv[i]);
        acc = fmaf(a.x, b.x, acc);
        acc = fmaf(a.y, b.y, acc);
    }
    return acc;
}

// Work: item = (b, 128-position tile, 128-unit chunk), chunk fastest; CTA p takes items p, p + gridDim.x, ...
// Summation order: the pre-activation of (row, unit) is the wgmma's K-ordered fp32 accumulation over hidden; a thread
// holds rows r0 and r0 + 8 and 32 units of each; per kv head it adds W2[j, c] h[c] over its units in register order,
// then the four threads of a row add theirs (xor 1, then xor 2), and lane qd == 0 writes the chunk's partial.
template <typename T, int kStages>
__global__ void __launch_bounds__(umma::kTmaCtaThreads, 1)
kvzap_mlp_kernel(const __grid_constant__ CUtensorMap mapX, const __grid_constant__ CUtensorMap mapW,
                 const uint16_t* __restrict__ b1, const uint16_t* __restrict__ w2, float* __restrict__ partial, int S,
                 int H, int hd, int n_tiles, int n_chunks, int n_kp, long long total, long long rows_total) {
    using L = ZapSmem<kStages>;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* smem = umma::smem_align_1024(smem_raw);
    auto* ring = reinterpret_cast<umma::TmaRing<kStages>*>(smem + L::kBarOff);
    uint16_t* s_b1 = reinterpret_cast<uint16_t*>(smem + L::kParamOff);
    uint16_t* s_w2 = s_b1 + hd;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
    if (tid == 0) {
        umma::prefetch_tmap(&mapX);
        umma::prefetch_tmap(&mapW);
        ring->init(umma::kTmaConsumerWarps);
        umma::mbar_fence_init();
    }
    for (int i = tid; i < hd; i += blockDim.x) s_b1[i] = b1[i];
    for (int i = tid; i < H * hd; i += blockDim.x) s_w2[i] = w2[i];
    __syncthreads();

    if (wg == 0) {
        if (tid == 0) {
            // ===== TMA producer =====
            uint32_t it_s = 0;
            for (long long it = blockIdx.x; it < total; it += gridDim.x) {
                const long long tf = it / n_chunks;
                const int chunk = (int)(it - tf * n_chunks);
                const int b = (int)(tf / n_tiles), tile = (int)(tf - (long long)b * n_tiles);
                for (int kp = 0; kp < n_kp; ++kp, ++it_s) {
                    const int st = ring->acquire(it_s, kZapStageBytes);
                    unsigned char* dst = smem + st * kZapStageBytes;
                    umma::tma_load_3d(dst, &mapX, ring->full(st), kp * 64, tile * kZapRows, b);
                    umma::tma_load_3d(dst + kZapRows * 128, &mapW, ring->full(st), kp * 64, chunk * kZapN, 0);
                }
            }
        }
    } else {
        // ===== consumers: wgmma, bias + GELU, fold with W2 =====
        const int cw = wg - 1, qd = lane & 3;
        uint32_t it_s = 0;
        for (long long it = blockIdx.x; it < total; it += gridDim.x) {
            const long long tf = it / n_chunks;
            const int chunk = (int)(it - tf * n_chunks);
            const int b = (int)(tf / n_tiles), tile = (int)(tf - (long long)b * n_tiles);
            float acc[kZapN / 2];
            int prev = -1;
            for (int kp = 0; kp < n_kp; ++kp, ++it_s) {
                const int st = ring->wait(it_s);
                const uint32_t base = umma::smem_u32(smem + st * kZapStageBytes);
                umma::wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < 4; ++ks)
                    umma::wgmma_ss<kZapN, F16Traits<T>::kMmaFormat>(
                        acc, umma::smem_desc_sw128(base + cw * (64 * 128) + ks * 32),
                        umma::smem_desc_sw128(base + kZapRows * 128 + ks * 32), (kp > 0 || ks > 0) ? 1u : 0u);
                umma::wgmma_commit();
                wgmma_wait_1();  // the previous panel's MMAs have completed: hand its stage back
                if (prev >= 0) ring->release(prev);
                prev = st;
            }
            umma::wgmma_wait_all();
            ring->release(prev);

            // register i: row r0 + 8 ((i / 2) & 1), unit 8 (i / 4) + 2 qd + (i & 1) of the chunk
            const int c0 = chunk * kZapN;
#pragma unroll
            for (int i = 0; i < kZapN / 2; ++i) {
                const int c = c0 + 8 * (i >> 2) + 2 * qd + (i & 1);
                acc[i] = c < hd ? gelu_erf(acc[i] + F16Traits<T>::to_float(s_b1[c])) : 0.f;
            }
            const int r0 = tile * kZapRows + cw * 64 + (warp & 3) * 16 + (lane >> 2);
            const long long row0 = (long long)b * S + r0;
            for (int j = 0; j < H; ++j) {
                const uint16_t* w2j = s_w2 + (size_t)j * hd;
                float p0 = 0.f, p1 = 0.f;
#pragma unroll
                for (int i = 0; i < kZapN / 2; ++i) {
                    const int c = c0 + 8 * (i >> 2) + 2 * qd + (i & 1);
                    const float w = c < hd ? F16Traits<T>::to_float(w2j[c]) : 0.f;
                    if ((i >> 1) & 1)
                        p1 = fmaf(w, acc[i], p1);
                    else
                        p0 = fmaf(w, acc[i], p0);
                }
                p0 += __shfl_xor_sync(0xFFFFFFFFu, p0, 1);
                p0 += __shfl_xor_sync(0xFFFFFFFFu, p0, 2);
                p1 += __shfl_xor_sync(0xFFFFFFFFu, p1, 1);
                p1 += __shfl_xor_sync(0xFFFFFFFFu, p1, 2);
                float* out = partial + ((long long)chunk * H + j) * rows_total + row0;
                if (qd == 0 && r0 < S) out[0] = p0;
                if (qd == 0 && r0 + 8 < S) out[8] = p1;
            }
        }
    }
}

// One hidden unit c per warp, every row r < rows (rows = B S <= kZapGemvRows): the lanes take 8-element slices of
// hidden (lane 8 l + 256 i) and add them in i order, then xor 16 ... 1; h = gelu(pre + b1[c]). Each CTA then writes
// partial[blockIdx][j][r] = sum of W2[j, c] h[c] over its units in ascending c.
template <typename T>
__global__ void __launch_bounds__(256) kvzap_gemv_kernel(const uint16_t* __restrict__ x, int64_t xb, int64_t xs, int S,
                                                         int rows, int hidden, int hd, const uint16_t* __restrict__ w1,
                                                         const uint16_t* __restrict__ b1,
                                                         const uint16_t* __restrict__ w2, int H,
                                                         float* __restrict__ partial) {
    __shared__ float s_h[kZapGemvUnits][kZapGemvRows];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int c = blockIdx.x * kZapGemvUnits + warp;
    if (c < hd) {
        const uint16_t* wr = w1 + (size_t)c * hidden;
        const float bias = F16Traits<T>::to_float(b1[c]);
        for (int r = 0; r < rows; ++r) {
            const uint16_t* xr = x + (int64_t)(r / S) * xb + (int64_t)(r % S) * xs;
            float acc = 0.f;
            for (int k = lane * 8; k < hidden; k += 256)
                acc = dot8<T>(*reinterpret_cast<const uint4*>(wr + k), *reinterpret_cast<const uint4*>(xr + k), acc);
            acc = warp_sum(acc);
            if (lane == 0) s_h[warp][r] = gelu_erf(acc + bias);
        }
    }
    __syncthreads();
    for (int t = threadIdx.x; t < H * rows; t += blockDim.x) {
        const int j = t / rows, r = t - j * rows;
        float p = 0.f;
        for (int w = 0; w < kZapGemvUnits; ++w) {
            const int cc = blockIdx.x * kZapGemvUnits + w;
            if (cc < hd) p = fmaf(F16Traits<T>::to_float(w2[(size_t)j * hd + cc]), s_h[w][r], p);
        }
        partial[((long long)blockIdx.x * H + j) * rows + r] = p;
    }
}

// scores[b, j, s] = round(sum of the row's partials in part order + b2[j])
template <typename T>
__global__ void kvzap_reduce_kernel(const float* __restrict__ partial, int n_parts, const uint16_t* __restrict__ b2,
                                    uint16_t* __restrict__ out, int S, int H, long long rows_total) {
    const long long n = rows_total * H;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long bj = i / S;
        const int s = (int)(i - bj * S), b = (int)(bj / H), j = (int)(bj - (long long)b * H);
        const long long r = (long long)b * S + s;
        float v = 0.f;
        for (int c = 0; c < n_parts; ++c) v += partial[((long long)c * H + j) * rows_total + r];
        out[i] = F16Traits<T>::from_float(v + F16Traits<T>::to_float(b2[j]));
    }
}

// Linear model: kZapLinRows rows per warp, kv heads in blocks of 8; per (row, head) the lanes add their 8-element
// slices (lane 8 l + 256 i) in i order, then xor 16 ... 1, then the bias; rounded once.
template <typename T>
__global__ void __launch_bounds__(256) kvzap_linear_kernel(const uint16_t* __restrict__ x, int64_t xb, int64_t xs, int S,
                                                           long long rows, int hidden, const uint16_t* __restrict__ w,
                                                           const uint16_t* __restrict__ bias, int H,
                                                           uint16_t* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const long long r0 = (blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5)) * kZapLinRows;
    if (r0 >= rows) return;
    const uint16_t* xr[kZapLinRows];
#pragma unroll
    for (int q = 0; q < kZapLinRows; ++q) {
        const long long r = r0 + q < rows ? r0 + q : r0;
        xr[q] = x + (r / S) * xb + (r % S) * xs;
    }
    for (int jb = 0; jb < H; jb += 8) {
        float acc[kZapLinRows][8];
#pragma unroll
        for (int q = 0; q < kZapLinRows; ++q)
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) acc[q][jj] = 0.f;
#pragma unroll 4
        for (int k = lane * 8; k < hidden; k += 256) {
            uint4 xv[kZapLinRows];
#pragma unroll
            for (int q = 0; q < kZapLinRows; ++q) xv[q] = *reinterpret_cast<const uint4*>(xr[q] + k);
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                if (jb + jj < H) {
                    const uint4 wv = *reinterpret_cast<const uint4*>(w + (size_t)(jb + jj) * hidden + k);
#pragma unroll
                    for (int q = 0; q < kZapLinRows; ++q) acc[q][jj] = dot8<T>(wv, xv[q], acc[q][jj]);
                }
            }
        }
#pragma unroll
        for (int q = 0; q < kZapLinRows; ++q) {
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                const float v = warp_sum(acc[q][jj]);
                const long long r = r0 + q;
                const int j = jb + jj;
                if (lane == 0 && r < rows && j < H) {
                    const long long b = r / S, s = r - b * S;
                    out[(b * H + j) * S + s] = F16Traits<T>::from_float(v + F16Traits<T>::to_float(bias[j]));
                }
            }
        }
    }
}

// ---- host launchers -------------------------------------------------------------------------------------------------
template <typename T, int kStages>
static cudaError_t launch_kvzap_mlp_t(const Dims& d, const void* x, int64_t xb, int64_t xs, int hidden, int hd,
                                      const void* w1, const void* b1, const void* w2, float* partial, int param_bytes,
                                      cudaStream_t st) {
    using L = ZapSmem<kStages>;
    const int n_tiles = (d.S + kZapRows - 1) / kZapRows;
    const int n_chunks = (hd + kZapN - 1) / kZapN;
    const int n_kp = (hidden + 63) / 64;
    const long long total = (long long)d.B * n_tiles * n_chunks;
    int n_workers = device_sm_count();
    if ((long long)n_workers > total) n_workers = (int)total;
    constexpr auto kern = kvzap_mlp_kernel<T, kStages>;
    cudaError_t e = ensure_dynamic_smem<kern>(umma::kSmemBudget);
    if (e != cudaSuccess) return e;
    const int smem = umma::smem_request(L::kParamOff + param_bytes);
    CUtensorMap mapX, mapW;
    // x [B][S][hidden] with element strides (xb, xs); a stride of a size-1 dim is replaced by a dense one
    const uint64_t row_stride = d.S > 1 ? (uint64_t)xs : (uint64_t)(hidden + 7) / 8 * 8;
    const uint64_t batch_stride = d.B > 1 ? (uint64_t)xb : row_stride * d.S;
    if ((e = make_tmap_rows(&mapX, x, hidden, d.S, row_stride, d.B, batch_stride, kZapRows)) != cudaSuccess) return e;
    // W1 [hd][hidden] as stored; units past hd read as zero and are dropped in the epilogue
    if ((e = make_tmap_rows(&mapW, w1, hidden, hd, hidden, 1, (uint64_t)hidden * hd, kZapN)) != cudaSuccess) return e;
    kern<<<n_workers, umma::kTmaCtaThreads, smem, st>>>(mapX, mapW, static_cast<const uint16_t*>(b1),
                                                        static_cast<const uint16_t*>(w2), partial, d.S, d.H, hd,
                                                        n_tiles, n_chunks, n_kp, total, (long long)d.B * d.S);
    return cudaPeekAtLastError();
}

cudaError_t launch_kvzap_score(const Dims& d, int dtype, const void* x, int64_t xb, int64_t xs, int hidden, int hd,
                               const void* w1, const void* b1, const void* w2, const void* b2, const Workspace& ws,
                               void* scores_out, cudaStream_t st) {
    const long long rows = (long long)d.B * d.S;
    return with_dtype(dtype, [&](auto t) -> cudaError_t {
        using T = decltype(t);
        const auto* xp = static_cast<const uint16_t*>(x);
        auto* out = static_cast<uint16_t*>(scores_out);
        if (hd == 0) {
            const long long warps = (rows + kZapLinRows - 1) / kZapLinRows;
            kvzap_linear_kernel<T><<<(unsigned)((warps + 7) / 8), 256, 0, st>>>(
                xp, xb, xs, d.S, rows, hidden, static_cast<const uint16_t*>(w1), static_cast<const uint16_t*>(b1), d.H,
                out);
            return cudaPeekAtLastError();
        }
        float* partial = static_cast<float*>(ws.scorer);
        int n_parts;
        cudaError_t e;
        if (rows <= kZapGemvRows) {
            n_parts = (hd + kZapGemvUnits - 1) / kZapGemvUnits;
            kvzap_gemv_kernel<T><<<n_parts, 32 * kZapGemvUnits, 0, st>>>(
                xp, xb, xs, d.S, (int)rows, hidden, hd, static_cast<const uint16_t*>(w1),
                static_cast<const uint16_t*>(b1), static_cast<const uint16_t*>(w2), d.H, partial);
            e = cudaPeekAtLastError();
        } else {
            n_parts = (hd + kZapN - 1) / kZapN;
            const int param_bytes = 2 * hd * (d.H + 1);
            e = param_bytes <= ZapSmem<4>::kParamMax
                    ? launch_kvzap_mlp_t<T, 4>(d, x, xb, xs, hidden, hd, w1, b1, w2, partial, param_bytes, st)
                    : launch_kvzap_mlp_t<T, 2>(d, x, xb, xs, hidden, hd, w1, b1, w2, partial, param_bytes, st);
        }
        if (e != cudaSuccess) return e;
        const long long n = rows * d.H;
        const int blocks = (int)(n < 256LL * 4096 ? (n + 255) / 256 : 4096);
        kvzap_reduce_kernel<T><<<blocks, 256, 0, st>>>(partial, n_parts, static_cast<const uint16_t*>(b2), out, d.S,
                                                       d.H, rows);
        return cudaPeekAtLastError();
    });
}

// ---- DMS threshold eviction -----------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ bool evicted(uint16_t bits, float thr) {
    return F16Traits<T>::to_float(bits) < thr;  // NaN compares false
}

__device__ __forceinline__ long long block_sum_256(long long v, long long* s_part) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = v;
    __syncthreads();
    long long t = 0;
    for (int w = 0; w < 8; ++w) t += s_part[w];
    __syncthreads();
    return t;
}

// Per (row, tile of kEvictTile positions): the evicted count, into counts[row * n_tiles + tile].
template <typename T>
__global__ void __launch_bounds__(256) evict_count_kernel(const uint16_t* __restrict__ scores, int64_t sb, int64_t sh,
                                                          int H, int n_evict, int n_tiles, float threshold,
                                                          long long* __restrict__ counts) {
    __shared__ long long s_part[8];
    const int row = blockIdx.x / n_tiles, tile = blockIdx.x - row * n_tiles, b = row / H, h = row - b * H;
    const float thr = F16Traits<T>::to_float(F16Traits<T>::from_float(threshold));
    const uint16_t* p = scores + (int64_t)b * sb + (int64_t)h * sh;
    const int lo = tile * kEvictTile, hi = min(n_evict, lo + kEvictTile);
    long long c = 0;
    for (int s = lo + threadIdx.x; s < hi; s += blockDim.x) c += evicted<T>(p[s], thr);
    c = block_sum_256(c, s_part);
    if (threadIdx.x == 0) counts[blockIdx.x] = c;
}

// counts -> exclusive offsets in place (row-major over (row, tile): torch.where order); the total into *count_out. One CTA of 1024 threads, contiguous segments.
__global__ void __launch_bounds__(1024) evict_scan_kernel(long long* __restrict__ counts, long long R,
                                                          int64_t* __restrict__ count_out) {
    __shared__ long long s_sum[1024];
    const long long per = (R + 1023) / 1024, lo = min(R, (long long)threadIdx.x * per), hi = min(R, lo + per);
    long long t = 0;
    for (long long i = lo; i < hi; ++i) t += counts[i];
    s_sum[threadIdx.x] = t;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {  // inclusive Hillis-Steele scan
        const long long v = threadIdx.x >= (unsigned)o ? s_sum[threadIdx.x - o] : 0;
        __syncthreads();
        s_sum[threadIdx.x] += v;
        __syncthreads();
    }
    long long run = s_sum[threadIdx.x] - t;
    for (long long i = lo; i < hi; ++i) {
        const long long c = counts[i];
        counts[i] = run;
        run += c;
    }
    if (threadIdx.x == 1023) *count_out = s_sum[1023];
}

template <typename T>
__global__ void __launch_bounds__(256) evict_write_kernel(const uint16_t* __restrict__ scores, int64_t sb, int64_t sh,
                                                          int H, int n_evict, int n_tiles, float threshold,
                                                          int64_t shift, const long long* __restrict__ offsets,
                                                          int64_t* __restrict__ b_out, int64_t* __restrict__ h_out,
                                                          int64_t* __restrict__ s_out) {
    __shared__ int s_warp[8];
    const int row = blockIdx.x / n_tiles, tile = blockIdx.x - row * n_tiles, b = row / H, h = row - b * H;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float thr = F16Traits<T>::to_float(F16Traits<T>::from_float(threshold));
    const uint16_t* p = scores + (int64_t)b * sb + (int64_t)h * sh;
    long long base = offsets[blockIdx.x];
    const int hi = min(n_evict, tile * kEvictTile + kEvictTile);
    for (int s0 = tile * kEvictTile; s0 < hi; s0 += 256) {
        const int s = s0 + threadIdx.x;
        const bool f = s < hi && evicted<T>(p[s], thr);
        const uint32_t ballot = __ballot_sync(0xFFFFFFFFu, f);
        if (lane == 0) s_warp[warp] = __popc(ballot);
        __syncthreads();
        int before = 0, tile = 0;
        for (int w = 0; w < 8; ++w) {
            before += w < warp ? s_warp[w] : 0;
            tile += s_warp[w];
        }
        if (f) {
            const long long pos = base + before + __popc(ballot & ((1u << lane) - 1u));
            b_out[pos] = b;
            h_out[pos] = h;
            s_out[pos] = (int64_t)s + shift;
        }
        base += tile;
        __syncthreads();
    }
}

cudaError_t launch_threshold_evict(int dtype, int B, int H, const void* scores, int64_t sb, int64_t sh, int n_evict,
                                   float threshold, int64_t shift, int64_t* b_out, int64_t* h_out, int64_t* s_out,
                                   int64_t* count_out, void* scratch, cudaStream_t st) {
    const int R = B * H, n_tiles = n_evict > 0 ? (n_evict + kEvictTile - 1) / kEvictTile : 1;
    auto* counts = static_cast<long long*>(scratch);
    const auto* sp = static_cast<const uint16_t*>(scores);
    const unsigned grid = (unsigned)R * n_tiles;  // (row, tile), tile fastest; below 2^31 (api.cu)
    return with_dtype(dtype, [&](auto t) -> cudaError_t {
        using T = decltype(t);
        evict_count_kernel<T><<<grid, 256, 0, st>>>(sp, sb, sh, H, n_evict, n_tiles, threshold, counts);
        evict_scan_kernel<<<1, 1024, 0, st>>>(counts, (long long)R * n_tiles, count_out);
        evict_write_kernel<T><<<grid, 256, 0, st>>>(sp, sb, sh, H, n_evict, n_tiles, threshold, shift, counts, b_out,
                                                    h_out, s_out);
        return cudaPeekAtLastError();
    });
}

}  // namespace kvp
