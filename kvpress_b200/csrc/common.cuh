// common.cuh — shared device helpers and the internal (C++) launcher interface.
// sm_90a only. No torch types anywhere in csrc/.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <type_traits>

#include "../../include/kvpress_b200.h"

namespace kvp {

// ---- tiling of the sequence axis for the select / compact stages --------------------------
constexpr int kTile = 256;          // positions per select/compact tile (one per thread)
constexpr int kTileThreads = 256;
constexpr int kSfxStride = 264;     // u16 per tile record: sfx[0..256], gt_hi at [257], padding
constexpr uint16_t kForcedKey = 0xFFFFu;  // ordered key of a forced-keep position
constexpr int kFinalizeTiles = 1;          // 256-position tiles per CTA of the finalize kernels (1: >5 waves at 128k, no tail)
constexpr int kScoreChunkGeneric = 256;   // positions per CTA of the plain streaming score kernels
constexpr int kLagMax = 1024;              // largest LagKV lag_size (partition length) the kernel scores
constexpr int kCurWindowMax = 1024;        // largest CUR local_window_size the kernel scores
constexpr int kCurRankMax = 32;            // most columns of a CUR projection G the kernel scores
constexpr int kSnapMaxRows = 512;          // most query rows G * window per kv head the SnapKV kernels score
// counters[] layout: [0] ticket, [1, 1+R) refine done, [1+R, 1+2R) row ready, then the slot below:
// order-preserving uint image of the largest valid score (for the reference's max+1 sentinel);
// [2+2R, 2+3R) score items done per row (fused Knorm kernel)
__host__ __device__ constexpr int kCounterMaxSlot(int R) { return 1 + 2 * R; }
// [3R + 8]: error flag. A bounded spin-wait that expires (a lost work item: library bug, or a device that
// cannot co-schedule the persistent grid) raises it instead of trapping the whole CUDA context; every CTA
// polls it with its ticket and drains. The host reads it back with kvp_workspace_check().
__host__ __device__ constexpr int kCounterErrSlot(int R) { return 3 * R + 8; }
constexpr uint32_t kSpinLimit = 1u << 22;  // x 64 ns nanosleep ~ 0.3 s

struct Strides3 {
    int64_t b, h, s;
};

// Device view of the scratch area (laid out by layout() in api.cu).
struct Workspace {
    uint16_t* keys;      // [R][S_pad] ordered 16-bit keys of the scores
    uint32_t* hist_hi;   // [R][256]   histogram of key >> 8
    uint32_t* hist_lo;   // [R][256]   histogram of key & 255 among keys with hi == threshold bin
    uint16_t* tile_sfx;  // [R][n_tiles][kSfxStride]
    uint32_t* counters;  // [0] work-queue ticket, [1 + row] refine items done, [1 + R + row] row ready;
                         // zeroed together with the histograms
    uint2* row_meta;     // [R] {threshold key T, ties to take}
    uint2* tile_prefix;  // [R][n_tiles] {kept (> T) + 1, tied (== T) + 1} positions in the tiles before;
                         // zero = row not scanned yet
    int R;
    void* scorer;        // scorer-specific scratch (SnapKV / ExpectedAttention / KeyDiff / CriticalKV /
                         // ObservedAttention / NonCausalAttention / CUR / Merging / ThinK; LagKV needs none)
    size_t scorer_bytes;
    int S_pad;
    int n_tiles;
};

struct Dims {
    int B, H, Hq, S, D, n_kept;
    int R;  // B * H rows
    Strides3 ks, vs;
};

// ---- 16-bit float -> ordered unsigned key (same for bf16 and fp16: sign-magnitude) --------
// inf_bits = 0x7F80 for bf16, 0x7C00 for fp16: anything above it (either sign) is a NaN, which
// torch.topk ranks above every number -> largest key.
__host__ __device__ __forceinline__ uint16_t ordered_key16(uint16_t bits, uint16_t inf_bits) {
    if ((bits & 0x7FFFu) > inf_bits) return 0xFFFFu;  // NaN
    if (bits == 0x8000u) bits = 0;                    // -0 == +0 (torch.topk compares by value)
    return (bits & 0x8000u) ? (uint16_t)(~bits) : (uint16_t)(bits | 0x8000u);
}
__host__ __device__ __forceinline__ uint16_t key16_to_bits(uint16_t key) {
    return (key & 0x8000u) ? (uint16_t)(key & 0x7FFFu) : (uint16_t)(~key);
}

// ---- float -> order-preserving uint32 image, and back --------------------------------------------
// Unsigned comparison of images is the float order, with -0 below +0 and NaNs outside +-inf by their sign bit; zero
// (the value counters are cleared to) is below every image of a number, so atomicMax on it works from a cleared slot.
__device__ __forceinline__ uint32_t ordered_f32(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ordered_f32_to_float(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

template <typename T>
struct F16Traits;
template <>
struct F16Traits<__nv_bfloat16> {
    static __device__ __forceinline__ float2 unpack2(uint32_t w) {
        return make_float2(__uint_as_float(w << 16), __uint_as_float(w & 0xFFFF0000u));
    }
    static __device__ __forceinline__ uint16_t from_float(float f) {
        return __bfloat16_as_ushort(__float2bfloat16_rn(f));
    }
    static __device__ __forceinline__ float to_float(uint16_t b) {
        return __uint_as_float(((uint32_t)b) << 16);
    }
    static constexpr uint16_t kInfBits = 0x7F80u;
    static constexpr int kMmaFormat = 1;  // wgmma operand type: BF16
};
template <>
struct F16Traits<__half> {
    static __device__ __forceinline__ float2 unpack2(uint32_t w) {
        __half2 h = *reinterpret_cast<__half2*>(&w);
        return __half22float2(h);
    }
    static __device__ __forceinline__ uint16_t from_float(float f) {
        return __half_as_ushort(__float2half_rn(f));
    }
    static __device__ __forceinline__ float to_float(uint16_t b) {
        return __half2float(__ushort_as_half(b));
    }
    static constexpr uint16_t kInfBits = 0x7C00u;
    static constexpr int kMmaFormat = 0;  // F16
};

// ---- host: the two dispatches every launcher shares -------------------------------------------------------------
// Calls f with a value of the cache's 16-bit type (KVP_BF16 or KVP_F16; api.cu rejects any other dtype).
template <typename F>
static inline decltype(auto) with_dtype(int dtype, F&& f) {
    if (dtype == KVP_BF16) return f(__nv_bfloat16{});
    return f(__half{});
}

// Lanes that cover one cache row with 16-byte loads (8 elements per lane), as instantiated by the CUDA-core score
// kernels: a row of D <= 256 elements takes the first entry >= D / 8. The tests read this list.
constexpr int kLanesPerRow[] = {4, 8, 16, 32};
constexpr int kNumLanesPerRow = sizeof(kLanesPerRow) / sizeof(kLanesPerRow[0]);

// Calls f with std::integral_constant<int, LPR> of the lane count of head_dim D.
template <int I = 0, typename F>
static inline void with_lanes_per_row(int D, F&& f) {
    constexpr int lpr = kLanesPerRow[I];
    if constexpr (I + 1 == kNumLanesPerRow) {
        f(std::integral_constant<int, lpr>{});
    } else {
        if (D / 8 <= lpr) f(std::integral_constant<int, lpr>{});
        else with_lanes_per_row<I + 1>(D, f);
    }
}

// ---- cache-hinted 128-bit global accesses ---------------------------------------------------
// 128-bit accesses take an explicit createpolicy handle through .L2::cache_hint.
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ int4 ldg_hint(const void* p, uint64_t pol) {
    int4 r;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.s32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p), "l"(pol));
    return r;
}
__device__ __forceinline__ int4 ldg_plain(const void* p) {
    int4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}
__device__ __forceinline__ void stg_hint(void* p, const int4& v, uint64_t pol) {
    asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.s32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(p),
                 "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "l"(pol)
                 : "memory");
}

// ---- programmatic dependent launch (PDL) ------------------------------------------------------------------
// The select+compact kernel is launched with cudaLaunchAttributeProgrammaticStreamSerialization: its CTAs may
// become resident while the LAST wave of the score / finalize kernel in front of it is still draining (that kernel
// calls pdl_launch_dependents() at its start) and park in pdl_wait() until that grid has completed and flushed, so
// the launch latency and the ramp of the persistent grid are off the critical path. Both are no-ops for a plain launch.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                     Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// ---- 256-bin suffix search, executed by ONE full warp ----------------------------------------
// Finds the largest bin b with sum_{i>=b} hist[i] >= need (need >= 1) and returns
// above = sum_{i>b} hist[i]. hist lives in shared memory. All 32 lanes get the result.
__device__ __forceinline__ void warp_suffix_find(const uint32_t* hist, uint32_t need, int lane,
                                                 int& bin, uint32_t& above) {
    const int top = 255 - 8 * lane;  // this lane owns bins top, top-1, ..., top-7
    uint32_t h[8];
    uint32_t lane_sum = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        h[i] = hist[top - i];
        lane_sum += h[i];
    }
    uint32_t incl = lane_sum;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, off);
        if (lane >= off) incl += t;
    }
    const unsigned crossed = __ballot_sync(0xFFFFFFFFu, incl >= need);
    int my_bin = 0;
    uint32_t my_above = 0;
    const int first = crossed ? (__ffs(crossed) - 1) : 31;
    if (lane == first) {
        uint32_t run = incl - lane_sum;
        my_bin = top - 7;
        my_above = incl - h[7];
        bool found = false;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            if (!found && run + h[i] >= need) {
                my_bin = top - i;
                my_above = run;
                found = true;
            }
            run += h[i];
        }
    }
    bin = __shfl_sync(0xFFFFFFFFu, my_bin, first);
    above = __shfl_sync(0xFFFFFFFFu, my_above, first);
}

// Adds a CTA's shared-memory histogram to the row histogram (call after a __syncthreads()).
__device__ __forceinline__ void flush_row_hist(const uint32_t* shist, int row, const Workspace& ws) {
    const int tid = threadIdx.x;
    if (tid < 256) {
        const uint32_t c = shist[tid];
        if (c) atomicAdd(&ws.hist_hi[(size_t)row * 256 + tid], c);
    }
}

// Adds each lane's bin (256: none) to the shared histogram. The atomics are warp-aggregated with match.any so heavily
// tied scores (bf16 norms take ~100 distinct values) do not serialise on one address. Every lane of the warp calls it.
__device__ __forceinline__ void warp_hist_add(uint32_t* shist, unsigned bin) {
    const unsigned peers = __match_any_sync(0xFFFFFFFFu, bin);
    if (bin < 256u && (threadIdx.x & 31) == (__ffs(peers) - 1)) atomicAdd(&shist[bin], __popc(peers));
}

// Common tail of every score kernel: KPT keys (and optionally scores) per thread staged in shared
// memory for a chunk of KPT*blockDim positions starting at s_begin -> coalesced global writes + row
// histogram of (key >> 8).
// Call with all threads of a 256-thread CTA after a __syncthreads(); shist must be zeroed.
template <int KPT, bool kFlushHist = true>
__device__ __forceinline__ void flush_chunk_keys(const uint16_t* skeys, const uint16_t* sscores,
                                                 uint32_t* shist, int row, int s_begin, int S,
                                                 const Workspace& ws, uint16_t* scores_out) {
    const int tid = threadIdx.x;
    const int s0 = s_begin + tid * KPT;
    uint16_t k[KPT];
#pragma unroll
    for (int i = 0; i < KPT; ++i) k[i] = ((s0 + i) < S) ? skeys[tid * KPT + i] : (uint16_t)0;
    // the keys buffer is padded to a multiple of kTile per row: unconditional vector store
    uint16_t* kdst = ws.keys + (size_t)row * ws.S_pad + s0;
    if (KPT == 4) {
        // a KPT*256-position chunk may reach past the row's padding (S_pad is a multiple of 256 only)
        if (s0 < ws.S_pad) {
            uint2 pk;
            pk.x = (uint32_t)k[0] | ((uint32_t)k[1 % KPT] << 16);
            pk.y = (uint32_t)k[2 % KPT] | ((uint32_t)k[3 % KPT] << 16);
            *reinterpret_cast<uint2*>(kdst) = pk;
        }
    } else {
#pragma unroll
        for (int i = 0; i < KPT; ++i) kdst[i] = k[i];
    }
    if (scores_out != nullptr) {
        uint16_t* dst = scores_out + (size_t)row * S + s0;
#pragma unroll
        for (int i = 0; i < KPT; ++i)
            if (s0 + i < S) dst[i] = sscores[tid * KPT + i];
    }
#pragma unroll
    for (int i = 0; i < KPT; ++i) warp_hist_add(shist, ((s0 + i) < S) ? (unsigned)(k[i] >> 8) : 256u);
    if (kFlushHist) {
        __syncthreads();
        flush_row_hist(shist, row, ws);
    }
}

// ---- the end of every score stage ------------------------------------------------------------------------------
// What the select + compact stage reads: each score rounded once to the cache dtype, its ordered key in ws.keys and
// the histogram of the key's high byte in ws.hist_hi.

// The one rounding: fp32 values as the presses define them, fp64 where a press evaluates its score in double.
template <typename T>
__device__ __forceinline__ uint16_t round_once(float v) {
    return F16Traits<T>::from_float(v);
}
template <typename T>
__device__ __forceinline__ uint16_t round_once(double v) {
    if constexpr (std::is_same<T, __nv_bfloat16>::value) return __bfloat16_as_ushort(__double2bfloat16(v));
    else return __half_as_ushort(__double2half(v));
}

// A score tile of a 256-thread CTA: thread tid owns positions s = s_begin + tid * KPT + i, i < KPT. Below S, a
// position in [forced_lo, forced_hi) is forced (key kForcedKey, score 0); any other gets value(i, s) rounded once and
// its ordered key. Both are staged in skeys / sscores (KPT * 256 each), then the keys, the scores (scores_out may be
// null) and the histogram go out through flush_chunk_keys; shist must be zeroed. Unless max_valid is null, raises
// *max_valid to the largest rounded score of the thread's unforced positions (see publish_max_valid).
template <typename T, int KPT, bool kFlushHist = true, typename Value>
__device__ __forceinline__ void score_tile_epilogue(uint16_t* skeys, uint16_t* sscores, uint32_t* shist, int row,
                                                    int s_begin, int S, int forced_lo, int forced_hi,
                                                    const Workspace& ws, uint16_t* scores_out, float* max_valid,
                                                    Value value) {
    const int tid = threadIdx.x;
#pragma unroll
    for (int i = 0; i < KPT; ++i) {
        const int s = s_begin + tid * KPT + i;
        uint16_t bits = 0, key = 0;
        if (s < S) {
            if (s >= forced_lo && s < forced_hi) {
                key = kForcedKey;
            } else {
                bits = round_once<T>(value(i, s));
                key = ordered_key16(bits, F16Traits<T>::kInfBits);
                if (max_valid) *max_valid = fmaxf(*max_valid, F16Traits<T>::to_float(bits));
            }
        }
        skeys[tid * KPT + i] = key;
        sscores[tid * KPT + i] = bits;
    }
    __syncthreads();
    flush_chunk_keys<KPT, kFlushHist>(skeys, sscores, shist, row, s_begin, S, ws, scores_out);
}

// Score kernels that stage their own keys (one position per thread): keys, scores and histogram for a compress
// call (want_keys), the scores alone for a score-only call. Call after a __syncthreads().
__device__ __forceinline__ void flush_or_store_scores(const uint16_t* skeys, const uint16_t* sscores, uint32_t* shist,
                                                      int row, int s_begin, int S, const Workspace& ws,
                                                      uint16_t* scores_out, bool want_keys) {
    const int tid = threadIdx.x;
    if (want_keys) flush_chunk_keys<1>(skeys, sscores, shist, row, s_begin, S, ws, scores_out);
    else if (s_begin + tid < S) scores_out[(size_t)row * S + s_begin + tid] = sscores[tid];
}

// Raises counters[kCounterMaxSlot] to the CTA's largest valid score m (-inf: none), for the reference's max + 1
// sentinel that fill_sentinel_kernel writes. Call with all threads of a 256-thread CTA; the CTA's shared histogram may
// be flushed after it returns.
__device__ __forceinline__ void publish_max_valid(float m, const Workspace& ws) {
    __shared__ float s_max[kTileThreads / 32];
    const int tid = threadIdx.x;
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xFFFFFFFFu, m, off));
    if ((tid & 31) == 0) s_max[tid >> 5] = m;
    __syncthreads();
    if (tid == 0) {
        m = s_max[0];
        for (int w = 1; w < kTileThreads / 32; ++w) m = fmaxf(m, s_max[w]);
        if (m > -INFINITY) atomicMax(&ws.counters[kCounterMaxSlot(ws.R)], ordered_f32(m));
    }
}

// ---- host: per-device launch properties, resolved once per (device, kernel) and cached (tmap.cu) ----
// Nothing below is re-queried on the launch path: the C-ABI calls are host-latency sensitive
// (DecodingPress compactions, per-layer prefill hooks).
int device_sm_count();                         // SM count of the CURRENT device
constexpr int kMaxDevices = 64;
// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (kernel, device). The kernel is the template argument, so
// every kernel has its own cache.
template <auto kKern>
static inline cudaError_t ensure_dynamic_smem(int bytes) {
    static unsigned long long done = 0;  // bit per device; a lost race only repeats the idempotent call
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < kMaxDevices && ((done >> dev) & 1ull)) return cudaSuccess;
    e = cudaFuncSetAttribute(kKern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess && dev >= 0 && dev < kMaxDevices) done |= 1ull << dev;
    return e;
}
// resident CTAs per SM of a kernel (occupancy query) once per (kernel, device)
template <auto kKern>
static inline int cached_ctas_per_sm(int threads, int dyn_smem = 0) {
    static int per_dev[kMaxDevices] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) dev = 0;
    if (per_dev[dev] == 0) {
        int per_sm = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kKern, threads, dyn_smem);
        per_dev[dev] = per_sm > 0 ? per_sm : 1;
    }
    return per_dev[dev];
}

// ---- host: workspace layouts ------------------------------------------------------------------
inline size_t align256(size_t x) { return (x + 255) / 256 * 256; }

// Hands out consecutive regions of a buffer, each 256-byte aligned. With a null base every region is null and only
// `bytes` is tallied, so one function both sizes a layout and carves it.
struct Carve {
    char* base;
    size_t bytes = 0;
    explicit Carve(void* b) : base(static_cast<char*>(b)) {}
    template <typename T>
    T* take(size_t count) {
        T* p = base ? reinterpret_cast<T*>(base + bytes) : nullptr;
        bytes = align256(bytes + count * sizeof(T));
        return p;
    }
};

// ---- launchers implemented in the .cu files (host, C++ linkage) -------------------------------
cudaError_t launch_knorm_score(const Dims& d, int dtype, const void* K, const Workspace& ws,
                               void* scores_out, bool want_keys, cudaStream_t st);
cudaError_t launch_knorm_fused(const Dims& d, int dtype, const void* K, const void* V, void* K_out,
                               void* V_out, int32_t* idx_out, void* scores_out, const Workspace& ws,
                               cudaStream_t st);
bool knorm_cluster_applicable(const Dims& d);
cudaError_t launch_knorm_cluster(const Dims& d, int dtype, const void* K, const void* V, void* K_out, void* V_out,
                                 int32_t* idx_out, void* scores_out, cudaStream_t st);
cudaError_t launch_keys_from_scores(const Dims& d, int dtype, const void* scores, int64_t sb, int64_t sh,
                                    const Workspace& ws, cudaStream_t st);
cudaError_t launch_select_compact(const Dims& d, const void* K, const void* V, void* K_out,
                                  void* V_out, int32_t* idx_out, const Workspace& ws,
                                  cudaStream_t st);
cudaError_t launch_select_compact_rerotate(const Dims& d, int dtype, const void* K, const void* V,
                                           void* K_out, void* V_out, int32_t* idx_out,
                                           const Workspace& ws, const float* inv_freq, cudaStream_t st);
cudaError_t launch_streaming_score(const Dims& d, int dtype, int n_sink, void* scores_out,
                                   cudaStream_t st);
cudaError_t launch_streaming_compress(const Dims& d, int n_sink, const void* K, const void* V,
                                      void* K_out, void* V_out, int32_t* idx_out,
                                      cudaStream_t st);

size_t snapkv_scratch_bytes(const Dims& d, int window);
cudaError_t launch_snapkv_score(const Dims& d, int dtype, const void* K, const void* q_window,
                                int window, int kernel_size, const Workspace& ws,
                                void* scores_out, cudaStream_t st);
size_t keydiff_scratch_bytes(const Dims& d);
cudaError_t launch_keydiff_score(const Dims& d, int dtype, const void* K, const Workspace& ws,
                                 void* scores_out, bool want_keys, cudaStream_t st);
size_t ea_scratch_bytes(const Dims& d);
cudaError_t launch_fill_sentinel(int dtype, void* scores_out, int R, int S, int lo, int hi,
                                 const Workspace& ws, cudaStream_t st);
cudaError_t launch_ea_score(const Dims& d, int dtype, const void* K, const void* V, const void* mu,
                            const void* cov, float eps, int n_sink, int use_vnorm,
                            const Workspace& ws, void* scores_out, cudaStream_t st);
size_t criticalkv_scratch_bytes(const Dims& d);
void* criticalkv_scratch_scores(const Dims& d, const Workspace& ws);
cudaError_t launch_criticalkv_score(const Dims& d, int dtype, const void* V, const void* base, int64_t sb,
                                    int64_t sh, const void* wo, int hidden, int64_t wo_stride, float eps, int n_first,
                                    const Workspace& ws, void* scores_out, cudaStream_t st);
size_t observed_attention_scratch_bytes(const Dims& d, int n_q);
cudaError_t launch_observed_attention_score(const Dims& d, int dtype, const void* K, const void* q, int n_q,
                                            float scaling, const Workspace& ws, void* scores_out, cudaStream_t st);
size_t non_causal_attention_scratch_bytes(const Dims& d);
bool non_causal_attention_supported(const Dims& d, int chunk_size);
cudaError_t launch_non_causal_attention_score(const Dims& d, int dtype, const void* K, const void* V, const void* q,
                                              int chunk_size, const Workspace& ws, void* scores_out, cudaStream_t st);
cudaError_t launch_lagkv_score(const Dims& d, int dtype, const void* K, const void* V, int n_sink, int lag_size,
                               int cross, const Workspace& ws, void* scores_out, bool want_keys, cudaStream_t st);
size_t cur_scratch_bytes(const Dims& d);
cudaError_t launch_cur_score(const Dims& d, int dtype, const void* K, const void* V, int num_sinks, int leverage_type,
                             int window, const float* G, int r, const Workspace& ws, void* scores_out,
                             cudaStream_t st);
size_t merging_scratch_bytes(const Dims& d);
int32_t* merging_scratch_kept(const Dims& d, const Workspace& ws);
cudaError_t launch_merging(const Dims& d, int dtype, const void* K, const void* V, const int32_t* kept, float threshold,
                           double merge_fraction, void* V_out, int32_t* target_out, float* sim_out, const Workspace& ws,
                           cudaStream_t st);
// ObservedAttention's column-sum pass (observed_attention.cu) over the key tiles [0, n_ktiles) of every row: colsum[s] =
// sum over the n_q query rows r of the kv head's G query heads of exp2(c q_r.k_s + cb[r]), causal for the query
// positions S - n_q + r. cb is [B Hq][n_q] in log2 units. D = 64 / 128 only (cudaErrorNotSupported otherwise).
cudaError_t launch_attention_colsum(const Dims& d, int dtype, const void* K, const void* q, int n_q, int n_ktiles,
                                    float c, const float* cb, float* colsum, int S_pad, cudaStream_t st);
size_t finch_scratch_bytes(const Dims& d, int window);
int32_t* finch_scratch_kept(const Dims& d, const Workspace& ws);
cudaError_t launch_finch_score(const Dims& d, int dtype, const void* K, const void* q_window, int window,
                               int normalize, const Workspace& ws, void* scores_out, cudaStream_t st);
// the chunk select and the gather of FinchPress's chunked selection (select_compact.cu) on the keys in ws; `kept` is
// [R][n_kept] scratch; inv_freq null: exact gathers
cudaError_t launch_select_compact_chunked(const Dims& d, int dtype, const void* K, const void* V, void* K_out,
                                          void* V_out, int32_t* idx_out, const Workspace& ws, int chunk_length,
                                          int chunk_kept, int tail_kept, int32_t* kept, const float* inv_freq,
                                          cudaStream_t st);
size_t think_scratch_bytes(const Dims& d);
// a memset of the row tickets, the reduce + select kernel and the zero kernel on `scratch` (think_scratch_bytes)
cudaError_t launch_think_prune(const Dims& d, int dtype, void* K, const void* q, int window, int n_pruned,
                               int32_t* pruned_out, float* scores_out, void* scratch, cudaStream_t st);
// CAMPress selects once per batch element, on the head mean of the scores: its selection regions are laid out for
// the B rows of cam_selection_dims(d), and cam_scratch_bytes(d) (sized for n_merge = S - n_kept) follows them.
Dims cam_selection_dims(const Dims& d);
size_t cam_scratch_bytes(const Dims& d);
// head mean + keys, selection, and with n_merge > 0 candidates and probabilities, then the merge + compaction; `ws`
// is carved for cam_selection_dims(d) and its selection regions are cleared
cudaError_t launch_cam_compress(const Dims& d, int dtype, const void* scores, int64_t sb, int64_t sh, const void* K,
                                const void* V, const float* A, int64_t ab, int64_t ah, int n_merge, int budget,
                                const float* u, void* K_out, void* V_out, float* A_out, int64_t ob, int64_t oh,
                                int32_t* idx_out, int32_t* merge_idx_out, float* prob_out, const Workspace& ws,
                                cudaStream_t st);

// KVzapPress (kvzap.cu): the shapes the kernels take, and the B S at or below which the W1-spread kernel runs
constexpr int kZapMaxHidden = 16384;
constexpr int kZapMaxHd = 2048;
constexpr int kZapMaxHeads = 32;
constexpr int kZapGemvRows = 32;
constexpr int kZapGemvUnits = 8;  // hidden units per CTA of the W1-spread kernel
// the partials [parts][Hkv][B S] fp32 (parts for hd = kZapMaxHd), then the scores a compress call selects on
size_t kvzap_scratch_bytes(const Dims& d);
void* kvzap_scratch_scores(const Dims& d, const Workspace& ws);
// hd == 0: the linear model (w1 = W, b1 = b); hd > 0: partials into ws.scorer, then the reduce
cudaError_t launch_kvzap_score(const Dims& d, int dtype, const void* x, int64_t xb, int64_t xs, int hidden, int hd,
                               const void* w1, const void* b1, const void* w2, const void* b2, const Workspace& ws,
                               void* scores_out, cudaStream_t st);
// per-(row, tile of kEvictTile positions) counts into `scratch` (8 B each), their scan, the ordered write
constexpr int kEvictTile = 4096;
cudaError_t launch_threshold_evict(int dtype, int B, int H, const void* scores, int64_t sb, int64_t sh, int n_evict,
                                   float threshold, int64_t shift, int64_t* b_out, int64_t* h_out, int64_t* s_out,
                                   int64_t* count_out, void* scratch, cudaStream_t st);

}  // namespace kvp
