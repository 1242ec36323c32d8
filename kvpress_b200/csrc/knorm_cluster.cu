// knorm_cluster.cu — KnormPress score + top-k + compaction of a SMALL cache in ONE launch, no scratch, no memset:
// the DecodingPress compaction (reference kvpress/presses/decoding_press.py:68-111 -> scorer_press.py:76-102 with
// knorm_press.py:38 as the score), e.g. [1, 8, 2560, 128] -> [1, 8, 2048, 128] every 512 generated tokens per layer.
//
// At these sizes (tens of MB) the call is latency-bound: the multi-kernel path spends its time in launch gaps, a
// memset node, global atomics and spin-waits between CTAs. Here one thread-block CLUSTER owns one (b, h) row:
//   1. every CTA requests its whole slice of the row up front as one bulk copy (cp.async.bulk, the TMA engine) per row —
//      every K row, and every V row when both fit — completing on one mbarrier: the slice is one memory round trip and
//      a few hundred instructions; then one thread per row scores it from shared memory (fp32 sum of squares, one
//      rounding; rows sit at a pitch of 2*D + 16 bytes so that the per-thread row reads are bank-conflict free);
//   2. the 16-bit ordered keys of the slice are pushed into the shared memory of every CTA of the cluster
//      (distributed shared memory), ONE cluster barrier;
//   3. every CTA now holds the keys of the whole row and derives the exact threshold, the tie budget and the number
//      of kept positions in front of its slice on its own (a search over the threshold's bits, two per step:
//      register-only counts, redux.sync warp sums, one barrier per step — no atomics);
//   4. it ranks its slice and writes the kept K (and V) rows from shared memory with one bulk store per row — V through
//      registers from global memory when it was not staged — to their final places (ascending positions, ties to the lowest positions — same rule as select_compact.cu).
// No global atomics, no flags, no workspace: the only inter-CTA communication is the key exchange.
#include <cooperative_groups.h>

#include "common.cuh"
#include "umma.cuh"

namespace cg = cooperative_groups;

namespace kvp {

constexpr int kClThreads = 256;
constexpr int kClMaxKeysPerThread = 24;  // keys of the row a thread holds in registers: S <= 256 * 24 = 6144
constexpr int kClMaxSmem = 200 * 1024;  // K slice + keys of the row + lists must fit one CTA's shared memory

struct ClusterPlan {
    int C;        // CTAs per cluster (= per row)
    int P;        // positions per CTA (multiple of 8)
    int v_smem;   // 1: the V rows of the slice are staged in shared memory too (they fit)
    int smem;     // dynamic shared memory bytes
    bool ok;
};

__host__ __device__ constexpr int cl_pitch(int D) { return D * 2; }  // bytes between staged rows (dense: runs of rows
                                                                      // move as one bulk copy)

static ClusterPlan cluster_plan(const Dims& d, int C) {
    ClusterPlan pl;
    pl.C = C;
    pl.P = ((d.S + C - 1) / C + 7) / 8 * 8;
    const size_t tile = (size_t)pl.P * cl_pitch(d.D);
    const size_t keys = (size_t)C * pl.P * 2;
    const size_t list = (size_t)pl.P * 4;
    pl.v_smem = (2 * tile + keys + list + 64 <= (size_t)kClMaxSmem) ? 1 : 0;
    pl.smem = (int)((pl.v_smem ? 2 : 1) * tile + keys + list + 64);
    pl.ok = pl.smem <= kClMaxSmem && d.S <= kClThreads * kClMaxKeysPerThread;
    return pl;
}

// one row: global -> shared through the bulk-copy engine, completion counted on `bar`
__device__ __forceinline__ void bulk_load_row(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     umma::smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(umma::smem_u32(bar))
                 : "memory");
}
// one row: shared -> global
__device__ __forceinline__ void bulk_store_row(void* gmem_dst, const void* smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst),
                 "r"(umma::smem_u32(smem_src)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void bulk_store_wait() {
    asm volatile("cp.async.bulk.commit_group;\n\tcp.async.bulk.wait_group.read 0;" ::: "memory");
}

template <typename T, int KPT>  // KPT: keys of the row per thread held in registers (S <= 256 * KPT)
__global__ void __launch_bounds__(kClThreads, 1)
knorm_cluster_kernel(const T* __restrict__ K, const T* __restrict__ V, Strides3 ks, Strides3 vs,
                     char* __restrict__ K_out, char* __restrict__ V_out, int32_t* __restrict__ idx_out,
                     uint16_t* __restrict__ scores_out, int H, int S, int D, int n_kept, int P, int v_smem) {
    extern __shared__ __align__(16) unsigned char smem[];
    cg::cluster_group cluster = cg::this_cluster();
    const int C = (int)cluster.num_blocks();
    const int rank = (int)cluster.block_rank();
    const int row = blockIdx.y, b = row / H, h = row % H;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int nvec = D >> 3;
    const int pitch = cl_pitch(D);
    const uint32_t row_bytes = (uint32_t)D * 2;

    const size_t tile_bytes = (size_t)P * pitch;
    unsigned char* ktile = smem;                     // [P] rows at `pitch`
    unsigned char* vtile = smem + tile_bytes;        // [P] rows, only if v_smem
    unsigned char* after = smem + (v_smem ? 2 : 1) * tile_bytes;
    uint16_t* all_keys = reinterpret_cast<uint16_t*>(after);                             // [C][P]
    int* list = reinterpret_cast<int*>(after + (size_t)C * P * 2);                       // [P] kept local positions
    __shared__ uint32_t red[2][8];
    __shared__ uint32_t red3[2][3][8];
    __shared__ __align__(8) uint64_t load_bar;

    // ---- 1. stage the slice [start, start + P): one bulk copy per row, all in flight at once --------------------------
    const int start = rank * P;
    const int n_rows = max(0, min(P, S - start));
    if (tid == 0) {
        umma::mbar_init(&load_bar, 1);
        umma::mbar_fence_init();
    }
    __syncthreads();
    {
        const char* k_src = reinterpret_cast<const char*>(K) + ((int64_t)b * ks.b + (int64_t)h * ks.h) * 2;
        const char* v_src = reinterpret_cast<const char*>(V) + ((int64_t)b * vs.b + (int64_t)h * vs.h) * 2;
        if (tid == 0) umma::mbar_arrive_expect_tx(&load_bar, (uint32_t)n_rows * row_bytes * (v_smem ? 2u : 1u));
        // rows that are dense in global memory (the usual cache layout) move as 16 KB bulk copies, a handful per CTA;
        // strided views fall back to one bulk copy per row (the copy engine then spends ~5 ns per row)
        constexpr int kChunk = 16384;
        const uint32_t slice_bytes = (uint32_t)n_rows * row_bytes;
        const int n_chunks = (int)((slice_bytes + kChunk - 1) / kChunk);
        if (ks.s == D) {
            for (int c = tid; c < n_chunks; c += kClThreads) {
                const uint32_t off = (uint32_t)c * kChunk, len = min((uint32_t)kChunk, slice_bytes - off);
                bulk_load_row(ktile + off, k_src + (int64_t)start * row_bytes + off, len, &load_bar);
            }
        } else {
            for (int r = tid; r < n_rows; r += kClThreads)
                bulk_load_row(ktile + (size_t)r * pitch, k_src + (int64_t)(start + r) * ks.s * 2, row_bytes, &load_bar);
        }
        if (v_smem) {
            if (vs.s == D) {
                for (int c = kClThreads - 1 - tid; c < n_chunks; c += kClThreads) {  // other threads than the K chunks
                    const uint32_t off = (uint32_t)c * kChunk, len = min((uint32_t)kChunk, slice_bytes - off);
                    bulk_load_row(vtile + off, v_src + (int64_t)start * row_bytes + off, len, &load_bar);
                }
            } else {
                for (int r = tid; r < n_rows; r += kClThreads)
                    bulk_load_row(vtile + (size_t)r * pitch, v_src + (int64_t)(start + r) * vs.s * 2, row_bytes, &load_bar);
            }
        }
    }
    // all CTAs of the cluster have started (their shared memory exists) before anyone writes into it; the barrier
    // overlaps the loads in flight
    cluster.sync();
    umma::mbar_wait(&load_bar, 0);

    // ---- score the slice from shared memory: one thread per row, fixed summation order ----------------------------------
    uint16_t* my_keys = all_keys + (size_t)rank * P;
    for (int r = tid; r < P; r += kClThreads) {
        uint16_t key = 0;
        if (r < n_rows) {
            // rows are dense (pitch = 2 D): a thread starts at piece r % nvec so that the 8 lanes of a quarter warp hit
            // 8 different bank groups; the order in which a row's pieces are summed therefore depends on the row's
            // place in the slice — a last-bit effect in fp32, far below the one rounding to the 16-bit score
            const int4* rp = reinterpret_cast<const int4*>(ktile + (size_t)r * pitch);
            float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
            int c = r % nvec;
            for (int j = 0; j < nvec; ++j) {
                const int4 v = rp[c];
                c = (c + 1 == nvec) ? 0 : c + 1;
                const float2 f0 = F16Traits<T>::unpack2((uint32_t)v.x), f1 = F16Traits<T>::unpack2((uint32_t)v.y);
                const float2 f2 = F16Traits<T>::unpack2((uint32_t)v.z), f3 = F16Traits<T>::unpack2((uint32_t)v.w);
                s0 = fmaf(f0.x, f0.x, s0); s1 = fmaf(f0.y, f0.y, s1);
                s2 = fmaf(f1.x, f1.x, s2); s3 = fmaf(f1.y, f1.y, s3);
                s0 = fmaf(f2.x, f2.x, s0); s1 = fmaf(f2.y, f2.y, s1);
                s2 = fmaf(f3.x, f3.x, s2); s3 = fmaf(f3.y, f3.y, s3);
            }
            // -sqrt(ss) rounded once to the storage dtype (negation is exact): knorm_press.py:38
            const uint16_t bits = F16Traits<T>::from_float(sqrtf((s0 + s1) + (s2 + s3))) ^ 0x8000u;
            key = ordered_key16(bits, F16Traits<T>::kInfBits);
            if (scores_out != nullptr) scores_out[(size_t)row * S + start + r] = bits;
        }
        my_keys[r] = key;
    }
    __syncthreads();

    // ---- 2. all-gather of the keys through distributed shared memory ---------------------------------------------
    {
        const int n8 = P / 4;  // 8-byte pieces (4 keys) of the slice
        const uint2* src = reinterpret_cast<const uint2*>(my_keys);
        for (int peer = 1; peer < C; ++peer) {
            const int dst_rank = (rank + peer) % C;  // spread the traffic over the peers
            uint2* dst = reinterpret_cast<uint2*>(cluster.map_shared_rank(all_keys, dst_rank) + (size_t)rank * P);
            for (int i = tid; i < n8; i += kClThreads) dst[i] = src[i];
        }
    }
    cluster.sync();  // release / acquire at cluster scope: every slice of all_keys is complete everywhere

    // ---- 3. exact threshold of the row, computed redundantly by every CTA -----------------------------------------
    // The whole row's keys sit in shared memory (position s at all_keys[s]: slices are contiguous); every thread takes
    // the positions tid, tid + 256, ... into registers. The threshold T = the n_kept-th largest key is found by a
    // search over its bits, two per step: T |= the largest 2-bit digit d with count(key >= T | d << shift) >= n_kept.
    // No shared-memory atomics: Knorm scores of a row take ~100 distinct values, histogram bins would be hammered by
    // every warp at once.
    uint32_t myk[KPT];
    const int n_mine = (S + kClThreads - 1) / kClThreads;  // <= KPT (launcher)
#pragma unroll
    for (int i = 0; i < KPT; ++i) {
        const int s = i * kClThreads + tid;
        myk[i] = (i < n_mine && s < S) ? (uint32_t)all_keys[s] + 1u : 0u;  // +1: 0 marks "no position", below any key
    }
    // block-wide sums of three counters: redux.sync per warp, one barrier; `slot` alternates between calls
    auto block_sum3 = [&](uint32_t a, uint32_t b2, uint32_t c, int slot, uint32_t (&out)[3]) {
        a = __reduce_add_sync(0xFFFFFFFFu, a);
        b2 = __reduce_add_sync(0xFFFFFFFFu, b2);
        c = __reduce_add_sync(0xFFFFFFFFu, c);
        if (lane == 0) {
            red3[slot][0][warp] = a;
            red3[slot][1][warp] = b2;
            red3[slot][2][warp] = c;
        }
        __syncthreads();
        out[0] = out[1] = out[2] = 0;
#pragma unroll
        for (int w = 0; w < 8; ++w) {
            out[0] += red3[slot][0][w];
            out[1] += red3[slot][1][w];
            out[2] += red3[slot][2][w];
        }
    };
    uint32_t T1 = 0;  // threshold in the shifted (+1) key space: 17 bits = bit 16 alone, then 8 two-bit digits
    int it = 0;
#pragma unroll 1
    for (int shift = 16; shift >= 0; shift -= 2, ++it) {
        const uint32_t c1 = T1 | (1u << shift), c2 = T1 | (2u << shift), c3 = T1 | (3u << shift);
        const bool single = shift == 16;  // digits 2 and 3 would be bits 17, 18: no key reaches them
        uint32_t n1 = 0, n2 = 0, n3 = 0;
#pragma unroll
        for (int i = 0; i < KPT; ++i) {
            n1 += myk[i] >= c1;
            n2 += myk[i] >= c2;
            n3 += myk[i] >= c3;
        }
        uint32_t tot[3];
        block_sum3(n1, single ? 0u : n2, single ? 0u : n3, it & 1, tot);
        const uint32_t need = (uint32_t)n_kept;
        if (!single && tot[2] >= need) T1 = c3;
        else if (!single && tot[1] >= need) T1 = c2;
        else if (tot[0] >= need) T1 = c1;
    }
    // kept (> T) positions of the row, and kept / tied positions in front of this CTA's slice
    uint32_t n_gt = 0, gt_b = 0, eq_b = 0;
#pragma unroll
    for (int i = 0; i < KPT; ++i) {
        const bool front = (i * kClThreads + tid) < start;
        n_gt += myk[i] > T1;
        gt_b += front && myk[i] > T1;
        eq_b += front && myk[i] == T1;
    }
    uint32_t tot[3];
    block_sum3(n_gt, gt_b, eq_b, it & 1, tot);
    const uint32_t T16 = T1 - 1u;                       // back to the 16-bit key space (T1 >= 1: n_kept >= 1)
    const uint32_t n_take = (uint32_t)n_kept - tot[0];  // ties (key == T) to take, lowest positions first
    const uint32_t gt_before = tot[1], eq_before = tot[2];
    __syncthreads();
    // ---- 4. rank the slice (position order) and copy the kept rows ------------------------------------------------
    uint32_t taken_eq = min(eq_before, n_take);  // ties already granted to lower positions
    const uint32_t out_base = gt_before + taken_eq;
    uint32_t count = 0;                          // kept rows of this slice so far
    for (int c0 = 0; c0 < P; c0 += kClThreads) {
        const int r = c0 + tid;
        const bool valid = r < n_rows;
        const uint32_t key = valid ? my_keys[r] : 0u;
        const bool is_gt = valid && key > T16;
        const bool is_eq = valid && key == T16;
        const unsigned m_gt = __ballot_sync(0xFFFFFFFFu, is_gt);
        const unsigned m_eq = __ballot_sync(0xFFFFFFFFu, is_eq);
        if (lane == 0) {
            red[0][warp] = __popc(m_gt);
            red[1][warp] = __popc(m_eq);
        }
        __syncthreads();
        uint32_t gt_rank = __popc(m_gt & ((1u << lane) - 1u));
        uint32_t eq_rank = __popc(m_eq & ((1u << lane) - 1u));
        uint32_t tot_gt = 0, tot_eq = 0;
#pragma unroll
        for (int w = 0; w < 8; ++w) {
            gt_rank += (w < warp) ? red[0][w] : 0u;
            eq_rank += (w < warp) ? red[1][w] : 0u;
            tot_gt += red[0][w];
            tot_eq += red[1][w];
        }
        const uint32_t tie_room = n_take - taken_eq;  // ties this chunk may still take
        if (is_gt || (is_eq && eq_rank < tie_room)) list[count + gt_rank + min(eq_rank, tie_room)] = r;
        const uint32_t took = min(tot_eq, tie_room);
        count += tot_gt + took;
        taken_eq += took;
        __syncthreads();
    }
    if (count == 0) return;
    const int64_t out_row0 = (int64_t)row * n_kept + out_base;
    if (idx_out != nullptr)
        for (uint32_t i = tid; i < count; i += kClThreads) idx_out[out_row0 + i] = start + list[i];
    char* k_dst = K_out + out_row0 * (int64_t)row_bytes;
    char* v_dst = V_out + out_row0 * (int64_t)row_bytes;
    // kept rows leave shared memory as bulk stores, one per RUN of consecutive kept positions (the tiles are dense and
    // were written by the same async proxy): at 80 % density that is ~5 rows per store
    for (uint32_t r = tid; r < count; r += kClThreads) {
        const int pos = list[r];
        if (r > 0 && list[r - 1] == pos - 1) continue;  // not the head of a run
        uint32_t len = 1;
        while (r + len < count && list[r + len] == pos + (int)len) ++len;
        bulk_store_row(k_dst + (int64_t)r * row_bytes, ktile + (size_t)pos * pitch, len * row_bytes);
        if (v_smem) bulk_store_row(v_dst + (int64_t)r * row_bytes, vtile + (size_t)pos * pitch, len * row_bytes);
    }
    if (!v_smem) {  // V was not staged: kept rows through registers
        const char* v_src = reinterpret_cast<const char*>(V) + ((int64_t)b * vs.b + (int64_t)h * vs.h) * 2;
        const uint64_t pol_first = l2_policy_evict_first();
        const int total = (int)count * nvec;
        constexpr int UC = 8;
        for (int base = tid; base < total; base += kClThreads * UC) {
            int4 vv[UC];
#pragma unroll
            for (int u = 0; u < UC; ++u) {
                const int i = base + u * kClThreads;
                if (i < total) {
                    const int r = i / nvec, cc = i - r * nvec;
                    vv[u] = ldg_hint(v_src + (int64_t)(start + list[r]) * vs.s * 2 + cc * 16, pol_first);
                }
            }
#pragma unroll
            for (int u = 0; u < UC; ++u) {
                const int i = base + u * kClThreads;
                if (i < total) {
                    const int r = i / nvec, cc = i - r * nvec;
                    stg_hint(v_dst + (int64_t)r * row_bytes + cc * 16, vv[u], pol_first);
                }
            }
        }
    }
    bulk_store_wait();  // shared memory must stay valid until the bulk stores have read it
}

template <typename T, int KPT>
static cudaError_t launch_cluster_t(const Dims& d, const ClusterPlan& pl, const void* K, const void* V, void* K_out,
                                    void* V_out, int32_t* idx_out, void* scores_out, cudaStream_t st) {
    constexpr auto kern = knorm_cluster_kernel<T, KPT>;
    cudaError_t e = ensure_dynamic_smem<kern>(kClMaxSmem);
    if (e != cudaSuccess) return e;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(pl.C, d.R, 1);
    cfg.blockDim = dim3(kClThreads, 1, 1);
    cfg.dynamicSmemBytes = (size_t)pl.smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = pl.C;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<const T*>(K), static_cast<const T*>(V), d.ks, d.vs,
                              static_cast<char*>(K_out), static_cast<char*>(V_out), idx_out,
                              static_cast<uint16_t*>(scores_out), d.H, d.S, d.D, d.n_kept, pl.P, pl.v_smem);
}

static bool choose_cluster(const Dims& d, ClusterPlan* pl) {
    if (d.R > 65535) return false;
    int C = 8;  // the portable maximum cluster size
    // few positions per row: a smaller cluster keeps every CTA busy
    while (C > 1 && (d.S + C - 1) / C < 64) C >>= 1;
    *pl = cluster_plan(d, C);
    return pl->ok;
}

bool knorm_cluster_applicable(const Dims& d) {
    ClusterPlan pl;
    return choose_cluster(d, &pl);
}

// Returns cudaErrorNotSupported when the cache is too large for the cluster path (the caller takes the
// multi-kernel path instead).
cudaError_t launch_knorm_cluster(const Dims& d, int dtype, const void* K, const void* V, void* K_out, void* V_out,
                                 int32_t* idx_out, void* scores_out, cudaStream_t st) {
    ClusterPlan pl;
    if (!choose_cluster(d, &pl)) return cudaErrorNotSupported;
    return with_dtype(dtype, [&](auto t) {
        using T = decltype(t);
        if (d.S <= kClThreads * 12) return launch_cluster_t<T, 12>(d, pl, K, V, K_out, V_out, idx_out, scores_out, st);
        return launch_cluster_t<T, kClMaxKeysPerThread>(d, pl, K, V, K_out, V_out, idx_out, scores_out, st);
    });
}

}  // namespace kvp
