// knorm.cu — stage S for KnormPress and for caller-supplied scores.
//
// Reference semantics (kvpress/presses/knorm_press.py:38): scores = -keys.norm(dim=-1)
//   = -sqrt(sum_d k_d^2), accumulated in fp32, rounded ONCE to the K dtype.
// One CTA scores one tile of kTile positions of one (b, h) row with 128-bit loads
// (a sub-warp of LPR lanes per 2*D-byte row, U independent loads in flight per lane), stages
// the 16-bit ordered keys in shared memory, writes them coalesced and adds the tile's
// histogram of (key >> 8) to the row histogram the select stage starts from.
#include "common.cuh"
#include "knorm_chunk.cuh"

namespace kvp {

template <typename T, int LPR>
__global__ void __launch_bounds__(kTileThreads)
knorm_score_kernel(const T* __restrict__ K, Strides3 ks, int H, int S, int D, Workspace ws,
                   uint16_t* __restrict__ scores_out, int want_keys) {
    __shared__ uint16_t skeys[kScoreChunk];
    __shared__ uint16_t sscores[kScoreChunk];
    __shared__ uint32_t shist[256];
    const int chunk = blockIdx.x, row = blockIdx.y, tid = threadIdx.x;
    shist[tid] = 0;  // kTileThreads == 256
    pdl_launch_dependents();  // the select+compact kernel behind this one may start to take residency
    knorm_score_chunk<T, LPR>(K, ks, row / H, row % H, chunk, S, D, skeys, sscores);
    __syncthreads();
    flush_or_store_scores(skeys, sscores, shist, row, chunk * kScoreChunk, S, ws, scores_out, want_keys);
}

template <typename T>
static cudaError_t launch_knorm_t(const Dims& d, const void* K, const Workspace& ws,
                                  void* scores_out, bool want_keys, cudaStream_t st) {
    dim3 grid((d.S + kScoreChunk - 1) / kScoreChunk, d.R);
    const T* Kp = static_cast<const T*>(K);
    uint16_t* so = static_cast<uint16_t*>(scores_out);
    with_lanes_per_row(d.D, [&](auto lpr) {
        knorm_score_kernel<T, lpr><<<grid, kTileThreads, 0, st>>>(Kp, d.ks, d.H, d.S, d.D, ws, so, want_keys ? 1 : 0);
    });
    return cudaPeekAtLastError();
}

cudaError_t launch_knorm_score(const Dims& d, int dtype, const void* K, const Workspace& ws,
                               void* scores_out, bool want_keys, cudaStream_t st) {
    return with_dtype(dtype, [&](auto t) {
        return launch_knorm_t<decltype(t)>(d, K, ws, scores_out, want_keys, st);
    });
}

// ---- caller-supplied scores -> keys + histogram ------------------------------------------------
__global__ void __launch_bounds__(kTileThreads)
keys_from_scores_kernel(const uint16_t* __restrict__ scores, int64_t sb, int64_t sh, int H, int S,
                        uint16_t inf_bits, Workspace ws) {
    __shared__ uint16_t skeys[kTile];
    __shared__ uint32_t shist[256];
    const int tile = blockIdx.x, row = blockIdx.y, tid = threadIdx.x;
    const int b = row / H, h = row % H;
    shist[tid] = 0;
    pdl_launch_dependents();  // the select+compact kernel behind this one may start to take residency
    const uint16_t* src = scores + (int64_t)b * sb + (int64_t)h * sh;
    const int s = tile * kTile + tid;
    skeys[tid] = (s < S) ? ordered_key16(src[s], inf_bits) : (uint16_t)0;
    __syncthreads();
    flush_chunk_keys<1>(skeys, nullptr, shist, row, tile * kTile, S, ws, nullptr);
}

cudaError_t launch_keys_from_scores(const Dims& d, int dtype, const void* scores, int64_t sb, int64_t sh,
                                    const Workspace& ws, cudaStream_t st) {
    const int n_tiles = (d.S + kTile - 1) / kTile;
    dim3 grid(n_tiles, d.R);
    const uint16_t inf_bits = with_dtype(dtype, [](auto t) { return F16Traits<decltype(t)>::kInfBits; });
    keys_from_scores_kernel<<<grid, kTileThreads, 0, st>>>(static_cast<const uint16_t*>(scores), sb, sh, d.H, d.S,
                                                           inf_bits, ws);
    return cudaPeekAtLastError();
}

}  // namespace kvp
