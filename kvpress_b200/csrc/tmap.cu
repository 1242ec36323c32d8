// tmap.cu — host-side helpers: cached device properties and TMA tensor-map encoding. The driver symbol cuTensorMapEncodeTiled is fetched
// through cudaGetDriverEntryPoint so the library has no link-time dependency on libcuda.
#include "common.cuh"
#include "umma.cuh"

namespace kvp {

// SM count of the current device, cached per device index (heterogeneous / MIG hosts size their
// persistent grids per device).
int device_sm_count() {
    static int cache[kMaxDevices] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) dev = 0;
    if (cache[dev] == 0) {
        int n = 0;
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        cache[dev] = n > 0 ? n : 132;
    }
    return cache[dev];
}

kvp_encode_tiled_fn get_encode_tiled() {
    static kvp_encode_tiled_fn fn = nullptr;  // immutable once resolved
    if (fn == nullptr) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) ==
                cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<kvp_encode_tiled_fn>(p);
    }
    return fn;
}

cudaError_t make_tmap_16bit(CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                            const uint64_t* strides_bytes, const uint32_t* box) {
    kvp_encode_tiled_fn enc = get_encode_tiled();
    if (enc == nullptr) return cudaErrorNotSupported;
    cuuint64_t gdim[5];
    cuuint64_t gstr[5];
    cuuint32_t bdim[5], estr[5];
    for (int i = 0; i < rank; ++i) {
        gdim[i] = dims[i];
        bdim[i] = box[i];
        estr[i] = 1;
        if (i > 0) gstr[i - 1] = strides_bytes[i];
    }
    const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank,
                           const_cast<void*>(base), gdim, gstr, bdim, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

cudaError_t make_tmap_cache(CUtensorMap* map, const void* base, const Dims& d, const Strides3& s, uint32_t box_rows) {
    const uint64_t row_b = (uint64_t)s.s * 2;
    const uint64_t h_b = d.H > 1 ? (uint64_t)s.h * 2 : row_b * (uint64_t)d.S;
    const uint64_t b_b = d.B > 1 ? (uint64_t)s.b * 2 : h_b * (uint64_t)d.H;
    const uint64_t dims[4] = {(uint64_t)d.D, (uint64_t)d.S, (uint64_t)d.H, (uint64_t)d.B};
    const uint64_t str[4] = {0, row_b, h_b, b_b};
    const uint32_t box[4] = {64, box_rows, 1, 1};
    return make_tmap_16bit(map, base, 4, dims, str, box);
}

cudaError_t make_tmap_rows(CUtensorMap* map, const void* base, uint64_t cols, uint64_t rows, uint64_t row_stride,
                           uint64_t heads, uint64_t head_stride, uint32_t box_rows) {
    const uint64_t dims[3] = {cols, rows, heads};
    const uint64_t str[3] = {0, row_stride * 2, head_stride * 2};
    const uint32_t box[3] = {64, box_rows, 1};
    return make_tmap_16bit(map, base, 3, dims, str, box);
}

}  // namespace kvp
