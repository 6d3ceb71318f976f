// vtp_b200 — host helpers: error buffer, device query, TMA tensor-map encoding via the driver entry point
// (resolved at run time with cudaGetDriverEntryPoint so the library has no link-time dependency on libcuda).
#include "host.h"

namespace vtp {

char* err_buf() {
    static thread_local char buf[512] = {0};
    return buf;
}

int num_sms() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 132;
    }
    return n;
}

typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                        const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                        CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_tmapEncodeTiled get_encode_fn() {
    static PFN_tmapEncodeTiled fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_tmapEncodeTiled>(p);
    }
    return fn;
}

int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box) {
    return make_tmap(out, base, VTP_BF16, rank, dims, strides_bytes, box);
}

int make_tmap(CUtensorMap* out, const void* base, int dtype, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
              const uint32_t* box) {
    PFN_tmapEncodeTiled fn = get_encode_fn();
    if (!fn) VTP_FAIL(VTP_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
    cuuint64_t gdim[5];
    cuuint64_t gstr[4];
    cuuint32_t bx[5], es[5];
    for (int i = 0; i < rank; ++i) gdim[i] = dims[i], bx[i] = box[i], es[i] = 1;
    for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
    CUresult r = fn(out, dtype == VTP_F32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
        VTP_FAIL(VTP_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d): rank=%d dims=[%llu,%llu] stride0=%llu box=[%u,%u]",
                 (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
                 (unsigned long long)(rank > 1 ? strides_bytes[0] : 0), box[0], rank > 1 ? box[1] : 0);
    return VTP_OK;
}

}  // namespace vtp

extern "C" const char* vtp_last_error(void) { return vtp::err_buf(); }
extern "C" int vtp_version(void) { return 100; }
extern "C" int vtp_check_device(void) {
    int dev = 0;
    cudaDeviceProp prop;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess)
        VTP_FAIL(VTP_ERR_CUDA, "no CUDA device");
    if (prop.major != 9 || prop.minor != 0)
        VTP_FAIL(VTP_ERR_ARCH, "device is sm_%d%d, this library is sm_90a only", prop.major, prop.minor);
    return VTP_OK;
}
