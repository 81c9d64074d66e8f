// Error reporting, device queries and tensor-map encoding shared by all entry points.
#include "tc_common.cuh"
#include <stdarg.h>
#include <mutex>
#include <unordered_map>

namespace gsb {

static thread_local char g_err[512] = "";

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int num_sms() {
    static int sms = 0;
    if (sms == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess ||
            cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0)
            sms = 132;
    }
    return sms;
}

int raise_dyn_smem(const void *kernel, size_t bytes) {
    static std::mutex mu;
    static std::unordered_map<const void *, size_t> largest;
    std::lock_guard<std::mutex> lock(mu);
    size_t &set = largest[kernel];
    if (bytes > set) {
        GSB_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
        set = bytes;
    }
    return GSB_OK;
}

// cuTensorMapEncodeTiled through the runtime's driver entry point, so that the library does not link libcuda
typedef CUresult (*TcEncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                    const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static TcEncodeTiledFn tc_encode_fn() {
    static TcEncodeTiledFn fn = nullptr;
    if (!fn) {
        void *ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<TcEncodeTiledFn>(ptr);
    }
    return fn;
}

int tc_make_tmap(CUtensorMap *map, CUtensorMapDataType type, const void *base, int rank, const uint64_t *dims,
                 const uint64_t *strides_bytes, const uint32_t *box) {
    TcEncodeTiledFn enc = tc_encode_fn();
    if (!enc) { set_error("cuTensorMapEncodeTiled entry point not available"); return GSB_ERR_CUDA; }
    cuuint64_t gdim[5], gstride[4];
    cuuint32_t bx[5], estr[5];
    for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; bx[i] = box[i]; estr[i] = 1; }
    for (int i = 0; i + 1 < rank; ++i) gstride[i] = strides_bytes[i];
    CUresult r = enc(map, type, (cuuint32_t)rank, const_cast<void *>(base), gdim, gstride, bx, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d)", (int)r); return GSB_ERR_CUDA; }
    return GSB_OK;
}

}  // namespace gsb

extern "C" int gsb_abi_version(void) { return GSB_ABI_VERSION; }
extern "C" const char *gsb_last_error(void) { return gsb::g_err; }
