// Library-level entry points of the C ABI: version, error string, device check, TMA descriptor encoding.
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "common.cuh"

namespace imagd {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

// IMAGD_PDL: 0 (default) no programmatic dependent launch; 1 every kernel lets its dependent start at once (the
// dependent's CTAs can take shared memory the running kernel still needs);
// 2 "late trigger": the tensor-core kernels release their dependent only when their own mainloop is done, so the next
// kernel's launch latency and prologue hide under this kernel's epilogue / tail instead of competing with its mainloop.
int pdl_mode() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("IMAGD_PDL");
        v = (e && e[0] >= '0' && e[0] <= '2') ? e[0] - '0' : 0;
    }
    return v;
}
bool pdl_enabled() { return pdl_mode() != 0; }

int cuda_fail(cudaError_t e, const char* what) {
    set_error("CUDA error %d (%s) at %s", static_cast<int>(e), cudaGetErrorString(e), what);
    return IMAGD_ERR_CUDA;
}

// cuTensorMapEncodeTiled is resolved through the runtime so the library carries no link-time dependency on
// libcuda.so (it must load — symbols only — on a CPU-only build box).
typedef CUresult (*encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static encode_tiled_fn g_encode = nullptr;
static std::once_flag g_encode_once;

static void resolve_encode() {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q);
    if (e == cudaSuccess && q == cudaDriverEntryPointSuccess) g_encode = reinterpret_cast<encode_tiled_fn>(fn);
}

int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box) {
    std::call_once(g_encode_once, resolve_encode);
    if (!g_encode) {
        set_error("cuTensorMapEncodeTiled not available (no CUDA driver?)");
        return IMAGD_ERR_CUDA;
    }
    cuuint64_t gdim[5];
    cuuint64_t gstr[4];
    cuuint32_t bdim[5];
    cuuint32_t estr[5];
    for (int i = 0; i < rank; ++i) {
        gdim[i] = dims[i];
        bdim[i] = box[i];
        estr[i] = 1;
        if (i > 0) {
            gstr[i - 1] = strides_bytes[i - 1];
            if (gstr[i - 1] % 16 != 0) {
                set_error("TMA stride %d = %llu bytes is not a multiple of 16", i,
                          static_cast<unsigned long long>(gstr[i - 1]));
                return IMAGD_ERR_ARG;
            }
        }
    }
    if (!aligned16(base)) {
        set_error("TMA base pointer %p is not 16-byte aligned", base);
        return IMAGD_ERR_ARG;
    }
    CUresult r = g_encode(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, static_cast<cuuint32_t>(rank),
                          const_cast<void*>(base), gdim, gstr, bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed: CUresult %d (rank %d dims %llu,%llu,%llu,%llu box %u,%u,%u,%u)",
                  static_cast<int>(r), rank, (unsigned long long)gdim[0], (unsigned long long)(rank > 1 ? gdim[1] : 0),
                  (unsigned long long)(rank > 2 ? gdim[2] : 0), (unsigned long long)(rank > 3 ? gdim[3] : 0), bdim[0],
                  rank > 1 ? bdim[1] : 0, rank > 2 ? bdim[2] : 0, rank > 3 ? bdim[3] : 0);
        return IMAGD_ERR_CUDA;
    }
    return IMAGD_OK;
}

}  // namespace imagd

extern "C" {

int imagd_version(void) { return 100; /* 0.1.0 */ }

const char* imagd_last_error(void) { return imagd::g_err; }

int imagd_device_check(void) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return imagd::cuda_fail(e, "cudaGetDevice");
    cudaDeviceProp p;
    e = cudaGetDeviceProperties(&p, dev);
    if (e != cudaSuccess) return imagd::cuda_fail(e, "cudaGetDeviceProperties");
    if (p.major != 9 || p.minor != 0) {
        imagd::set_error("device %s is sm_%d%d; this library is built for sm_90a only", p.name, p.major, p.minor);
        return IMAGD_ERR_ARCH;
    }
    return p.major * 10 + p.minor;
}

}  // extern "C"
