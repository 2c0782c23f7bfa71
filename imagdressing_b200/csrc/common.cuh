// Host-side helpers shared by the C-ABI translation units: error recording, TMA descriptor encoding.
#pragma once
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cuda.h>
#include <atomic>

#include <cuda_runtime.h>

#include "../../include/imagd_b200.h"

namespace imagd {

constexpr int kNumSms = 132;  // H100 SXM: grid caps of the grid-stride / chunked kernels

void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);

#define IMAGD_CHECK_ARG(cond, ...)     \
    do {                               \
        if (!(cond)) {                 \
            ::imagd::set_error(__VA_ARGS__); \
            return IMAGD_ERR_ARG;      \
        }                              \
    } while (0)

#define IMAGD_CUDA(call)                                   \
    do {                                                   \
        cudaError_t e__ = (call);                          \
        if (e__ != cudaSuccess) return ::imagd::cuda_fail(e__, #call); \
    } while (0)

// Opt a kernel into more than 48 KB of dynamic shared memory, once per device (the attribute lives in the device's
// context; one process may drive several GPUs) and safely from several host threads.
#define IMAGD_SET_MAX_SMEM(kernel, bytes)                                                               \
    do {                                                                                                \
        static std::atomic<bool> done__[16];                                                            \
        int dev__ = 0;                                                                                  \
        IMAGD_CUDA(cudaGetDevice(&dev__));                                                              \
        if (dev__ < 0 || dev__ >= 16 || !done__[dev__].load(std::memory_order_acquire)) {               \
            IMAGD_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes)); \
            if (dev__ >= 0 && dev__ < 16) done__[dev__].store(true, std::memory_order_release);         \
        }                                                                                               \
    } while (0)

#define IMAGD_LAUNCH_CHECK(name)                               \
    do {                                                       \
        cudaError_t e__ = cudaGetLastError();                  \
        if (e__ != cudaSuccess) return ::imagd::cuda_fail(e__, name);  \
    } while (0)

// Encode a tiled bf16 TMA descriptor (SWIZZLE_128B, OOB zero fill). dims/strides innermost first;
// strides_bytes has rank-1 entries (stride of dim 1..rank-1). Returns IMAGD_OK or an error code.
int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box);

// Launch, optionally with the programmatic-dependent-launch attribute (IMAGD_PDL=1 in the environment enables it).
bool pdl_enabled();
int pdl_mode();  // 0 off, 1 early trigger, 2 late trigger (api.cu)
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              Args... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace imagd
