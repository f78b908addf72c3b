// Shared helpers for libwts (sm_90a only).
#pragma once
#include <stdlib.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/wts.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libwts is written for sm_90a (H100) only"
#endif

namespace wts {

void set_error(const char* fmt, ...);

#define WTS_CUDA_CHECK(expr)                                                              \
    do {                                                                                  \
        cudaError_t _e = (expr);                                                          \
        if (_e != cudaSuccess) {                                                          \
            ::wts::set_error("%s failed at %s:%d: %s", #expr, __FILE__, __LINE__,         \
                             cudaGetErrorString(_e));                                     \
            return -1;                                                                    \
        }                                                                                 \
    } while (0)

#define WTS_LAUNCH_CHECK()                                                                \
    do {                                                                                  \
        cudaError_t _e = cudaGetLastError();                                              \
        if (_e != cudaSuccess) {                                                          \
            ::wts::set_error("kernel launch failed at %s:%d: %s", __FILE__, __LINE__,     \
                             cudaGetErrorString(_e));                                     \
            return -1;                                                                    \
        }                                                                                 \
    } while (0)

constexpr unsigned FULL_MASK = 0xffffffffu;

// row pitch (elements) of a segment's cost matrix (WtsSegDesc.flags bit 1: rows padded to 16 bytes of float32)
__host__ __device__ inline int seg_pitch(const WtsSegDesc& sd) { return (sd.flags & WTS_SEG_PITCH16) ? ((sd.F + 3) & ~3) : sd.F; }

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(FULL_MASK, v, o));
    return v;
}
__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(FULL_MASK, v, o));
    return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL_MASK, v, o);
    return v;
}


// ---- programmatic dependent launch (PDL).  Decode-step kernels are launched with the programmatic-stream-
// serialization attribute: a kernel calls pdl_launch() at its top (lets the NEXT kernel's CTAs become resident and
// run their prologue) and pdl_wait() before it touches global memory (blocks until the PREVIOUS kernel has
// completed and flushed).  Every CTA must pass pdl_wait() before it exits, so completion stays transitive.
// Without the launch attribute both instructions are no-ops.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

inline bool pdl_enabled()
{
    static const bool on = [] { const char* e = getenv("WTS_PDL"); return e ? atoi(e) != 0 : true; }();
    return on;
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args)
{
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace wts
