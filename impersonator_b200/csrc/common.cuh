// Shared helpers for the lwb_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/lwb_b200.h"

namespace lwb {

void set_error(const char* fmt, ...);

#define LWB_CHECK_ARG(cond, msg)                                                   \
    do { if (!(cond)) { lwb::set_error("%s: %s", __func__, msg); return LWB_E_INVALID; } } while (0)

#define LWB_CUDA_OK(expr)                                                          \
    do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) {                       \
        lwb::set_error("%s: %s -> %s", __func__, #expr, cudaGetErrorString(e__));  \
        return LWB_E_CUDA; } } while (0)

#define LWB_LAUNCH_OK()                                                            \
    do { cudaError_t e__ = cudaGetLastError(); if (e__ != cudaSuccess) {           \
        lwb::set_error("%s: launch failed -> %s", __func__, cudaGetErrorString(e__)); \
        return LWB_E_CUDA; } } while (0)

static inline int ceil_div(long a, long b) { return (int)((a + b - 1) / b); }

int sm_count();                      // of the current device
constexpr int kMaxDevices = 64;
int device_slot();                   // current device ordinal (clamped to kMaxDevices - 1): index of per-device caches

// Programmatic dependent launch (LWB_PDL, default on): kernels launched through launch_pdl may be scheduled while the
// previous kernel of the stream drains; each of them executes pdl_wait() before its first global-memory access and
// pdl_trigger() to let its own successor do the same.  Both are no-ops for a kernel launched the plain way.
bool pdl_enabled();
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args)
{
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// One full 32-byte sector per lane: two adjacent 16-byte accesses (sm_90 has no 256-bit load / store).  Addresses must be
// 32-byte aligned.
__device__ __forceinline__ void ldg_f32x8(const float* p, float* v) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void stg_f32x8(float* p, const float* v) {
    reinterpret_cast<float4*>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
    reinterpret_cast<float4*>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
}

}  // namespace lwb
