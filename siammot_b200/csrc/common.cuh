// Shared helpers for the SiamMOT kernels (sm_90a, H100).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/smot.h"

namespace smot {

void set_error(const char* fmt, ...);

#define SMOT_CHECK_ARG(cond, ...)                 \
  do {                                            \
    if (!(cond)) {                                \
      ::smot::set_error(__VA_ARGS__);             \
      return SMOT_ERR_INVALID;                    \
    }                                             \
  } while (0)

#define SMOT_CHECK_LAUNCH(name)                                              \
  do {                                                                       \
    cudaError_t e__ = cudaGetLastError();                                    \
    if (e__ != cudaSuccess) {                                                \
      ::smot::set_error("%s: launch failed: %s", name, cudaGetErrorString(e__)); \
      return SMOT_ERR_CUDA;                                                  \
    }                                                                        \
  } while (0)

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// Opt `kernel` into `bytes` of dynamic shared memory.  The attribute is per device and a process may drive several
// GPUs, so the largest grant is remembered per device (one static table per call site = per kernel instance).
constexpr int SMOT_MAX_DEVICES = 64;
#define SMOT_ENSURE_SMEM(kernel, bytes, what)                                                                            \
  do {                                                                                                                   \
    static int granted__[::smot::SMOT_MAX_DEVICES];                                                                      \
    int dev__ = 0;                                                                                                       \
    cudaGetDevice(&dev__);                                                                                               \
    const int want__ = (int)(bytes);                                                                                     \
    if (dev__ >= 0 && dev__ < ::smot::SMOT_MAX_DEVICES && want__ > 48 * 1024 && granted__[dev__] < want__) {             \
      cudaError_t e__ = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, want__);               \
      if (e__ != cudaSuccess) {                                                                                          \
        ::smot::set_error("%s: cudaFuncSetAttribute(%d bytes): %s", what, want__, cudaGetErrorString(e__));              \
        return SMOT_ERR_CUDA;                                                                                            \
      }                                                                                                                  \
      granted__[dev__] = want__;                                                                                         \
    }                                                                                                                    \
  } while (0)

// ---- programmatic dependent launch (PDL) ---------------------------------------------------
// The detection stage is ~110 short kernels in one CUDA graph; at 5-15 us each, the drain -> launch -> prologue
// gap between consecutive kernels is a large share of the frame.  Kernels launched through launch_pdl() may begin
// while their predecessor in the stream is still running: they do everything that does not touch the predecessor's
// data first (barrier init, staging constant weights), then pdl_wait() blocks until the predecessor
// has completed and its writes are visible.  pdl_launch_dependents() at the top lets the NEXT kernel start the same
// way once every CTA of this grid is running.  Both are no-ops for kernels launched the ordinary way.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

bool pdl_enabled();  // capi.cu: on unless SMOT_PDL=0
int sm_count();      // capi.cu: multiprocessors of the current device (cached per device)

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid, cfg.blockDim = block, cfg.dynamicSmemBytes = smem, cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  cfg.attrs = attr, cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// ---- storage-type <-> float -------------------------------------------------------------
__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }

// load 4 consecutive elements as floats (16B for f32, 8B for f16); pointer must be aligned
__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 ld4(const __half* p) {
  uint2 r = *reinterpret_cast<const uint2*>(p);
  float2 a = __half22float2(*reinterpret_cast<__half2*>(&r.x));
  float2 b = __half22float2(*reinterpret_cast<__half2*>(&r.y));
  return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ void st4(__half* p, float4 v) {
  __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
  uint2 r;
  r.x = *reinterpret_cast<uint32_t*>(&a);
  r.y = *reinterpret_cast<uint32_t*>(&b);
  *reinterpret_cast<uint2*>(p) = r;
}

// monotone float -> uint32 key (larger float => larger key); -0 and +0 get the same key (they compare equal, so the index
// decides their order), NaN sorts high
__device__ __forceinline__ uint32_t float_key(float f) {
  uint32_t u = f == 0.f ? 0u : __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// IoU with the legacy "+1" pixel convention (maskrcnn_benchmark csrc/cuda/nms.cu devIoU)
__device__ __forceinline__ float iou_plus1(const float4 a, const float4 b) {
  float left = fmaxf(a.x, b.x), right = fminf(a.z, b.z);
  float top = fmaxf(a.y, b.y), bottom = fminf(a.w, b.w);
  float width = fmaxf(right - left + 1.f, 0.f), height = fmaxf(bottom - top + 1.f, 0.f);
  float inter = width * height;
  float sa = (a.z - a.x + 1.f) * (a.w - a.y + 1.f);
  float sb = (b.z - b.x + 1.f) * (b.w - b.y + 1.f);
  return inter / (sa + sb - inter);
}

}  // namespace smot
