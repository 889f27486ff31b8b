// Minimal CUDA-on-CPU execution model -- TEST INFRASTRUCTURE (tests/test_kernels_on_cpu.py).
//
// Lets g++ compile the SOURCE TEXT of simple libsmot kernels (no tensor-core / TMA / warp-shuffle instructions) and run it on
// the host: a block's threads are OS threads that meet at __syncthreads(), blocks run one after the other, dynamic shared
// memory is one static buffer.  The few helpers of csrc/common.cuh those kernels use are restated for the host (float only);
// IEEE division / square root stand in for the _rn intrinsics and the build uses -ffp-contract=off like nvcc's -fmad=false.
// This checks the kernels' logic (indexing, staging, ordering) against the oracle without a GPU; their GPU execution --
// including the fp16 instantiations -- is what the `-m gpu` tests check.
#pragma once
#include <algorithm>
#include <barrier>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <functional>
#include <thread>
#include <vector>

#ifdef SHIM_WITH_CUDA_FP16
// kernels that use __half / uint4: CUDA's own host-compilable vector and fp16 headers (plain g++ takes them)
#include <vector_types.h>
#include <vector_functions.h>
#include <cuda_fp16.h>
#undef __forceinline__
#undef __launch_bounds__
#undef __align__
#else
struct uint3 { unsigned x, y, z; };
struct dim3 { unsigned x, y, z; dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {} };
struct alignas(16) float4 { float x, y, z, w; };
struct alignas(16) int4 { int x, y, z, w; };
static inline float4 make_float4(float a, float b, float c, float d) { return float4{a, b, c, d}; }
#endif

static thread_local uint3 cpu_threadIdx, cpu_blockIdx;
static uint3 cpu_blockDim, cpu_gridDim;
static std::barrier<>* cpu_barrier = nullptr;
#define threadIdx cpu_threadIdx
#define blockIdx cpu_blockIdx
#define blockDim cpu_blockDim
#define gridDim cpu_gridDim

#ifndef SHIM_WITH_CUDA_FP16
#define __global__
#define __device__
#define __host__
#define __shared__
#endif
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __align__(n) alignas(n)
static inline void __syncthreads() { cpu_barrier->arrive_and_wait(); }
static inline float __fdiv_rn(float a, float b) { return a / b; }
static inline float __fsqrt_rn(float a) { return std::sqrt(a); }
static inline float __int_as_float(int v) { float f; std::memcpy(&f, &v, 4); return f; }
using std::max;
using std::min;

// dynamic shared memory of the block that is running (blocks are sequential): the H100 opt-in maximum per block
alignas(128) unsigned char cpu_dynamic_smem[227 * 1024];

namespace smot {
// csrc/common.cuh, host restatement of what the simple kernels use
inline void pdl_launch_dependents() {}
inline void pdl_wait() {}
inline float to_f(float v) { return v; }
template <typename T> inline T from_f(float v);
template <> inline float from_f<float>(float v) { return v; }
inline float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
inline void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
#ifdef SHIM_WITH_CUDA_FP16
inline float to_f(__half v) { return __half2float(v); }
template <> inline __half from_f<__half>(float v) { return __float2half_rn(v); }
inline float4 ld4(const __half* p) {
  uint2 r = *reinterpret_cast<const uint2*>(p);
  float2 a = __half22float2(*reinterpret_cast<__half2*>(&r.x));
  float2 b = __half22float2(*reinterpret_cast<__half2*>(&r.y));
  return make_float4(a.x, a.y, b.x, b.y);
}
inline void st4(__half* p, float4 v) {
  __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
  uint2 r;
  r.x = *reinterpret_cast<uint32_t*>(&a);
  r.y = *reinterpret_cast<uint32_t*>(&b);
  *reinterpret_cast<uint2*>(p) = r;
}
#endif
}  // namespace smot

// run `body` for every thread of every block
static inline void cpu_launch(dim3 grid, dim3 block, const std::function<void()>& body) {
  cpu_blockDim = uint3{block.x, block.y, block.z};
  cpu_gridDim = uint3{grid.x, grid.y, grid.z};
  const unsigned nthreads = block.x * block.y * block.z;
  for (unsigned bz = 0; bz < grid.z; ++bz)
    for (unsigned by = 0; by < grid.y; ++by)
      for (unsigned bx = 0; bx < grid.x; ++bx) {
        std::barrier<> bar((std::ptrdiff_t)nthreads);
        cpu_barrier = &bar;
        std::vector<std::thread> pool;
        pool.reserve(nthreads);
        for (unsigned t = 0; t < nthreads; ++t)
          pool.emplace_back([&, t] {
            cpu_threadIdx = uint3{t % block.x, (t / block.x) % block.y, t / (block.x * block.y)};
            cpu_blockIdx = uint3{bx, by, bz};
            body();
            bar.arrive_and_drop();   // a thread that returned early no longer takes part in later barriers
          });
        for (auto& th : pool) th.join();
      }
}
