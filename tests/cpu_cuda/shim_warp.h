// Warp-collective instructions emulated on the host -- TEST INFRASTRUCTURE on top of shim.h (a block's threads are OS threads).
// Every warp of the running block has a 32-thread barrier; a collective publishes the calling lane's operand, meets the other
// 31 lanes at the barrier, computes its result from all 32 operands, and meets them again before the slot can be reused.
// All lanes of the warp must take part (the kernels built over this header only use full-warp masks).
//   __ballot_sync, __match_any_sync (32-bit), __reduce_or_sync, __shfl_down_sync (32-bit), __syncwarp
// plus the integer intrinsics __popc, __popcll, __clzll, __ffs, atomicAdd on 32-bit integers and __float_as_uint.
// The selection kernels (csrc/select_nms.cu) -- validated on the GPU -- run through the same emulation, which is what
// validates it.
#pragma once
#include "shim.h"

#include <atomic>
#include <bit>

constexpr int CPU_MAX_WARPS = 32;
struct CpuWarp {
  std::barrier<>* bar = nullptr;
  uint32_t addr[32];
  uint32_t a[32][4], b[32][2];
  uint32_t v[32];
};
static CpuWarp cpu_warps[CPU_MAX_WARPS];
static inline CpuWarp& cpu_my_warp() { return cpu_warps[threadIdx.x >> 5]; }
static inline void __syncwarp(unsigned = 0xffffffffu) { cpu_my_warp().bar->arrive_and_wait(); }

// publish this lane's 32-bit operand, run f(all 32 operands, lane) once every lane has published, return its result
template <typename F>
static inline uint32_t cpu_warp_collective(uint32_t mine, F f) {
  CpuWarp& w = cpu_my_warp();
  const int lane = threadIdx.x & 31;
  w.v[lane] = mine;
  w.bar->arrive_and_wait();
  const uint32_t r = f(w.v, lane);
  w.bar->arrive_and_wait();
  return r;
}

static inline unsigned __ballot_sync(unsigned, bool pred) {
  return cpu_warp_collective(pred ? 1u : 0u, [](const uint32_t* v, int) {
    unsigned m = 0u;
    for (int l = 0; l < 32; ++l) m |= (v[l] & 1u) << l;
    return m;
  });
}
static inline unsigned __match_any_sync(unsigned, unsigned value) {
  return cpu_warp_collective(value, [](const uint32_t* v, int lane) {
    unsigned m = 0u;
    for (int l = 0; l < 32; ++l) m |= (v[l] == v[lane] ? 1u : 0u) << l;
    return m;
  });
}
static inline unsigned __reduce_or_sync(unsigned, unsigned value) {
  return cpu_warp_collective(value, [](const uint32_t* v, int) {
    unsigned m = 0u;
    for (int l = 0; l < 32; ++l) m |= v[l];
    return m;
  });
}
// lanes whose source lane + delta is past the warp keep their own value
static inline unsigned __shfl_down_sync(unsigned, unsigned value, int delta) {
  return cpu_warp_collective(value, [delta](const uint32_t* v, int lane) { return lane + delta < 32 ? v[lane + delta] : v[lane]; });
}

static inline int __popc(unsigned x) { return std::popcount(x); }
static inline int __popcll(unsigned long long x) { return std::popcount(x); }
static inline int __clzll(long long x) { return x ? std::countl_zero((unsigned long long)x) : 64; }
static inline int __ffs(int x) { return x ? std::countr_zero((unsigned)x) + 1 : 0; }
static inline unsigned atomicAdd(unsigned* p, unsigned v) { return std::atomic_ref<unsigned>(*p).fetch_add(v); }
static inline int atomicAdd(int* p, int v) { return std::atomic_ref<int>(*p).fetch_add(v); }
static inline unsigned __float_as_uint(float f) { return std::bit_cast<unsigned>(f); }

// cpu_launch for kernels with warp collectives: per-warp barriers for the block that is running
static inline void cpu_launch_warps(dim3 grid, dim3 block, const std::function<void()>& body) {
  const unsigned nwarps = block.x / 32;
  std::vector<std::barrier<>*> bars;
  for (unsigned i = 0; i < nwarps; ++i) {
    bars.push_back(new std::barrier<>(32));
    cpu_warps[i].bar = bars.back();
  }
  cpu_launch(grid, block, body);
  for (auto* b : bars) delete b;
}
