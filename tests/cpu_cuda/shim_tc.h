// Warp-collective and asynchronous-copy instructions of the EMM correlation kernels, emulated on the host -- TEST
// INFRASTRUCTURE on top of shim.h (a block's threads are OS threads).  Emulated with their PTX semantics:
//   ldmatrix.sync.aligned.m8n8.x4.shared.b16      lanes 8i..8i+7 give the row addresses of matrix i; lane L receives, of every
//                                                 matrix, the 32-bit word (row L/4, halves 2(L%4), 2(L%4)+1)
//   mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32   fragment layout of the PTX ISA (g = L/4, t = L%4):
//                                                 a0 (g, 2t..) a1 (g+8, 2t..) a2 (g, 2t+8..) a3 (g+8, 2t+8..);
//                                                 b0 (k = 2t.., n = g) b1 (k = 2t+8.., n = g); c0 c1 (g, 2t 2t+1) c2 c3 (g+8, ..)
//   mbarrier.init / arrive.expect_tx / try_wait.parity, cp.async.bulk.shared.global with complete_tx (one phase)
// Shared-memory "addresses" are byte offsets into the shim's dynamic shared-memory buffer, as on the GPU.
// xcorr_mma_kernel -- validated on the GPU -- runs through the same emulation, which is what validates the emulation.
#pragma once
#define SHIM_WITH_CUDA_FP16
#include "shim_warp.h"

#include <cstdlib>

static inline uint32_t cpu_smem_offset(const void* p) { return (uint32_t)((const unsigned char*)p - cpu_dynamic_smem); }
#define __cvta_generic_to_shared(p) ((size_t)cpu_smem_offset(p))
static inline void __trap() { std::abort(); }

static inline float cpu_h2f(uint32_t word, int hi) {
  __half h;
  const uint16_t bits = (uint16_t)(hi ? (word >> 16) : (word & 0xffffu));
  std::memcpy(&h, &bits, 2);
  return __half2float(h);
}

namespace smot {

inline void xm_ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  CpuWarp& w = cpu_my_warp();
  const int lane = threadIdx.x & 31;
  w.addr[lane] = addr;
  w.bar->arrive_and_wait();
  uint32_t r[4];
  for (int i = 0; i < 4; ++i)
    std::memcpy(&r[i], cpu_dynamic_smem + w.addr[i * 8 + (lane >> 2)] + (lane & 3) * 4, 4);
  w.bar->arrive_and_wait();
  r0 = r[0], r1 = r[1], r2 = r[2], r3 = r[3];
}

// ldmatrix .x2: lanes 0..7 / 8..15 give the row addresses of matrices 0 / 1 (the other lanes' addresses are ignored)
inline void xm_ldmatrix_x2(uint32_t addr, uint32_t& r0, uint32_t& r1) {
  CpuWarp& w = cpu_my_warp();
  const int lane = threadIdx.x & 31;
  w.addr[lane] = addr;
  w.bar->arrive_and_wait();
  uint32_t r[2];
  for (int i = 0; i < 2; ++i)
    std::memcpy(&r[i], cpu_dynamic_smem + w.addr[i * 8 + (lane >> 2)] + (lane & 3) * 4, 4);
  w.bar->arrive_and_wait();
  r0 = r[0], r1 = r[1];
}

// mma.m16n8k8: a0 (g, 2t..) a1 (g+8, 2t..); b0 (k = 2t.., n = g); c as for k16
inline void xm_mma_k8(float* c, uint32_t a0, uint32_t a1, uint32_t b0) {
  CpuWarp& w = cpu_my_warp();
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  w.a[lane][0] = a0, w.a[lane][1] = a1, w.b[lane][0] = b0;
  w.bar->arrive_and_wait();
  auto A = [&](int r, int k) { return cpu_h2f(w.a[(r & 7) * 4 + (k >> 1)][r >= 8 ? 1 : 0], k & 1); };
  auto B = [&](int k, int n) { return cpu_h2f(w.b[n * 4 + (k >> 1)][0], k & 1); };
  float d[4];
  for (int e = 0; e < 4; ++e) {
    const int r = g + (e >= 2 ? 8 : 0), n = 2 * t + (e & 1);
    float acc = c[e];
    for (int k = 0; k < 8; ++k) acc += A(r, k) * B(k, n);
    d[e] = acc;
  }
  w.bar->arrive_and_wait();
  for (int e = 0; e < 4; ++e) c[e] = d[e];
}

inline void xm_mma(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  CpuWarp& w = cpu_my_warp();
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  for (int i = 0; i < 4; ++i) w.a[lane][i] = a[i];
  w.b[lane][0] = b0, w.b[lane][1] = b1;
  w.bar->arrive_and_wait();
  auto A = [&](int r, int k) { return cpu_h2f(w.a[(r & 7) * 4 + ((k & 7) >> 1)][(r >= 8 ? 1 : 0) + (k >= 8 ? 2 : 0)], k & 1); };
  auto B = [&](int k, int n) { return cpu_h2f(w.b[n * 4 + ((k & 7) >> 1)][k >= 8 ? 1 : 0], k & 1); };
  float d[4];
  for (int e = 0; e < 4; ++e) {
    const int r = g + (e >= 2 ? 8 : 0), n = 2 * t + (e & 1);
    float acc = c[e];
    for (int k = 0; k < 16; ++k) acc += A(r, k) * B(k, n);
    d[e] = acc;
  }
  w.bar->arrive_and_wait();
  for (int e = 0; e < 4; ++e) c[e] = d[e];
}

// mbarriers (one phase each), keyed by their shared-memory address: `pending` transaction bytes after the arming arrive
struct CpuMbar { std::atomic<long> pending{0}; std::atomic<int> armed{0}; };
static CpuMbar cpu_mbars[64];
static inline CpuMbar& cpu_mbar(uint32_t bar) { return cpu_mbars[(bar >> 3) & 63u]; }
inline void xp_mbar_init(uint32_t bar, uint32_t) { cpu_mbar(bar).pending = 0, cpu_mbar(bar).armed = 0; }
inline void xp_mbar_expect_tx(uint32_t bar, uint32_t bytes) { cpu_mbar(bar).pending += (long)bytes, cpu_mbar(bar).armed = 1; }
inline bool xp_mbar_try_wait(uint32_t bar, uint32_t) { return cpu_mbar(bar).armed.load() == 1 && cpu_mbar(bar).pending.load() == 0; }
inline void xp_bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  if ((dst & 15u) || ((uintptr_t)src & 15u) || (bytes & 15u)) { std::fprintf(stderr, "cp.async.bulk: misaligned operand\n"); std::abort(); }
  if (bar & 7u) { std::fprintf(stderr, "mbarrier: misaligned\n"); std::abort(); }
  std::memcpy(cpu_dynamic_smem + dst, src, bytes);
  cpu_mbar(bar).pending -= (long)bytes;
}

}  // namespace smot
