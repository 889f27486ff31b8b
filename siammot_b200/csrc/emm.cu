// EMM tracker kernels: depthwise cross-correlation and the fused upsample+decode.
//
// smot_xcorr  (xcorr.py:37-45).  NHWC: a lane owns one channel, so every shared/global access of a
//   warp is a contiguous run of channels.  Per (track, 32-channel group) the S*S search window and
//   the T*T template are staged once in shared memory; each warp then produces output rows with a
//   register-blocked row convolution (for each template row u: S window values + T taps in
//   registers -> O*T FMAs), i.e. ~5 FMAs per shared-memory load, so the kernel is bound by the
//   FP32 FMA pipe, not by shared memory or HBM (see DESIGN.md for the roofline).
//
// smot_emm_decode  (track_core.py:69-76,101-135,184-225).  The reference materialises seven
//   bicubic x16 maps (55 MB at 30 tracks) and runs ~15 elementwise / reduction kernels over them.
//   Here nothing is materialised: a CTA upsamples its slice separably (horizontal pass into shared
//   memory, vertical pass in registers), evaluates the penalised score per pixel and keeps only the
//   arg-max (packed 64-bit atomicMax: score bits << 32 | ~index, so ties resolve to the first index
//   like torch.argmax).
#include <stdlib.h>

#include "common.cuh"

namespace smot {

// =============================================================================================
// xcorr
// =============================================================================================
// Staging keeps the search window in its storage type (fp16 windows cost half the shared memory, so three
// CTAs fit per SM) and the template in fp32.  grid = (C/32, tracks, 2): blockIdx.z selects output rows
// [8z, 8z+8) -> a CTA stages only the O/2 + T - 1 window rows it needs; warp w owns output row 8z + w.
template <typename T, int S, int TT>
__global__ void __launch_bounds__(256) xcorr_kernel(const T* __restrict__ x, const T* __restrict__ k, T* __restrict__ out,
                                                    int C) {
  constexpr int O = S - TT + 1;
  constexpr int CG = 32;
  constexpr int RH = O / 2;            // output rows per CTA
  constexpr int XR = RH + TT - 1;      // window rows per CTA
  static_assert(O % 2 == 0 && RH <= 8, "row split assumes <= 8 rows per CTA (one per warp)");
  extern __shared__ __align__(16) unsigned char xc_raw[];
  T* xs = reinterpret_cast<T*>(xc_raw);                                           // [XR*S][CG]
  float* ks = reinterpret_cast<float*>(xc_raw + ((XR * S * CG * sizeof(T) + 15) / 16) * 16);  // [TT*TT][CG]
  const int n = blockIdx.y, c0 = blockIdx.x * CG, r0 = blockIdx.z * RH;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const T* xb = x + ((size_t)n * S * S + (size_t)r0 * S) * C + c0;
  const T* kb = k + (size_t)n * TT * TT * C + c0;
  constexpr int VEC = 16 / sizeof(T);  // elements per 16-byte chunk
  for (int i = threadIdx.x; i < XR * S * (CG / VEC); i += blockDim.x) {
    const int pos = i / (CG / VEC), q = (i % (CG / VEC)) * VEC;
    *reinterpret_cast<uint4*>(xs + pos * CG + q) = *reinterpret_cast<const uint4*>(xb + (size_t)pos * C + q);
  }
  for (int i = threadIdx.x; i < TT * TT * (CG / 4); i += blockDim.x) {
    const int pos = i / (CG / 4), q = (i % (CG / 4)) * 4;
    *reinterpret_cast<float4*>(ks + pos * CG + q) = ld4(kb + (size_t)pos * C + q);
  }
  __syncthreads();
  if (warp >= RH) return;
  const int i = warp;  // local output row
  float acc[O];
#pragma unroll
  for (int j = 0; j < O; ++j) acc[j] = 0.f;
  for (int u = 0; u < TT; ++u) {
    float xr[S], kr[TT];
#pragma unroll
    for (int j = 0; j < S; ++j) xr[j] = to_f(xs[((i + u) * S + j) * CG + lane]);
#pragma unroll
    for (int v = 0; v < TT; ++v) kr[v] = ks[(u * TT + v) * CG + lane];
#pragma unroll
    for (int v = 0; v < TT; ++v)
#pragma unroll
      for (int j = 0; j < O; ++j) acc[j] = fmaf(xr[j + v], kr[v], acc[j]);
  }
  T* ob = out + ((size_t)n * O * O + (size_t)(r0 + i) * O) * C + c0 + lane;
#pragma unroll
  for (int j = 0; j < O; ++j) ob[(size_t)j * C] = from_f<T>(acc[j]);
}

// ---------------------------------------------------------------------------------------------
// Tensor-core form of the depthwise correlation (fp16 storage, fp32 accumulation).
// For one (track, channel):  Out(16x16) = sum_u X[u:u+16, 0:32) * B_u,  B_u[m][j] = K[u][m-j] (banded
// Toeplitz of template row u, zero outside 0 <= m-j < 15): 15 x (2 k-steps x 2 n-tiles) mma.sync.m16n8k16,
// ~2.1x redundant MACs on a pipe >10x faster than the FP32 FMAs -> the kernel is bound by staging, so the
// staging is what is organised carefully:
//  * one CTA = 16 channels of one track, one warp per channel in the MMA phase;
//  * window: a warp copies one (window row, 8-channel group) per step, lane = column: 16-byte global loads
//    (all issued before the first store), 2-byte transposing stores into per-channel planes
//    xT[c][row][col] (row pitch 80 B -> ldmatrix and the stores are bank-conflict free);
//  * template: staged the same way straight into TWO zero-padded copies of every template row
//    (kz[c][u][p][32]: K[u][v] at half 8 - p + v), so that a B fragment register (K[u][d], K[u][d+1]) is ONE
//    aligned 32-bit load for even and odd d alike.  With d0 = 2t - g the four MMAs of a (u) step need only the
//    words at d0, d0+8, d0+16: the operands at d0-8 and d0+24 are structurally zero (15 taps);
//  * results leave through the (dead) first 512 B of the warp's own window plane, packed half2, and are
//    written with 16-byte stores.
// ---------------------------------------------------------------------------------------------
constexpr int XM_CG = 16;                 // channels per CTA
constexpr int XM_WARPS = 16;              // one channel per warp
constexpr int XM_PITCH = 40;              // halves per window row in xT (30 data + 2 zero + pad; 80 B)
constexpr int XM_CSTRIDE = 30 * XM_PITCH + 8;  // halves between channel planes of xT (2416 B, 16-byte multiple)
constexpr int XM_KROW = 32;               // halves per zero-padded template-row copy
constexpr int XM_KPLANE = 15 * 2 * XM_KROW;    // halves per channel in kz
constexpr int XM_SMEM = (XM_CG * XM_CSTRIDE + XM_CG * XM_KPLANE) * 2;
static_assert(XM_CG == XM_WARPS, "the MMA phase maps one channel to one warp");
static_assert((XM_CG * XM_CSTRIDE * 2) % 16 == 0 && (XM_CSTRIDE * 2) % 16 == 0, "16-byte alignment of the planes");

__device__ __forceinline__ void xm_ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void xm_mma(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(XM_WARPS * 32) xcorr_mma_kernel(const __half* __restrict__ x, const __half* __restrict__ k,
                                                                 __half* __restrict__ out, int C) {
  constexpr int S = 30, TT = 15, O = 16;
  constexpr int XSTEPS = (S * 2 + XM_WARPS - 1) / XM_WARPS;    // (window row, channel half) pairs per warp
  constexpr int KSTEPS = (TT * 2 + XM_WARPS - 1) / XM_WARPS;   // (template row, channel half) pairs per warp
  extern __shared__ __align__(16) unsigned char xm_raw[];
  __half* xT = reinterpret_cast<__half*>(xm_raw);     // [CG][CSTRIDE]
  __half* kz = xT + XM_CG * XM_CSTRIDE;             // [CG][TT][2][KROW]
  const int n = blockIdx.y, c0 = blockIdx.x * XM_CG;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // ---- global loads first (in flight while the zero fill runs)
  const __half* xb = x + (size_t)n * S * S * C + c0;
  const __half* kb = k + (size_t)n * TT * TT * C + c0;
  uint4 xv[XSTEPS], kv[KSTEPS];
#pragma unroll
  for (int it = 0; it < XSTEPS; ++it) {
    const int idx = it * XM_WARPS + warp, r = idx >> 1, q = idx & 1;
    if (idx < S * 2 && lane < S) xv[it] = *reinterpret_cast<const uint4*>(xb + (size_t)(r * S + lane) * C + q * 8);
  }
#pragma unroll
  for (int it = 0; it < KSTEPS; ++it) {
    const int idx = it * XM_WARPS + warp, u = idx >> 1, q = idx & 1;
    if (idx < TT * 2 && lane < TT) kv[it] = *reinterpret_cast<const uint4*>(kb + (size_t)(u * TT + lane) * C + q * 8);
  }
  // ---- zero fill: the padded template rows entirely, columns 30/31 of every window row
  {
    uint4* kz4 = reinterpret_cast<uint4*>(kz);
    for (int i = tid; i < XM_CG * XM_KPLANE / 8; i += XM_WARPS * 32) kz4[i] = make_uint4(0u, 0u, 0u, 0u);
    if (tid < XM_CG * S) {
      const int c = tid / S, r = tid - c * S;
      *reinterpret_cast<uint32_t*>(xT + c * XM_CSTRIDE + r * XM_PITCH + S) = 0u;
    }
  }
  // ---- transposing stores of the window
#pragma unroll
  for (int it = 0; it < XSTEPS; ++it) {
    const int idx = it * XM_WARPS + warp, r = idx >> 1, q = idx & 1;
    if (idx < S * 2 && lane < S) {
      const __half* h = reinterpret_cast<const __half*>(&xv[it]);
      __half* dst = xT + (q * 8) * XM_CSTRIDE + r * XM_PITCH + lane;
#pragma unroll
      for (int e = 0; e < 8; ++e) dst[e * XM_CSTRIDE] = h[e];
    }
  }
  __syncthreads();  // template zero fill complete before the template values land
#pragma unroll
  for (int it = 0; it < KSTEPS; ++it) {
    const int idx = it * XM_WARPS + warp, u = idx >> 1, q = idx & 1;
    if (idx < TT * 2 && lane < TT) {
      const __half* h = reinterpret_cast<const __half*>(&kv[it]);
      __half* dst = kz + (q * 8) * XM_KPLANE + u * 2 * XM_KROW + 8 + lane;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        dst[e * XM_KPLANE] = h[e];                  // copy 0: K[u][v] at half 8 + v
        dst[e * XM_KPLANE + XM_KROW - 1] = h[e];    // copy 1: K[u][v] at half 7 + v
      }
    }
  }
  __syncthreads();
  // ---- MMA phase: warp = channel
  const int g = lane >> 2, t = lane & 3;
  const int a_row = (lane & 7) + ((lane >> 3) & 1) * 8, a_kh = lane >> 4;
  const int par = g & 1;
  const int c = warp;
  const uint32_t a_s = (uint32_t)__cvta_generic_to_shared(xT + c * XM_CSTRIDE + a_row * XM_PITCH + a_kh * 8);
  // word (8 - par + d0) / 2 of copy `par`, d0 = 2t - g in [-7, 6]
  const uint32_t* kzw = reinterpret_cast<const uint32_t*>(kz + c * XM_KPLANE + par * XM_KROW) + ((8 + 2 * t - g - par) >> 1);
  float acc[2][4];
#pragma unroll
  for (int j = 0; j < 2; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[j][e] = 0.f;
#pragma unroll 5
  for (int u = 0; u < TT; ++u) {
    const uint32_t k0 = kzw[u * XM_KROW], k8 = kzw[u * XM_KROW + 4], k16 = kzw[u * XM_KROW + 8];  // K[u][d0 + {0,8,16} (+1)]
    uint32_t af[4];
    // B[k][n] = K[u][k - n]; register b0 holds k = 16ks + 2t (+1), b1 the same + 8; n = 8nt + g
    xm_ldmatrix_x4(a_s + (uint32_t)(u * XM_PITCH * 2), af[0], af[1], af[2], af[3]);             // window cols 0..15
    xm_mma(acc[0], af, k0, k8);      // nt 0: d = d0, d0 + 8
    xm_mma(acc[1], af, 0u, k0);      // nt 1: d = d0 - 8 (no tap), d0
    xm_ldmatrix_x4(a_s + (uint32_t)(u * XM_PITCH * 2 + 32), af[0], af[1], af[2], af[3]);        // window cols 16..31
    xm_mma(acc[0], af, k16, 0u);     // nt 0: d = d0 + 16, d0 + 24 (no tap)
    xm_mma(acc[1], af, k8, k16);     // nt 1: d = d0 + 8, d0 + 16
  }
  // ---- D fragments -> the warp's own (now dead) window plane as [O*O] halves, then 16-byte stores
  __syncwarp();
  {
    __half2* ost = reinterpret_cast<__half2*>(xT + c * XM_CSTRIDE);
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      ost[g * 8 + nt * 4 + t] = __floats2half2_rn(acc[nt][0], acc[nt][1]);
      ost[(g + 8) * 8 + nt * 4 + t] = __floats2half2_rn(acc[nt][2], acc[nt][3]);
    }
  }
  __syncthreads();
  {
    const int q = warp & 1, pos = (warp >> 1) * 32 + lane;   // 256 positions x 2 channel halves = 512 threads
    const __half* src = xT + (q * 8) * XM_CSTRIDE + pos;
    __align__(16) __half h[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) h[e] = src[e * XM_CSTRIDE];
    *reinterpret_cast<uint4*>(out + ((size_t)n * O * O + pos) * C + c0 + q * 8) = *reinterpret_cast<const uint4*>(h);
  }
}

__device__ __forceinline__ void xm_ldmatrix_x2(uint32_t addr, uint32_t& r0, uint32_t& r1) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0, %1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(addr));
}
__device__ __forceinline__ void xm_mma_k8(float* c, uint32_t a0, uint32_t a1, uint32_t b0) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5}, {%6}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(b0));
}

// ---------------------------------------------------------------------------------------------
// Planar-input form of the tensor-core correlation (developer switch SMOT_XCORR_PLANAR, see DESIGN.md section 5.2).
//
// ncu on xcorr_mma_kernel puts the time in the window staging, not in the MMAs:
// 21.6 k global load requests touching 25 sectors each (a warp gathers 30 x 16 B at a 256-byte stride; every sector is
// requested twice), long-scoreboard + LSU-throttle stalls on 60 % of the issue slots, tensor pipe at 17 % of its rate.
// Here the search windows arrive CHANNEL-PLANAR from smot_roi_align_planar -- per (track, channel) a plane of
// XM_CSTRIDE halves with rows XM_PITCH apart, i.e. exactly the shared-memory image the MMA phase reads -- so the window
// staging of a CTA is four bulk async copies (cp.async.bulk, 38 656 B, complete_tx on one mbarrier) issued by a
// dedicated warp: no per-thread loads, no transposing stores, full-line L2 reads.  Columns 30 / 31 of every window row
// are zero in the producer's buffer (they meet structurally-zero B rows, but 0 x NaN must not happen).
//
// Programmatic dependent launch: everything that does not depend on the predecessor -- barrier init, zero fill and
// staging of the templates (written to HBM before the predecessor even started) -- runs before griddepcontrol.wait and
// overlaps the tail of the ROIAlign; the copy warp waits, then issues the bulk copies.  The MMA phase and the result
// path are those of xcorr_mma_kernel, instruction for instruction, so the outputs are bit-identical.
// ---------------------------------------------------------------------------------------------
// The channel group of a CTA is a template parameter (CG planes = CG MMA warps + 1 copy warp): the (track, channel) planes are
// independent, so CG only sets the granularity of the grid.  30 tracks x 128 channels are 240 CTAs of 16 planes -- 1.6 per SM,
// i.e. 92 SMs run 32 planes and 56 run 16 -- or 960 CTAs of 4 planes, at most 7 per SM = 28 planes (see DESIGN.md section 5.2
// for the measured ladder).  Template vectors are CG halves wide (at most 16 B), result vectors likewise.
template <int CG>
struct XpGeom {
  static_assert(CG == 2 || CG == 4 || CG == 8 || CG == 16, "channel group");
  static constexpr int WARPS = CG;                              // MMA warps (one plane each)
  static constexpr int THREADS = (CG + 1) * 32;                 // + 1 copy warp
  static constexpr int MMA_THREADS = CG * 32;
  static constexpr int X_HALVES = CG * XM_CSTRIDE, K_HALVES = CG * XM_KPLANE;
  static constexpr int BAR_OFF = (X_HALVES + K_HALVES) * 2;     // mbarriers behind the two staging areas
  static constexpr int COPIES = CG >= 4 ? CG / 2 : CG;          // bulk copies per CTA (2 planes each), one mbarrier per copy
  static constexpr int PLANES_PER_COPY = CG / COPIES;
  static constexpr int SMEM = BAR_OFF + 8 * COPIES;
  static constexpr int VH = CG < 8 ? CG : 8;                    // halves per template / result vector
  static constexpr int NCH = CG / VH;                           // vectors per position
  static constexpr int K_ITEMS = 15 * 15 * NCH;                 // template vectors per CTA
  static constexpr int K_ITERS = (K_ITEMS + MMA_THREADS - 1) / MMA_THREADS;
  static_assert(BAR_OFF % 8 == 0, "mbarrier alignment");
  static_assert(CG % COPIES == 0 && (PLANES_PER_COPY * XM_CSTRIDE * 2) % 16 == 0, "bulk copy size must be a 16-byte multiple");
};
template <int VH> struct XpVec;
template <> struct XpVec<2> { using type = uint32_t; };
template <> struct XpVec<4> { using type = uint2; };
template <> struct XpVec<8> { using type = uint4; };

__device__ __forceinline__ void xp_mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void xp_mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool xp_mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void xp_bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}

#ifdef SMOT_XCORR_TRACE
// developer build only (tools/xcorr_lab.py): per-warp phase stamps, [cta][warp][8] x (globaltimer, clock64 | smid << 48)
__device__ unsigned long long* g_xp_trace = nullptr;
extern "C" int smot_xcorr_trace_buffer(void* buf) { return cudaMemcpyToSymbol(g_xp_trace, &buf, sizeof(buf)) == cudaSuccess ? 0 : 1; }
#define XP_STAMP(slot)                                                                                                    \
  do {                                                                                                                    \
    if (g_xp_trace && (threadIdx.x & 31) == 0) {                                                                          \
      unsigned long long gt__;                                                                                            \
      unsigned sm__;                                                                                                      \
      asm volatile("mov.u64 %0, %globaltimer;" : "=l"(gt__));                                                             \
      asm volatile("mov.u32 %0, %smid;" : "=r"(sm__));                                                                    \
      unsigned long long* t__ = g_xp_trace + ((((size_t)blockIdx.y * gridDim.x + blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5)) * 8 + (slot)) * 2; \
      t__[0] = gt__, t__[1] = ((unsigned long long)clock64() & 0xffffffffffffull) | ((unsigned long long)sm__ << 48);    \
    }                                                                                                                     \
  } while (0)
#else
#define XP_STAMP(slot) do { } while (0)
#endif

// One plane: Out(16x16) = sum_u X[u:u+16, :32] * B_u on mma.sync from the plane's window image xw (shared memory, rows XM_PITCH
// apart) and its zero-padded template image kw; acc = the warp's D fragments (two n8 tiles).  Shared by the planar kernels.
template <int MMA_MODE>
__device__ __forceinline__ void xp_plane_mma(const __half* xw, const __half* kw, int lane, float (&acc)[2][4]) {
  constexpr int TT = 15;
  const int g = lane >> 2, t = lane & 3;
  const int a_row = (lane & 7) + ((lane >> 3) & 1) * 8, a_kh = lane >> 4;
  const int par = g & 1;
  const uint32_t a_s = (uint32_t)__cvta_generic_to_shared(xw + a_row * XM_PITCH + a_kh * 8);
  // the two copies of a template row sit 64 B apart: lanes with par = 0 / 1 read disjoint bank halves (conflict-free; a
  // pair-interleaved image with 64-bit loads was measured SLOWER: both copies then alias the same banks)
  const uint32_t* kzw = reinterpret_cast<const uint32_t*>(kw + par * XM_KROW) + ((8 + 2 * t - g - par) >> 1);
#pragma unroll
  for (int j = 0; j < 2; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[j][e] = 0.f;
  if constexpr (MMA_MODE == 0) {
#pragma unroll 5
    for (int u = 0; u < TT; ++u) {
      const uint32_t k0 = kzw[u * XM_KROW], k8 = kzw[u * XM_KROW + 4], k16 = kzw[u * XM_KROW + 8];
      uint32_t af[4];
      xm_ldmatrix_x4(a_s + (uint32_t)(u * XM_PITCH * 2), af[0], af[1], af[2], af[3]);
      xm_mma(acc[0], af, k0, k8);
      xm_mma(acc[1], af, 0u, k0);
      xm_ldmatrix_x4(a_s + (uint32_t)(u * XM_PITCH * 2 + 32), af[0], af[1], af[2], af[3]);
      xm_mma(acc[0], af, k16, 0u);
      xm_mma(acc[1], af, k8, k16);
    }
  } else {
    // one template row: window rows [u, u+16) as fragments lo (cols 0..15) / hi (cols 16..31)
    auto row_step = [&](const uint32_t* lo, const uint32_t* hi, int u) {
      const uint32_t k0 = kzw[u * XM_KROW], k8 = kzw[u * XM_KROW + 4], k16 = kzw[u * XM_KROW + 8];
      xm_mma(acc[0], lo, k0, k8);              // out cols 0..7  <- window cols 0..15
      xm_mma_k8(acc[1], lo[2], lo[3], k0);     // out cols 8..15 <- window cols 8..15   (cols 0..7 meet no tap)
      xm_mma_k8(acc[0], hi[0], hi[1], k16);    // out cols 0..7  <- window cols 16..23  (cols 24..31 meet no tap)
      xm_mma(acc[1], hi, k8, k16);             // out cols 8..15 <- window cols 16..31
    };
    // lanes 0..15 address the x2 loads: rows (lane & 7) + 16 of the pair's 24-row span, column half (lane >> 3) & 1
    const uint32_t a_x2 = (uint32_t)__cvta_generic_to_shared(xw + ((lane & 7) + 16) * XM_PITCH + ((lane >> 3) & 1) * 8);
#pragma unroll
    for (int u = 0; u < 7; ++u) {
      uint32_t lo[4], hi[4], lo2[4], hi2[4];
      xm_ldmatrix_x4(a_s + (uint32_t)(u * XM_PITCH * 2), lo[0], lo[1], lo[2], lo[3]);
      xm_ldmatrix_x4(a_s + (uint32_t)(u * XM_PITCH * 2 + 32), hi[0], hi[1], hi[2], hi[3]);
      // rows u+8..u+15 are the second row block of the fragments above; rows u+16..u+23 are new
      lo2[0] = lo[1], lo2[2] = lo[3], hi2[0] = hi[1], hi2[2] = hi[3];
      xm_ldmatrix_x2(a_x2 + (uint32_t)(u * XM_PITCH * 2), lo2[1], lo2[3]);
      xm_ldmatrix_x2(a_x2 + (uint32_t)(u * XM_PITCH * 2 + 32), hi2[1], hi2[3]);
      row_step(lo, hi, u);
      row_step(lo2, hi2, u + 8);
    }
    {
      uint32_t lo[4], hi[4];
      xm_ldmatrix_x4(a_s + (uint32_t)(7 * XM_PITCH * 2), lo[0], lo[1], lo[2], lo[3]);
      xm_ldmatrix_x4(a_s + (uint32_t)(7 * XM_PITCH * 2 + 32), hi[0], hi[1], hi[2], hi[3]);
      row_step(lo, hi, 7);
    }
  }
}

// MMA_MODE 0: the MMA phase of xcorr_mma_kernel, instruction for instruction (bit-identical results).
// MMA_MODE 1 (default): the same contraction with the structurally-zero work removed --
//   * of the four m16n8k16 per template row, two have an all-zero B half (taps d0-8 and d0+24 do not exist): they become
//     m16n8k8 on the live half (window columns 8..15 for output columns 8..15, 16..23 for output columns 0..7): 3 instead of
//     4 k16-equivalents per row, -25 % tensor work;
//   * template rows u and u+8 read window rows u..u+15 and u+8..u+23: the second block of the first is the first block of
//     the second, so the pair costs ldmatrix x4 + x2 per column half instead of 2 x4 (-25 % shared-memory wavefronts).
//   The accumulation order differs from mode 0 (fp32 rounding), so the results agree to fp16 rounding, not bit for bit.
// The results do not depend on CG (the planes are independent and each is computed by one warp in a fixed order).
template <int MMA_MODE, int CG>
__global__ void __launch_bounds__(XpGeom<CG>::THREADS) xcorr_planar_kernel(const __half* __restrict__ xp, const __half* __restrict__ k,
                                                                          __half* __restrict__ out, int C) {
  using G = XpGeom<CG>;
  using KVec = typename XpVec<G::VH>::type;
  constexpr int S = 30, TT = 15, O = 16;
  static_assert(S * XM_PITCH + 8 == XM_CSTRIDE, "plane = 30 rows of XM_PITCH halves + 8");
  extern __shared__ __align__(128) unsigned char xp_raw[];
  __half* xT = reinterpret_cast<__half*>(xp_raw);     // [CG][CSTRIDE]: filled by the bulk copies
  __half* kz = xT + G::X_HALVES;                      // [CG][TT][2][KROW]
  const uint32_t bar = (uint32_t)__cvta_generic_to_shared(xp_raw + G::BAR_OFF);   // COPIES mbarriers, 8 bytes apart
  const int n = blockIdx.y, c0 = blockIdx.x * CG;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool copy_warp = warp == G::WARPS;
  pdl_launch_dependents();
  XP_STAMP(0);
  // ---- prologue (independent of the predecessor's output): template vectors to registers, zero fill of the padded copies
  const __half* kb = k + (size_t)n * TT * TT * C + c0;
  KVec kv[G::K_ITERS];
  if (!copy_warp) {
#pragma unroll
    for (int it = 0; it < G::K_ITERS; ++it) {
      const int i = it * G::MMA_THREADS + tid;
      // item = (vector column q, tap p), q-major: the lanes of a warp hold consecutive taps of ONE column, so the 2-byte
      // scatter below lands in consecutive halves (a tap-major order put neighbouring lanes 15 KB apart = on one bank)
      if (i < G::K_ITEMS) kv[it] = *reinterpret_cast<const KVec*>(kb + (size_t)(i % (TT * TT)) * C + (i / (TT * TT)) * 8);
    }
    uint4* kz4 = reinterpret_cast<uint4*>(kz);
    for (int i = tid; i < G::K_HALVES / 8; i += G::MMA_THREADS) kz4[i] = make_uint4(0u, 0u, 0u, 0u);
  } else if (lane == 0) {
#pragma unroll
    for (int i = 0; i < G::COPIES; ++i) xp_mbar_init(bar + 8 * i, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();  // template zero fill complete; the mbarriers are initialised for every thread
  XP_STAMP(1);
  if (copy_warp) {
    // ---- window: wait for the producer of the planes, then one bulk copy per plane pair, each onto its own mbarrier:
    // a warp starts as soon as ITS plane is there, the tensor pipe is busy from the first arrival on
    pdl_wait();
    XP_STAMP(2);
    if (lane == 0) {
      constexpr uint32_t BYTES = G::PLANES_PER_COPY * XM_CSTRIDE * 2;
      const __half* src = xp + ((size_t)n * C + c0) * XM_CSTRIDE;
#pragma unroll
      for (int i = 0; i < G::COPIES; ++i) {
        xp_mbar_expect_tx(bar + 8 * i, BYTES);
        xp_bulk_g2s((uint32_t)__cvta_generic_to_shared(xT) + i * BYTES, reinterpret_cast<const unsigned char*>(src) + (size_t)i * BYTES,
                    BYTES, bar + 8 * i);
      }
    }
  } else {
#pragma unroll
    for (int it = 0; it < G::K_ITERS; ++it) {
      const int i = it * G::MMA_THREADS + tid;
      if (i < G::K_ITEMS) {
        const int p = i % (TT * TT), q = i / (TT * TT), u = p / TT, v = p % TT;
        const __half* h = reinterpret_cast<const __half*>(&kv[it]);
        __half* dst = kz + (q * 8) * XM_KPLANE + u * 2 * XM_KROW + 8 + v;
#pragma unroll
        for (int e = 0; e < G::VH; ++e) {
          dst[e * XM_KPLANE] = h[e];                  // copy 0: K[u][v] at half 8 + v
          dst[e * XM_KPLANE + XM_KROW - 1] = h[e];    // copy 1: K[u][v] at half 7 + v
        }
      }
    }
    XP_STAMP(2);
  }
  __syncthreads();  // templates staged (nothing so far depends on the predecessor: under PDL this all ran beside its tail)
  XP_STAMP(3);
  float acc[2][4];
  const int g = lane >> 2, t = lane & 3;
  const int c = warp;
  if (!copy_warp) {
    // bounded wait for the windows (wall clock, 2 s): a mis-programmed copy must fail the launch, never hang the GPU
    unsigned long long t_start = 0;
    const uint32_t my_bar = bar + 8 * (warp / G::PLANES_PER_COPY);
    for (uint32_t spin = 0; !xp_mbar_try_wait(my_bar, 0); ++spin) {
      if ((spin & 255u) == 255u) {
        unsigned long long now;
        asm volatile("mov.u64 %0, %globaltimer;" : "=l"(now));
        if (t_start == 0) t_start = now;
        if (now - t_start > 2000000000ull) {
          printf("smot xcorr_planar: bulk copy wait timed out (block %d,%d thread %d)\n", blockIdx.x, blockIdx.y, tid);
          __trap();
        }
      }
    }
    XP_STAMP(4);
    // ---- MMA phase: warp = channel (identical to xcorr_mma_kernel) + D fragments -> the warp's own (now dead) window plane
    xp_plane_mma<MMA_MODE>(xT + c * XM_CSTRIDE, kz + c * XM_KPLANE, lane, acc);
    XP_STAMP(5);
    // ---- D fragments -> the warp's own (now dead) window plane as [O*O] halves
    __syncwarp();
    __half2* ost = reinterpret_cast<__half2*>(xT + c * XM_CSTRIDE);
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      ost[g * 8 + nt * 4 + t] = __floats2half2_rn(acc[nt][0], acc[nt][1]);
      ost[(g + 8) * 8 + nt * 4 + t] = __floats2half2_rn(acc[nt][2], acc[nt][3]);
    }
  }
  __syncthreads();
  XP_STAMP(6);
  if (!copy_warp) {
    pdl_wait();  // the result stores must not pass the predecessor (back-to-back launches share `out`); long returned by now
    // O*O positions x NCH result vectors: a warp takes 32 consecutive positions of one vector column
#pragma unroll
    for (int i = tid; i < O * O * G::NCH; i += G::MMA_THREADS) {
      const int q = i / (O * O), pos = i % (O * O);
      const __half* src = xT + (q * 8) * XM_CSTRIDE + pos;
      __align__(16) __half h[G::VH];
#pragma unroll
      for (int e = 0; e < G::VH; ++e) h[e] = src[e * XM_CSTRIDE];
      *reinterpret_cast<KVec*>(out + ((size_t)n * O * O + pos) * C + c0 + q * 8) = *reinterpret_cast<const KVec*>(h);
    }
  }
  XP_STAMP(7);
}

// ---------------------------------------------------------------------------------------------
// Flat form of the planar kernel for launches that fit ONE wave (n * C <= 28 planes per SM).
// (Developer variant, measured SLOWER than the 16-plane CTAs -- see xcorr_flat_enabled() -- and therefore not the default.)
// With 16 planes per CTA, 3840 planes are 240 CTAs on 132 SMs: 108 SMs run 32 planes, 24 run 16, and the launch ends with the
// loaded ones.  Here the plane list is cut into 4-plane
// units (a unit never straddles a track or an 8-byte channel vector) and CTA b of gridDim.x takes units
// [b * U / grid, (b + 1) * U / grid): 24 or 28 planes on EVERY SM, one CTA per SM, one MMA warp per plane (up to 28 + the copy
// warp).  Templates and results move as 8-byte vectors (a unit's four channels).  Per-plane arithmetic is xp_plane_mma's, so the
// results are the same bits as xcorr_planar_kernel's.
// ---------------------------------------------------------------------------------------------
constexpr int XF_MAX_UNITS = 7, XF_MAX_PLANES = 4 * XF_MAX_UNITS;
constexpr int XF_THREADS = (XF_MAX_PLANES + 1) * 32, XF_MMA_THREADS = XF_MAX_PLANES * 32;
constexpr int XF_BAR_OFF = XF_MAX_PLANES * (XM_CSTRIDE + XM_KPLANE) * 2;
constexpr int XF_SMEM = XF_BAR_OFF + 8 * (XF_MAX_PLANES / 2);
constexpr int XF_K_ITERS = (15 * 15 * XF_MAX_UNITS + XF_MMA_THREADS - 1) / XF_MMA_THREADS;
static_assert(XF_BAR_OFF % 8 == 0 && XF_THREADS <= 1024, "flat kernel geometry");

template <int MMA_MODE>
__global__ void __launch_bounds__(XF_THREADS, 1) xcorr_flat_kernel(const __half* __restrict__ xp, const __half* __restrict__ k,
                                                                   __half* __restrict__ out, int C, int units_total) {
  constexpr int TT = 15, O = 16;
  extern __shared__ __align__(128) unsigned char xp_raw[];
  __half* xT = reinterpret_cast<__half*>(xp_raw);                   // [28][CSTRIDE]
  __half* kz = xT + XF_MAX_PLANES * XM_CSTRIDE;                     // [28][TT][2][KROW]
  const uint32_t bar = (uint32_t)__cvta_generic_to_shared(xp_raw + XF_BAR_OFF);   // one mbarrier per plane pair
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool copy_warp = warp == XF_MAX_PLANES;
  const int u0 = (int)(((long long)blockIdx.x * units_total) / gridDim.x);
  const int u1 = (int)(((long long)(blockIdx.x + 1) * units_total) / gridDim.x);
  const int units = u1 - u0, planes = 4 * units, p0 = 4 * u0;      // units <= XF_MAX_UNITS (checked by the launcher)
  pdl_launch_dependents();
  // ---- prologue (independent of the predecessor): this CTA's templates to registers (8 bytes = a unit's channels of one tap),
  // unit-major so that a warp's scatter below lands in consecutive halves; zero fill of the padded copies
  uint2 kv[XF_K_ITERS];
  if (!copy_warp) {
#pragma unroll
    for (int it = 0; it < XF_K_ITERS; ++it) {
      const int i = it * XF_MMA_THREADS + tid, unit = i / (TT * TT), tap = i - unit * (TT * TT);
      if (unit < units) {
        const int plane = p0 + 4 * unit, n = plane / C, c = plane - n * C;
        kv[it] = *reinterpret_cast<const uint2*>(k + ((size_t)n * TT * TT + tap) * C + c);
      }
    }
    uint4* kz4 = reinterpret_cast<uint4*>(kz);
    for (int i = tid; i < planes * XM_KPLANE / 8; i += XF_MMA_THREADS) kz4[i] = make_uint4(0u, 0u, 0u, 0u);
  } else if (lane == 0) {
    for (int i = 0; i < XF_MAX_PLANES / 2; ++i) xp_mbar_init(bar + 8 * i, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  if (copy_warp) {
    pdl_wait();
    if (lane == 0) {
      constexpr uint32_t BYTES = 2 * XM_CSTRIDE * 2;
      const unsigned char* src = reinterpret_cast<const unsigned char*>(xp + (size_t)p0 * XM_CSTRIDE);
      for (int i = 0; i < planes / 2; ++i) {
        xp_mbar_expect_tx(bar + 8 * i, BYTES);
        xp_bulk_g2s((uint32_t)__cvta_generic_to_shared(xT) + i * BYTES, src + (size_t)i * BYTES, BYTES, bar + 8 * i);
      }
    }
  } else {
#pragma unroll
    for (int it = 0; it < XF_K_ITERS; ++it) {
      const int i = it * XF_MMA_THREADS + tid, unit = i / (TT * TT), tap = i - unit * (TT * TT);
      if (unit < units) {
        const int u = tap / TT, v = tap - u * TT;
        const __half* h = reinterpret_cast<const __half*>(&kv[it]);
        __half* dst = kz + (unit * 4) * XM_KPLANE + u * 2 * XM_KROW + 8 + v;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          dst[e * XM_KPLANE] = h[e];                  // copy 0: K[u][v] at half 8 + v
          dst[e * XM_KPLANE + XM_KROW - 1] = h[e];    // copy 1: K[u][v] at half 7 + v
        }
      }
    }
  }
  __syncthreads();  // templates staged
  if (!copy_warp && warp < planes) {
    unsigned long long t_start = 0;
    const uint32_t my_bar = bar + 8 * (warp >> 1);
    for (uint32_t spin = 0; !xp_mbar_try_wait(my_bar, 0); ++spin) {
      if ((spin & 255u) == 255u) {
        unsigned long long now;
        asm volatile("mov.u64 %0, %globaltimer;" : "=l"(now));
        if (t_start == 0) t_start = now;
        if (now - t_start > 2000000000ull) {
          printf("smot xcorr_flat: bulk copy wait timed out (block %d thread %d)\n", blockIdx.x, tid);
          __trap();
        }
      }
    }
    float acc[2][4];
    xp_plane_mma<MMA_MODE>(xT + warp * XM_CSTRIDE, kz + warp * XM_KPLANE, lane, acc);
    __syncwarp();
    const int g = lane >> 2, t = lane & 3;
    __half2* ost = reinterpret_cast<__half2*>(xT + warp * XM_CSTRIDE);
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      ost[g * 8 + nt * 4 + t] = __floats2half2_rn(acc[nt][0], acc[nt][1]);
      ost[(g + 8) * 8 + nt * 4 + t] = __floats2half2_rn(acc[nt][2], acc[nt][3]);
    }
  }
  __syncthreads();
  if (!copy_warp) {
    pdl_wait();  // the result stores must not pass the predecessor
    for (int i = tid; i < O * O * units; i += XF_MMA_THREADS) {
      const int unit = i / (O * O), pos = i - unit * (O * O);
      const int plane = p0 + 4 * unit, n = plane / C, c = plane - n * C;
      const __half* src = xT + (unit * 4) * XM_CSTRIDE + pos;
      __align__(8) __half h[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) h[e] = src[e * XM_CSTRIDE];
      *reinterpret_cast<uint2*>(out + ((size_t)n * O * O + pos) * C + c) = *reinterpret_cast<const uint2*>(h);
    }
  }
}

// generic fallback for unusual geometries: one thread per output element
template <typename T>
__global__ void xcorr_generic_kernel(const T* __restrict__ x, const T* __restrict__ k, T* __restrict__ out, int n, int C,
                                     int S, int TT) {
  const int O = S - TT + 1;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)n * O * O * C) return;
  const int c = (int)(idx % C);
  size_t r = idx / C;
  const int j = (int)(r % O), i = (int)((r / O) % O), t = (int)(r / ((size_t)O * O));
  const T* xb = x + (size_t)t * S * S * C + c;
  const T* kb = k + (size_t)t * TT * TT * C + c;
  float acc = 0.f;
  for (int u = 0; u < TT; ++u)
    for (int v = 0; v < TT; ++v) acc = fmaf(to_f(xb[(size_t)((i + u) * S + j + v) * C]), to_f(kb[(size_t)(u * TT + v) * C]), acc);
  out[idx] = from_f<T>(acc);
}

template <typename T, int S, int TT>
static int launch_xcorr(const void* x, const void* k, void* out, int n, int C, cudaStream_t st) {
  constexpr int XR = (S - TT + 1) / 2 + TT - 1;
  const size_t smem = ((size_t)XR * S * 32 * sizeof(T) + 15) / 16 * 16 + (size_t)TT * TT * 32 * sizeof(float);
  SMOT_ENSURE_SMEM((xcorr_kernel<T, S, TT>), smem, "smot_xcorr");
  xcorr_kernel<T, S, TT><<<dim3(C / 32, n, 2), 256, smem, st>>>((const T*)x, (const T*)k, (T*)out, C);
  SMOT_CHECK_LAUNCH("smot_xcorr");
  return SMOT_OK;
}

// =============================================================================================
// fused bicubic upsample + decode
// =============================================================================================
constexpr int EMM_CH = 7;

constexpr int EMM_MAX_BAND = 64;   // rows of the upsampled map per CTA (= the upsampling factor, 16 in every shipped configuration)
struct CubicTap {
  int idx[4];
  float w[4];
};

// ATen upsample_bicubic2d (align_corners=False, A=-0.75): source index, taps clamped to the map
__device__ __forceinline__ CubicTap cubic_taps(int dst, float scale, int in_size) {
  const float A = -0.75f;
  const float src = scale * ((float)dst + 0.5f) - 0.5f;
  const float fl = floorf(src);
  const float t = src - fl;
  const int i0 = (int)fl;
  CubicTap c;
#pragma unroll
  for (int j = 0; j < 4; ++j) c.idx[j] = min(max(i0 - 1 + j, 0), in_size - 1);
  const float x0 = t + 1.f, x3 = (1.f - t) + 1.f, x2 = 1.f - t;
  c.w[0] = ((A * x0 - 5.f * A) * x0 + 8.f * A) * x0 - 4.f * A;
  c.w[1] = ((A + 2.f) * t - (A + 3.f)) * t * t + 1.f;
  c.w[2] = ((A + 2.f) * x2 - (A + 3.f)) * x2 * x2 + 1.f;
  c.w[3] = ((A * x3 - 5.f * A) * x3 + 8.f * A) * x3 - 4.f * A;
  return c;
}

struct DecodeArgs {
  const float* maps;
  int map_ld, n, O, up, T;
  const float* sr;
  const float* tboxes;
  const float* hann;  // [O*up]
  float pad;
  int use_centerness;
  float sigma, one_minus_sigma;
  int img_w, img_h, amodal;
  int rows_per_cta, rows_max;
  unsigned long long* best;  // [n]
  float* out_boxes;
  float* out_conf;
  int* out_valid;
};

__device__ __forceinline__ float hsum4(const float* v, const float* w) {
  // ((w0*v0 + w1*v1) + w2*v2) + w3*v3, same association as ATen's interpolate loop
  return ((w[0] * v[0] + w[1] * v[1]) + w[2] * v[2]) + w[3] * v[3];
}

struct PixelEval {
  float score, p1, tlbr[4];
};

// everything after the upsampled channel values are known (decode_response, track_core.py:101-118)
__device__ __forceinline__ PixelEval eval_pixel(const float* c, float box_w, float box_h, float win, int use_centerness,
                                                float sigma, float one_minus_sigma) {
  PixelEval e;
  const float m = fmaxf(c[0], c[1]);
  const float e0 = expf(c[0] - m), e1 = expf(c[1] - m);
  e.p1 = __fdiv_rn(e1, e0 + e1);
  float conf = e.p1;
  if (use_centerness) conf = e.p1 * __fdiv_rn(1.f, 1.f + expf(-c[2]));
  float sw = __fdiv_rn(c[5] + c[3], box_w), sh = __fdiv_rn(c[6] + c[4], box_h);
  sw = fmaxf(sw, __fdiv_rn(1.f, sw));
  sh = fmaxf(sh, __fdiv_rn(1.f, sh));
  const float pen = expf((-sw * sh + 1.f) * 0.1f);
  e.score = (conf * pen) * one_minus_sigma + sigma * win;
#pragma unroll
  for (int j = 0; j < 4; ++j) e.tlbr[j] = c[3 + j];
  return e;
}

// grid (row bands, tracks): a CTA scores rows [y0, y1) of the upsampled map.  It upsamples horizontally only the
// source rows its band touches (rows_per_cta / up + 4 at most), so the staging buffer is a few tens of KB and
// several CTAs share an SM; the arithmetic per pixel is unchanged.
__global__ void __launch_bounds__(256) emm_score_kernel(const DecodeArgs a) {
  extern __shared__ __align__(16) float dec_smem[];
  const int O = a.O, OW = a.O * a.up;
  float* maps_s = dec_smem;                 // [O*O][EMM_CH]
  float* tmp = dec_smem + O * O * EMM_CH;   // [EMM_CH][rows_max][OW] horizontally upsampled rows r_lo..r_hi
  const int n = blockIdx.y;
  const float scale = 1.f / (float)a.up;
  const int y0 = blockIdx.x * a.rows_per_cta, y1 = min(OW, y0 + a.rows_per_cta);
  const int r_lo = cubic_taps(y0, scale, O).idx[0], r_hi = cubic_taps(y1 - 1, scale, O).idx[3];  // <= rows_max rows
  const float* mp = a.maps + (size_t)n * O * O * a.map_ld;
  for (int i = threadIdx.x + r_lo * O * EMM_CH; i < (r_hi + 1) * O * EMM_CH; i += blockDim.x)
    maps_s[i] = mp[(size_t)(i / EMM_CH) * a.map_ld + (i % EMM_CH)];
  // the vertical taps and the window weight of the band's rows: once per CTA instead of once per pixel (same values)
  __shared__ CubicTap ty_s[EMM_MAX_BAND];
  __shared__ float hann_y[EMM_MAX_BAND];
  if ((int)threadIdx.x < y1 - y0) {
    CubicTap t = cubic_taps(y0 + (int)threadIdx.x, scale, O);
#pragma unroll
    for (int j = 0; j < 4; ++j) t.idx[j] = (t.idx[j] - r_lo) * OW;   // element offset of the tap's row inside a channel of `tmp`
    ty_s[threadIdx.x] = t;
    hann_y[threadIdx.x] = a.hann[y0 + threadIdx.x];
  }
  __syncthreads();
  for (int x = threadIdx.x; x < OW; x += blockDim.x) {
    const CubicTap tx = cubic_taps(x, scale, O);
    for (int r = r_lo; r <= r_hi; ++r)
#pragma unroll
      for (int ch = 0; ch < EMM_CH; ++ch) {
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = maps_s[(r * O + tx.idx[j]) * EMM_CH + ch];
        tmp[(ch * a.rows_max + (r - r_lo)) * OW + x] = hsum4(v, tx.w);
      }
  }
  __syncthreads();
  const float box_w = a.tboxes[n * 4 + 2] - a.tboxes[n * 4 + 0];
  const float box_h = a.tboxes[n * 4 + 3] - a.tboxes[n * 4 + 1];
  unsigned long long best = 0ull;
  for (int x = threadIdx.x; x < OW; x += blockDim.x) {
    const float wx = a.hann[x];
    const float* tcol = tmp + x;
    const int ch_stride = a.rows_max * OW;
    for (int y = y0; y < y1; ++y) {
      const CubicTap ty = ty_s[y - y0];
      float c[EMM_CH];
#pragma unroll
      for (int ch = 0; ch < EMM_CH; ++ch) {
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = tcol[ch * ch_stride + ty.idx[j]];
        c[ch] = hsum4(v, ty.w);
      }
      const PixelEval e = eval_pixel(c, box_w, box_h, hann_y[y - y0] * wx, a.use_centerness, a.sigma, a.one_minus_sigma);
      // scores are >= 0 here (conf, pen, window >= 0), so the raw float bits order like the floats
      const unsigned idx = (unsigned)(y * OW + x);
      const unsigned long long key = ((unsigned long long)__float_as_uint(fmaxf(e.score, 0.f)) << 32) |
                                     (unsigned long long)(0xFFFFFFFFu - idx);
      best = key > best ? key : best;
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
    best = other > best ? other : best;
  }
  if ((threadIdx.x & 31) == 0) atomicMax(&a.best[n], best);
}

__global__ void emm_finalize_kernel(const DecodeArgs a) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= a.n) return;
  const int O = a.O, OW = a.O * a.up;
  const unsigned idx = 0xFFFFFFFFu - (unsigned)(a.best[n] & 0xFFFFFFFFull);
  const int y = (int)(idx / OW), x = (int)(idx % OW);
  const float scale = 1.f / (float)a.up;
  const CubicTap tx = cubic_taps(x, scale, O), ty = cubic_taps(y, scale, O);
  const float* mp = a.maps + (size_t)n * O * O * a.map_ld;
  float c[EMM_CH];
  for (int ch = 0; ch < EMM_CH; ++ch) {
    float rowv[4];
    for (int i = 0; i < 4; ++i) {
      float v[4];
      for (int j = 0; j < 4; ++j) v[j] = mp[(size_t)(ty.idx[i] * O + tx.idx[j]) * a.map_ld + ch];
      rowv[i] = hsum4(v, tx.w);
    }
    c[ch] = hsum4(rowv, ty.w);
  }
  const float* tb = a.tboxes + n * 4;
  const PixelEval e = eval_pixel(c, tb[2] - tb[0], tb[3] - tb[1], a.hann[y] * a.hann[x], a.use_centerness, a.sigma,
                                 a.one_minus_sigma);
  // get_locations (track_core.py:184-225): SR box sampled on an (S*up)^2 grid, S = O + T - 1
  const float* s = a.sr + n * 4;
  const int s_full = (O + 2 * (a.T / 2)) * a.up;
  const int border = (a.T / 2) * a.up;
  const float stride_w = __fdiv_rn(s[2] - s[0], (float)(s_full - 1));
  const float stride_h = __fdiv_rn(s[3] - s[1], (float)(s_full - 1));
  const float cx = (s[0] + (float)(border + x) * stride_w) - a.pad;
  const float cy = (s[1] + (float)(border + y) * stride_h) - a.pad;
  float x1 = cx - e.tlbr[0], y1 = cy - e.tlbr[1], x2 = cx + e.tlbr[2], y2 = cy + e.tlbr[3];
  int valid = 1;
  if (!a.amodal) {
    x1 = fminf(fmaxf(x1, 0.f), (float)a.img_w - 1.f), y1 = fminf(fmaxf(y1, 0.f), (float)a.img_h - 1.f);
    x2 = fminf(fmaxf(x2, 0.f), (float)a.img_w - 1.f), y2 = fminf(fmaxf(y2, 0.f), (float)a.img_h - 1.f);
    valid = (y2 > y1) && (x2 > x1);
  }
  reinterpret_cast<float4*>(a.out_boxes)[n] = make_float4(x1, y1, x2, y2);
  a.out_conf[n] = e.p1;
  a.out_valid[n] = valid;
}

}  // namespace smot

using namespace smot;

extern "C" int smot_xcorr(const void* x, const void* k, void* out, int n, int channels, int S, int T, int dtype,
                          void* stream) {
  SMOT_CHECK_ARG(n >= 0 && channels > 0 && T >= 1 && S >= T, "smot_xcorr: bad geometry n=%d C=%d S=%d T=%d", n, channels, S, T);
  if (n == 0) return SMOT_OK;
  SMOT_CHECK_ARG(x && k && out, "smot_xcorr: null argument");
  SMOT_CHECK_ARG(dtype == SMOT_F32 || dtype == SMOT_F16, "smot_xcorr: bad dtype %d", dtype);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == SMOT_F16 && S == 30 && T == 15 && channels % XM_CG == 0 &&
      (((uintptr_t)x | (uintptr_t)k | (uintptr_t)out) & 15) == 0) {
    SMOT_ENSURE_SMEM(xcorr_mma_kernel, XM_SMEM, "smot_xcorr(mma)");
    xcorr_mma_kernel<<<dim3(channels / XM_CG, n), XM_WARPS * 32, XM_SMEM, st>>>((const __half*)x, (const __half*)k, (__half*)out, channels);
    SMOT_CHECK_LAUNCH("smot_xcorr(mma)");
    return SMOT_OK;
  }
  const bool fast = channels % 32 == 0 && (((uintptr_t)x | (uintptr_t)k) & 15) == 0;
  if (fast && S == 30 && T == 15)
    return dtype == SMOT_F32 ? launch_xcorr<float, 30, 15>(x, k, out, n, channels, st)
                             : launch_xcorr<__half, 30, 15>(x, k, out, n, channels, st);
  const int O = S - T + 1;
  const size_t total = (size_t)n * O * O * channels;
  const unsigned blocks = (unsigned)((total + 255) / 256);
  if (dtype == SMOT_F32)
    xcorr_generic_kernel<float><<<blocks, 256, 0, st>>>((const float*)x, (const float*)k, (float*)out, n, channels, S, T);
  else
    xcorr_generic_kernel<__half><<<blocks, 256, 0, st>>>((const __half*)x, (const __half*)k, (__half*)out, n, channels, S, T);
  SMOT_CHECK_LAUNCH("smot_xcorr(generic)");
  return SMOT_OK;
}

// the trimmed MMA phase is the default; developer switch SMOT_XCORR_PLANAR=1 selects the untrimmed one (read once)
static bool xcorr_planar_trimmed() {
  static const bool on = [] {
    const char* e = getenv("SMOT_XCORR_PLANAR");
    return !(e && e[0] == '1');
  }();
  return on;
}

// planes per CTA: 16 while all CTAs are resident at once (two per SM), 8 beyond that (the fastest of 2 / 4 / 8 / 16 at
// 30 and 80 tracks when it was chosen; not re-measured on the H100).  Developer switch SMOT_XCORR_CG (read once).
static int xcorr_planar_cg(int planes) {
  static const int forced = [] {
    const char* e = getenv("SMOT_XCORR_CG");
    const int v = e ? atoi(e) : 0;
    return (v == 2 || v == 4 || v == 8 || v == 16) ? v : 0;
  }();
  if (forced) return forced;
  return planes <= 16 * 2 * sm_count() ? 16 : 8;
}

extern "C" int smot_xcorr_planar(const void* x_planar, const void* k, void* out, int n, int channels, void* stream) {
  return smot_xcorr_planar_mode(x_planar, k, out, n, channels, xcorr_planar_trimmed() ? 1 : 0, stream);
}

// developer switch SMOT_XCORR_FLAT=1 (read once): the flat form whenever the planes fit one wave of 28 per SM.  OFF by default:
// measured slower than 16-plane CTAs at 30 x 128 when it was written -- the balance it buys (28 instead
// of 32 planes on the busiest SM) is worth less than what one 29-warp CTA per SM loses: its phases (template staging, wait for
// the windows, MMA, result path) cannot overlap with those of a second CTA, its block barriers span 928 threads, and templates /
// results move as 8-byte instead of 16-byte vectors.
static bool xcorr_flat_enabled() {
  static const bool on = [] {
    const char* e = getenv("SMOT_XCORR_FLAT");
    return e && e[0] == '1';
  }();
  return on;
}

extern "C" int smot_xcorr_planar_mode(const void* x_planar, const void* k, void* out, int n, int channels, int mma_mode,
                                      void* stream) {
  if (xcorr_flat_enabled() && channels % 4 == 0 && (long long)n * channels <= (long long)XF_MAX_PLANES * sm_count())
    return smot_xcorr_planar_cfg(x_planar, k, out, n, channels, mma_mode, 0, stream);
  int cg = xcorr_planar_cg(n * channels);
  while (cg > 2 && channels % cg) cg >>= 1;
  return smot_xcorr_planar_cfg(x_planar, k, out, n, channels, mma_mode, cg, stream);
}

template <int MODE, int CG>
static cudaError_t launch_xcorr_planar(const void* x, const void* k, void* out, int n, int C, cudaStream_t st) {
  using G = XpGeom<CG>;
  if (G::SMEM > 48 * 1024) {
    static bool granted[::smot::SMOT_MAX_DEVICES];
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev >= 0 && dev < ::smot::SMOT_MAX_DEVICES && !granted[dev]) {
      cudaError_t e = cudaFuncSetAttribute(xcorr_planar_kernel<MODE, CG>, cudaFuncAttributeMaxDynamicSharedMemorySize, G::SMEM);
      if (e != cudaSuccess) return e;
      granted[dev] = true;
    }
  }
  return launch_pdl(xcorr_planar_kernel<MODE, CG>, dim3(C / CG, n), dim3(G::THREADS), G::SMEM, st, (const __half*)x, (const __half*)k,
                    (__half*)out, C);
}

extern "C" int smot_xcorr_planar_cfg(const void* x_planar, const void* k, void* out, int n, int channels, int mma_mode,
                                     int channel_group, void* stream) {
  const int cg = channel_group;
  SMOT_CHECK_ARG(mma_mode == 0 || mma_mode == 1, "smot_xcorr_planar: mma_mode %d", mma_mode);
  SMOT_CHECK_ARG(cg == 0 || cg == 2 || cg == 4 || cg == 8 || cg == 16, "smot_xcorr_planar: channel group %d (0 = flat, 2, 4, 8 or 16)", cg);
  SMOT_CHECK_ARG(n >= 0 && channels > 0 && channels % (cg ? cg : 4) == 0,
                 "smot_xcorr_planar: bad geometry n=%d C=%d (C must be a multiple of %d)", n, channels, cg ? cg : 4);
  if (n == 0) return SMOT_OK;
  SMOT_CHECK_ARG(x_planar && k && out, "smot_xcorr_planar: null argument");
  SMOT_CHECK_ARG((((uintptr_t)x_planar | (uintptr_t)k | (uintptr_t)out) & 15) == 0, "smot_xcorr_planar: operands must be 16-byte aligned");
  static_assert(XM_CSTRIDE == SMOT_XCORR_PLANE && XM_PITCH == SMOT_XCORR_ROW_PITCH, "smot.h states the plane layout");
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e;
  if (cg == 0) {   // flat form: one CTA per SM, 4-plane units dealt evenly
    const int units = n * channels / 4, sms = sm_count();
    SMOT_CHECK_ARG(units <= XF_MAX_UNITS * sms, "smot_xcorr_planar: %d planes do not fit one wave of the flat form (%d SMs x %d)",
                   n * channels, sms, XF_MAX_PLANES);
    const int grid = units < sms ? units : sms;
    if (mma_mode == 1) {
      SMOT_ENSURE_SMEM(xcorr_flat_kernel<1>, XF_SMEM, "smot_xcorr_planar");
      e = launch_pdl(xcorr_flat_kernel<1>, dim3(grid), dim3(XF_THREADS), XF_SMEM, st, (const __half*)x_planar, (const __half*)k,
                     (__half*)out, channels, units);
    } else {
      SMOT_ENSURE_SMEM(xcorr_flat_kernel<0>, XF_SMEM, "smot_xcorr_planar");
      e = launch_pdl(xcorr_flat_kernel<0>, dim3(grid), dim3(XF_THREADS), XF_SMEM, st, (const __half*)x_planar, (const __half*)k,
                     (__half*)out, channels, units);
    }
    if (e != cudaSuccess) {
      set_error("smot_xcorr_planar: launch failed: %s", cudaGetErrorString(e));
      return SMOT_ERR_CUDA;
    }
    SMOT_CHECK_LAUNCH("smot_xcorr_planar(flat)");
    return SMOT_OK;
  }
#define SMOT_XP_CASE(MODE, CGV) \
  case (MODE) * 32 + (CGV): e = launch_xcorr_planar<MODE, CGV>(x_planar, k, out, n, channels, st); break
  switch (mma_mode * 32 + cg) {
    SMOT_XP_CASE(0, 2); SMOT_XP_CASE(0, 4); SMOT_XP_CASE(0, 8); SMOT_XP_CASE(0, 16);
    SMOT_XP_CASE(1, 2); SMOT_XP_CASE(1, 4); SMOT_XP_CASE(1, 8); SMOT_XP_CASE(1, 16);
    default: e = cudaErrorInvalidValue;
  }
#undef SMOT_XP_CASE
  if (e != cudaSuccess) {
    set_error("smot_xcorr_planar: launch failed: %s", cudaGetErrorString(e));
    return SMOT_ERR_CUDA;
  }
  SMOT_CHECK_LAUNCH("smot_xcorr_planar");
  return SMOT_OK;
}

extern "C" int smot_emm_decode(const float* maps, int map_ld, int n, int O, int up, int T, const float* sr,
                               const float* tboxes, const float* hann, float pad, int use_centerness, double sigma,
                               int img_w, int img_h, int amodal, float* out_boxes, float* out_conf, int* out_valid,
                               void* scratch, void* stream) {
  SMOT_CHECK_ARG(n >= 0 && O >= 1 && up >= 1 && T >= 1 && map_ld >= EMM_CH, "smot_emm_decode: bad arguments");
  if (n == 0) return SMOT_OK;
  SMOT_CHECK_ARG(maps && sr && tboxes && hann && out_boxes && out_conf && out_valid && scratch, "smot_emm_decode: null argument");
  const int OW = O * up;
  SMOT_CHECK_ARG(up <= EMM_MAX_BAND, "smot_emm_decode: upsampling factor %d > %d", up, EMM_MAX_BAND);
  const int rows_per_cta = up;                        // one source-row period per band
  const int rows_max = min(O, rows_per_cta / up + 4);  // source rows a band can touch (4 taps)
  const size_t smem = ((size_t)O * O * EMM_CH + (size_t)EMM_CH * rows_max * OW) * sizeof(float);
  SMOT_CHECK_ARG(smem <= 200 * 1024, "smot_emm_decode: response map %dx%d (x%d) does not fit shared memory", O, O, up);
  cudaStream_t st = (cudaStream_t)stream;
  SMOT_ENSURE_SMEM(emm_score_kernel, smem, "smot_emm_decode");
  DecodeArgs a;
  a.maps = maps, a.map_ld = map_ld, a.n = n, a.O = O, a.up = up, a.T = T, a.sr = sr, a.tboxes = tboxes, a.hann = hann;
  a.pad = pad, a.use_centerness = use_centerness, a.sigma = (float)sigma, a.one_minus_sigma = (float)(1.0 - sigma), a.img_w = img_w, a.img_h = img_h, a.amodal = amodal;
  a.rows_per_cta = rows_per_cta, a.rows_max = rows_max;
  a.best = (unsigned long long*)scratch;
  a.out_boxes = out_boxes, a.out_conf = out_conf, a.out_valid = out_valid;
  cudaError_t e = cudaMemsetAsync(scratch, 0, (size_t)n * 8, st);
  if (e != cudaSuccess) {
    set_error("smot_emm_decode: memset: %s", cudaGetErrorString(e));
    return SMOT_ERR_CUDA;
  }
  emm_score_kernel<<<dim3((OW + a.rows_per_cta - 1) / a.rows_per_cta, n), 256, smem, st>>>(a);
  SMOT_CHECK_LAUNCH("smot_emm_decode(score)");
  emm_finalize_kernel<<<(n + 63) / 64, 64, 0, st>>>(a);
  SMOT_CHECK_LAUNCH("smot_emm_decode(finalize)");
  return SMOT_OK;
}
