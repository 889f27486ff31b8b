// High-resolution, low-channel convolutions of the DLA-34 stem (fp16 storage, fp32 accumulation):
//   base_layer 7x7 3->16, level0 3x3 16->16, level1 3x3/2 16->32, level2.tree1.conv1 3x3/2 32->64
//   (dla.py:257-260,278-287,34-38).  They hold ~10 % of the FLOPs but ~35 % of the activation bytes: at
//   704x1280 each reads or writes 14-29 MB and their GEMM N (16..64) and K (147..288) are far too small
//   for a 128-wide wgmma tile, so the bound is HBM, not the tensor pipe.
// Design: a CTA stages the input halo of an 8x32 (stride 1) or 4x32 (stride 2) output tile ONCE in
// shared memory (cp.async, zero-fill outside the image = the conv padding) plus the whole weight,
// every warp then walks the filter taps with warp-level mma.sync.m16n8k16 (A fragments via ldmatrix
// straight out of the halo, pixel pitch padded by 16 B against bank conflicts), and the fp16 result is
// staged back through shared memory so global stores are full 16-byte, pixel-contiguous chunks.
#include "common.cuh"

namespace smot {

struct HiresArgs {
  const __half* in;
  const __half* wt;
  const float* scale;
  const float* bias;
  __half* out;
  int H, W, in_ld, OH, OW, out_ld, relu;
};

__device__ __forceinline__ uint32_t hs_smem(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cp_async16(void* dst, const void* src, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(hs_smem(dst)), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async8(void* dst, const void* src, bool valid) {
  const int sz = valid ? 8 : 0;
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(hs_smem(dst)), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void mma_16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// ---------------------------------------------------------------------------------------------
// 3x3, pad 1, stride 1|2, CIN in {16,32}, COUT in {16,32,64}
// ---------------------------------------------------------------------------------------------
template <int CIN, int COUT, int STRIDE>
struct Hires3 {
  static constexpr int TW = 32;
  static constexpr int TH = STRIDE == 1 ? 8 : 4;
  static constexpr int MT = STRIDE == 1 ? 2 : 1;  // 16-pixel M tiles per warp (8 warps)
  static constexpr int IH = (TH - 1) * STRIDE + 3, IW = (TW - 1) * STRIDE + 3;
  static constexpr int PITCH = CIN * 2 + 16;      // bytes per halo pixel (16 B pad)
  static constexpr int K = 9 * CIN, KP = K + 8;   // weight row pitch in halves (16 B pad)
  static constexpr int HALO_BYTES = ((IH * IW * PITCH + 127) / 128) * 128;
  static constexpr int W_BYTES = COUT * KP * 2;
  static constexpr int OUT_BYTES = TH * TW * COUT * 2;
  static constexpr int SMEM = HALO_BYTES + W_BYTES;
  static_assert(OUT_BYTES <= HALO_BYTES, "output staging reuses the halo region");
};

template <int CIN, int COUT, int STRIDE>
__global__ void __launch_bounds__(256) conv3x3_hires_kernel(const HiresArgs a) {
  using C = Hires3<CIN, COUT, STRIDE>;
  extern __shared__ __align__(128) unsigned char hs_raw[];
  unsigned char* halo = hs_raw;
  __half* wsm = reinterpret_cast<__half*>(hs_raw + C::HALO_BYTES);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int ox0 = blockIdx.x * C::TW, oy0 = blockIdx.y * C::TH;
  const int img = blockIdx.z;
  const __half* in = a.in + (size_t)img * a.H * a.W * a.in_ld;
  const int ix0 = ox0 * STRIDE - 1, iy0 = oy0 * STRIDE - 1;
  // ---- stage weights [COUT][K] -> [COUT][KP] and the input halo (zero-filled outside the image)
  pdl_launch_dependents();
  constexpr int WCH = C::K / 8;  // 16-byte chunks per weight row
  for (int i = tid; i < COUT * WCH; i += 256) {
    const int n = i / WCH, q = i - n * WCH;
    cp_async16(wsm + n * C::KP + q * 8, a.wt + (size_t)n * C::K + q * 8, true);
  }
  pdl_wait();  // the weights are constants; the input belongs to the previous kernel
  constexpr int PCH = CIN / 8;  // 16-byte chunks per pixel
  for (int i = tid; i < C::IH * C::IW * PCH; i += 256) {
    const int p = i / PCH, q = i - p * PCH;
    const int py = p / C::IW, px = p - py * C::IW;
    const int gy = iy0 + py, gx = ix0 + px;
    const bool ok = gy >= 0 && gy < a.H && gx >= 0 && gx < a.W;
    const __half* src = ok ? in + ((size_t)gy * a.W + gx) * a.in_ld + q * 8 : in;
    cp_async16(halo + p * C::PITCH + q * 16, src, ok);
  }
  cp_async_wait_all();
  __syncthreads();

  // ---- warp tiling: stride 1: warp = output row, 2 M-tiles; stride 2: warp -> (row, half)
  const int oy_l = STRIDE == 1 ? warp : (warp >> 1);
  const int mt0 = STRIDE == 1 ? 0 : (warp & 1);
  float acc[C::MT][COUT / 8][4];
#pragma unroll
  for (int m = 0; m < C::MT; ++m)
#pragma unroll
    for (int j = 0; j < COUT / 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[m][j][e] = 0.f;
  // ldmatrix lane roles
  const int a_row = (lane & 7) + ((lane >> 3) & 1) * 8;  // A: matrices (r0-7,k0-7),(r8-15,k0-7),(r0-7,k8-15),(r8-15,k8-15)
  const int a_kh = lane >> 4;
  const int b_row = (lane & 7) + ((lane >> 4) & 1) * 8;  // B: matrices (n0-7,k0-7),(n0-7,k8-15),(n8-15,k0-7),(n8-15,k8-15)
  const int b_kh = (lane >> 3) & 1;
  const uint32_t halo_s = hs_smem(halo), w_s = hs_smem(wsm);
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int s = 0; s < 3; ++s)
#pragma unroll
      for (int kc = 0; kc < CIN / 16; ++kc) {
        uint32_t af[C::MT][4];
#pragma unroll
        for (int m = 0; m < C::MT; ++m) {
          const int iy = oy_l * STRIDE + r;
          const int ix = ((mt0 + m) * 16 + a_row) * STRIDE + s;
          ldmatrix_x4(halo_s + (iy * C::IW + ix) * C::PITCH + kc * 32 + a_kh * 16, af[m][0], af[m][1], af[m][2], af[m][3]);
        }
        const int kbase = (r * 3 + s) * CIN + kc * 16;
#pragma unroll
        for (int jp = 0; jp < COUT / 16; ++jp) {
          uint32_t b0, b1, b2, b3;
          ldmatrix_x4(w_s + ((jp * 16 + b_row) * C::KP + kbase + b_kh * 8) * 2, b0, b1, b2, b3);
#pragma unroll
          for (int m = 0; m < C::MT; ++m) {
            mma_16816(acc[m][jp * 2], af[m], b0, b1);
            mma_16816(acc[m][jp * 2 + 1], af[m], b2, b3);
          }
        }
      }
  __syncthreads();  // everyone is done reading the halo: reuse it as the output staging tile
  __half* ost = reinterpret_cast<__half*>(halo);
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int m = 0; m < C::MT; ++m)
#pragma unroll
    for (int j = 0; j < COUT / 8; ++j) {
      const int n = j * 8 + 2 * t;
      const float s0 = a.scale ? a.scale[n] : 1.f, s1 = a.scale ? a.scale[n + 1] : 1.f;
      const float c0 = a.bias ? a.bias[n] : 0.f, c1 = a.bias ? a.bias[n + 1] : 0.f;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int ox_l = (mt0 + m) * 16 + g + h * 8;
        float v0 = __fadd_rn(__fmul_rn(acc[m][j][2 * h], s0), c0);
        float v1 = __fadd_rn(__fmul_rn(acc[m][j][2 * h + 1], s1), c1);
        if (a.relu) v0 = fmaxf(v0, 0.f), v1 = fmaxf(v1, 0.f);
        *reinterpret_cast<__half2*>(ost + (oy_l * C::TW + ox_l) * COUT + n) = __floats2half2_rn(v0, v1);
      }
    }
  __syncthreads();
  constexpr int OCH = COUT / 8;  // 16-byte chunks per output pixel
  __half* out = a.out + (size_t)img * a.OH * a.OW * a.out_ld;
  for (int i = tid; i < C::TH * C::TW * OCH; i += 256) {
    const int p = i / OCH, q = i - p * OCH;
    const int py = p / C::TW, px = p - py * C::TW;
    const int oy = oy0 + py, ox = ox0 + px;
    if (oy < a.OH && ox < a.OW)
      *reinterpret_cast<uint4*>(out + ((size_t)oy * a.OW + ox) * a.out_ld + q * 8) =
          *reinterpret_cast<const uint4*>(ost + p * COUT + q * 8);
  }
}

// ---------------------------------------------------------------------------------------------
// stem: 7x7, pad 3, stride 1, 3 (stored as 4) -> 16 channels.  K per filter row = 8 pixels x 4 ch = 32
// (the 8th pixel and the 4th channel meet zero weights), i.e. 14 k-steps of m16n8k16.
// ---------------------------------------------------------------------------------------------
constexpr int ST_TW = 32, ST_TH = 8, ST_IH = ST_TH + 6, ST_IW = 40, ST_COUT = 16;

__global__ void __launch_bounds__(256) stem7x7_hires_kernel(const HiresArgs a) {
  __shared__ __align__(16) __half halo[ST_IH * ST_IW * 4];       // 8 B per pixel
  __shared__ __align__(16) __half wsm[ST_COUT * 7 * 32];         // [cout][r][(s*4 + c)], zero padded
  __shared__ __align__(16) __half ost[ST_TH * ST_TW * ST_COUT];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int ox0 = blockIdx.x * ST_TW, oy0 = blockIdx.y * ST_TH;
  const __half* in = a.in + (size_t)blockIdx.z * a.H * a.W * a.in_ld;
  pdl_launch_dependents();
  for (int i = tid; i < ST_COUT * 7 * 32; i += 256) {
    const int n = i / 224, rem = i - n * 224, r = rem / 32, k = rem - r * 32;
    const int s = k >> 2, c = k & 3;
    wsm[i] = (s < 7 && c < 3) ? a.wt[((size_t)n * 49 + r * 7 + s) * 3 + c] : __float2half(0.f);
  }
  pdl_wait();
  for (int p = tid; p < ST_IH * ST_IW; p += 256) {
    const int py = p / ST_IW, px = p - py * ST_IW;
    const int gy = oy0 - 3 + py, gx = ox0 - 3 + px;
    const bool ok = gy >= 0 && gy < a.H && gx >= 0 && gx < a.W;
    cp_async8(halo + p * 4, ok ? in + ((size_t)gy * a.W + gx) * a.in_ld : in, ok);
  }
  cp_async_wait_all();
  __syncthreads();
  const int g = lane >> 2, t = lane & 3;
  float acc[2][2][4];
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[m][j][e] = 0.f;
  const uint32_t* hw = reinterpret_cast<const uint32_t*>(halo);  // 2 words per pixel
  const uint32_t* ww = reinterpret_cast<const uint32_t*>(wsm);   // 16 words per (cout, r)
#pragma unroll
  for (int r = 0; r < 7; ++r)
#pragma unroll
    for (int kb = 0; kb < 2; ++kb) {
      uint32_t bf[2][2];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int base = ((j * 8 + g) * 7 + r) * 16 + kb * 8 + t;
        bf[j][0] = ww[base];
        bf[j][1] = ww[base + 4];
      }
#pragma unroll
      for (int m = 0; m < 2; ++m) {
        // A(row i, k) = halo[(warp + r) row][(m*16 + i) pixel + k/4][k%4]: word index = pixel*2 + k/2
        const int rowbase = ((warp + r) * ST_IW + m * 16) * 2 + kb * 8 + t;
        uint32_t af[4];
        af[0] = hw[rowbase + g * 2];
        af[1] = hw[rowbase + (g + 8) * 2];
        af[2] = hw[rowbase + g * 2 + 4];
        af[3] = hw[rowbase + (g + 8) * 2 + 4];
        mma_16816(acc[m][0], af, bf[0][0], bf[0][1]);
        mma_16816(acc[m][1], af, bf[1][0], bf[1][1]);
      }
    }
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int n = j * 8 + 2 * t;
      const float s0 = a.scale ? a.scale[n] : 1.f, s1 = a.scale ? a.scale[n + 1] : 1.f;
      const float c0 = a.bias ? a.bias[n] : 0.f, c1 = a.bias ? a.bias[n + 1] : 0.f;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int ox_l = m * 16 + g + h * 8;
        float v0 = __fadd_rn(__fmul_rn(acc[m][j][2 * h], s0), c0);
        float v1 = __fadd_rn(__fmul_rn(acc[m][j][2 * h + 1], s1), c1);
        if (a.relu) v0 = fmaxf(v0, 0.f), v1 = fmaxf(v1, 0.f);
        *reinterpret_cast<__half2*>(ost + (warp * ST_TW + ox_l) * ST_COUT + n) = __floats2half2_rn(v0, v1);
      }
    }
  __syncthreads();
  __half* out = a.out + (size_t)blockIdx.z * a.OH * a.OW * a.out_ld;
  for (int i = tid; i < ST_TH * ST_TW * 2; i += 256) {
    const int p = i >> 1, q = i & 1;
    const int py = p / ST_TW, px = p - py * ST_TW;
    const int oy = oy0 + py, ox = ox0 + px;
    if (oy < a.OH && ox < a.OW)
      *reinterpret_cast<uint4*>(out + ((size_t)oy * a.OW + ox) * a.out_ld + q * 8) =
          *reinterpret_cast<const uint4*>(ost + p * ST_COUT + q * 8);
  }
}

// ---------------------------------------------------------------------------------------------
// Persistent forms of the two stride-1 layers (stem 7x7 3->16, level0 3x3 16->16), the widest maps of the network.
//
// The kernels above re-stage the weights in every one of 3520 CTAs and fetch every A fragment once per filter row it meets:
// per warp-tile 170 (stem) / 27 (level0) shared-memory instructions for 56 / 36 MMAs, which is what bounds them (ncu, round 2:
// 58.6 / 32.3 us against MMA floors of 11 / 7 us and HBM floors of 5.5 / 8.9 us).  Here
//   * one CTA per SM walks 32x32-pixel output tiles; the input halo of tile i+1 arrives by cp.async under the MMAs of tile i
//     (two halo buffers, one block barrier per tile);
//   * the weights live in REGISTERS as ready-made B fragments for the whole kernel (56 / 36 registers), scale / bias likewise;
//   * a warp owns FOUR output rows: the fragments of input row y are loaded once and meet every (output row, filter row) pair
//     they belong to -- 10 / 6 row loads instead of 28 / 12;
//   * the result leaves through a per-warp staging row (no block barrier): 16-byte stores, one output row = one contiguous KB.
// Every output accumulates its taps in the order of the kernels above (filter row, then k chunk / tap), so the results are
// bit-identical to theirs.
// Measured and dropped: hoisting the per-thread halo offsets out of the tile loop (one register per copy, interior tiles
// without bounds tests).  Fewer instructions, but the enumeration that makes the shared-memory offset implicit leaves every
// third lane idle, so a warp's cp.async covers fewer contiguous bytes: level0 26.0 -> 28.5 us, level1 18.7 -> 20.6 us.
// ---------------------------------------------------------------------------------------------
constexpr int HP_TW = 32, HP_TH = 32, HP_ROWS = 4;     // tile, output rows per warp (8 warps)
constexpr int HP_OPITCH = 24;                          // halves per staged output pixel (16 + 8: conflict-free fragment stores)

// fragment (16 pixels x 16 channels as two n8 halves) -> warp-private staging row -> 16-byte global stores
__device__ __forceinline__ void hp_store_row(__half* ost_w, const float (*acc)[2][4], const float* sc, const float* bi, int relu,
                                             __half* out_row, int out_ld, int ox0, int OW, int lane) {
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float v0 = __fadd_rn(__fmul_rn(acc[m][j][2 * h], sc[j * 2]), bi[j * 2]);
        float v1 = __fadd_rn(__fmul_rn(acc[m][j][2 * h + 1], sc[j * 2 + 1]), bi[j * 2 + 1]);
        if (relu) v0 = fmaxf(v0, 0.f), v1 = fmaxf(v1, 0.f);
        *reinterpret_cast<__half2*>(ost_w + (m * 16 + g + h * 8) * HP_OPITCH + j * 8 + 2 * t) = __floats2half2_rn(v0, v1);
      }
  __syncwarp();
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int c = i * 32 + lane, px = c >> 1, q = c & 1;
    if (ox0 + px < OW)
      *reinterpret_cast<uint4*>(out_row + (size_t)px * out_ld + q * 8) = *reinterpret_cast<const uint4*>(ost_w + px * HP_OPITCH + q * 8);
  }
  __syncwarp();
}

// stem: halo = (32 + 6) rows x 40 pixels x 4 halves, origin (oy0 - 3, ox0 - 4) so that every 16-byte chunk (2 pixels) is
// aligned and lies entirely inside or outside the image (W even)
constexpr int SP_IH = HP_TH + 6, SP_IW = 40;
constexpr int SP_HALO = SP_IH * SP_IW * 4;             // halves per buffer
constexpr int SP_SMEM = (2 * SP_HALO + 8 * 32 * HP_OPITCH) * 2;

__global__ void __launch_bounds__(256, 1) stem7x7_persist_kernel(const HiresArgs a, int tiles_x, int tiles_y, int ntiles) {
  extern __shared__ __align__(128) unsigned char hp_raw[];
  __half* halo = reinterpret_cast<__half*>(hp_raw);                 // [2][SP_IH][SP_IW][4]
  __half* ost = halo + 2 * SP_HALO;                                 // [8 warps][32][HP_OPITCH]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  pdl_launch_dependents();
  // ---- constants to registers: B fragments of all 7 filter rows x 2 k-chunks x 2 channel halves
  // k = s * 4 + c (filter column s, input channel c); s = 7 and c = 3 meet zeros
  uint32_t bw[7][2][2][2];
#pragma unroll
  for (int r = 0; r < 7; ++r)
#pragma unroll
    for (int kb = 0; kb < 2; ++kb)
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int k = kb * 16 + hh * 8 + 2 * t, sx = k >> 2, c = k & 3, n = j * 8 + g;   // (k, k+1) = channels (c, c+1) of column sx
          const __half* w = a.wt + ((size_t)n * 49 + r * 7 + sx) * 3;
          const __half z = __float2half(0.f);
          const __half lo = sx < 7 ? w[c] : z, hi = (sx < 7 && c == 0) ? w[1] : z;        // c is 0 or 2; channel 3 does not exist
          bw[r][kb][j][hh] = (uint32_t)__half_as_ushort(lo) | ((uint32_t)__half_as_ushort(hi) << 16);
        }
  float sc[4], bi[4];
#pragma unroll
  for (int j = 0; j < 2; ++j)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int n = j * 8 + 2 * t + e;
      sc[j * 2 + e] = a.scale ? a.scale[n] : 1.f, bi[j * 2 + e] = a.bias ? a.bias[n] : 0.f;
    }
  pdl_wait();  // the weights are constants; the input belongs to the previous kernel
  const int per_img = tiles_x * tiles_y;
  auto load_halo = [&](int tile, int buf) {
    const int img = tile / per_img, rem = tile - img * per_img, ty = rem / tiles_x, tx = rem - ty * tiles_x;
    const __half* in = a.in + (size_t)img * a.H * a.W * 4;
    const int iy0 = ty * HP_TH - 3, ix0 = tx * HP_TW - 4;
    __half* dst = halo + buf * SP_HALO;
    for (int i = tid; i < SP_IH * (SP_IW / 2); i += 256) {
      const int py = i / (SP_IW / 2), pc = i - py * (SP_IW / 2);
      const int gy = iy0 + py, gx = ix0 + pc * 2;
      const bool ok = gy >= 0 && gy < a.H && gx >= 0 && gx < a.W;
      cp_async16(dst + (py * SP_IW + pc * 2) * 4, ok ? in + ((size_t)gy * a.W + gx) * 4 : in, ok);
    }
  };
  int tile = blockIdx.x, cur = 0;
  if (tile < ntiles) load_halo(tile, 0);
  for (; tile < ntiles; tile += gridDim.x, cur ^= 1) {
    cp_async_wait_all();
    __syncthreads();  // this tile's halo is complete for every thread; everyone is done with the other buffer
    if (tile + (int)gridDim.x < ntiles) load_halo(tile + gridDim.x, cur ^ 1);
    const uint32_t* hw = reinterpret_cast<const uint32_t*>(halo + cur * SP_HALO);  // 2 words per pixel
    float acc[HP_ROWS][2][2][4];
#pragma unroll
    for (int y = 0; y < HP_ROWS; ++y)
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[y][m][j][e] = 0.f;
#pragma unroll
    for (int rho = 0; rho < HP_ROWS + 6; ++rho)      // input row warp*4 + rho of the halo
#pragma unroll
      for (int kb = 0; kb < 2; ++kb) {
        uint32_t af[2][4];
#pragma unroll
        for (int m = 0; m < 2; ++m) {
          // A(row i, k) = halo[row][pixel 1 + m*16 + i + k/4][k%4]: word = pixel * 2 + k / 2   (+1: the halo starts at ox0 - 4)
          const int base = ((warp * HP_ROWS + rho) * SP_IW + 1 + m * 16) * 2 + kb * 8 + t;
          af[m][0] = hw[base + g * 2];
          af[m][1] = hw[base + (g + 8) * 2];
          af[m][2] = hw[base + g * 2 + 4];
          af[m][3] = hw[base + (g + 8) * 2 + 4];
        }
#pragma unroll
        for (int y = 0; y < HP_ROWS; ++y) {
          const int r = rho - y;
          if (r >= 0 && r < 7) {
#pragma unroll
            for (int m = 0; m < 2; ++m) {
              mma_16816(acc[y][m][0], af[m], bw[r][kb][0][0], bw[r][kb][0][1]);
              mma_16816(acc[y][m][1], af[m], bw[r][kb][1][0], bw[r][kb][1][1]);
            }
          }
        }
      }
    const int img = tile / per_img, rem = tile - img * per_img, ty = rem / tiles_x, tx = rem - ty * tiles_x;
    __half* out = a.out + (size_t)img * a.OH * a.OW * a.out_ld;
#pragma unroll
    for (int y = 0; y < HP_ROWS; ++y) {
      const int oy = ty * HP_TH + warp * HP_ROWS + y;
      if (oy < a.OH)
        hp_store_row(ost + warp * 32 * HP_OPITCH, acc[y], sc, bi, a.relu, out + ((size_t)oy * a.OW + tx * HP_TW) * a.out_ld, a.out_ld,
                     tx * HP_TW, a.OW, lane);
    }
  }
}

// level0: 3x3, pad 1, stride 1, 16 -> 16.  Halo = 34 x 34 pixels, 48 B per pixel (32 + 16 pad: conflict-free ldmatrix).
constexpr int L0_IH = HP_TH + 2, L0_IW = HP_TW + 2, L0_PITCH = 48;
constexpr int L0_HALO = L0_IH * L0_IW * L0_PITCH;      // bytes per buffer
constexpr int L0_SMEM = 2 * L0_HALO + 8 * 32 * HP_OPITCH * 2;

__global__ void __launch_bounds__(256, 1) conv3x3_c16_persist_kernel(const HiresArgs a, int tiles_x, int tiles_y, int ntiles) {
  extern __shared__ __align__(128) unsigned char hp_raw[];
  unsigned char* halo = hp_raw;                                                  // [2][L0_IH][L0_IW][L0_PITCH]
  __half* ost = reinterpret_cast<__half*>(hp_raw + 2 * L0_HALO);                 // [8 warps][32][HP_OPITCH]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  pdl_launch_dependents();
  // B fragments of the 9 taps: b0 = W[n = j*8 + g][tap][2t, 2t+1], b1 = ...[2t+8, 2t+9]   (weights [16][3][3][16])
  uint32_t bw[9][2][2];
#pragma unroll
  for (int tap = 0; tap < 9; ++tap)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
        bw[tap][j][hh] = *reinterpret_cast<const uint32_t*>(a.wt + ((size_t)(j * 8 + g) * 9 + tap) * 16 + hh * 8 + 2 * t);
  float sc[4], bi[4];
#pragma unroll
  for (int j = 0; j < 2; ++j)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int n = j * 8 + 2 * t + e;
      sc[j * 2 + e] = a.scale ? a.scale[n] : 1.f, bi[j * 2 + e] = a.bias ? a.bias[n] : 0.f;
    }
  pdl_wait();
  const int per_img = tiles_x * tiles_y;
  auto load_halo = [&](int tile, int buf) {
    const int img = tile / per_img, rem = tile - img * per_img, ty = rem / tiles_x, tx = rem - ty * tiles_x;
    const __half* in = a.in + (size_t)img * a.H * a.W * a.in_ld;
    const int iy0 = ty * HP_TH - 1, ix0 = tx * HP_TW - 1;
    unsigned char* dst = halo + buf * L0_HALO;
    for (int i = tid; i < L0_IH * L0_IW * 2; i += 256) {
      const int p = i >> 1, q = i & 1;
      const int py = p / L0_IW, px = p - py * L0_IW;
      const int gy = iy0 + py, gx = ix0 + px;
      const bool ok = gy >= 0 && gy < a.H && gx >= 0 && gx < a.W;
      cp_async16(dst + p * L0_PITCH + q * 16, ok ? in + ((size_t)gy * a.W + gx) * a.in_ld + q * 8 : in, ok);
    }
  };
  const int a_row = (lane & 7) + ((lane >> 3) & 1) * 8, a_kh = lane >> 4;
  int tile = blockIdx.x, cur = 0;
  if (tile < ntiles) load_halo(tile, 0);
  for (; tile < ntiles; tile += gridDim.x, cur ^= 1) {
    cp_async_wait_all();
    __syncthreads();
    if (tile + (int)gridDim.x < ntiles) load_halo(tile + gridDim.x, cur ^ 1);
    const uint32_t halo_s = hs_smem(halo + cur * L0_HALO);
    float acc[HP_ROWS][2][2][4];
#pragma unroll
    for (int y = 0; y < HP_ROWS; ++y)
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[y][m][j][e] = 0.f;
#pragma unroll
    for (int rho = 0; rho < HP_ROWS + 2; ++rho)
#pragma unroll
      for (int sx = 0; sx < 3; ++sx) {
        uint32_t af[2][4];
#pragma unroll
        for (int m = 0; m < 2; ++m)
          ldmatrix_x4(halo_s + (((warp * HP_ROWS + rho) * L0_IW + m * 16 + a_row + sx) * L0_PITCH) + a_kh * 16, af[m][0], af[m][1], af[m][2],
                      af[m][3]);
#pragma unroll
        for (int y = 0; y < HP_ROWS; ++y) {
          const int r = rho - y;
          if (r >= 0 && r < 3) {
#pragma unroll
            for (int m = 0; m < 2; ++m) {
              mma_16816(acc[y][m][0], af[m], bw[r * 3 + sx][0][0], bw[r * 3 + sx][0][1]);
              mma_16816(acc[y][m][1], af[m], bw[r * 3 + sx][1][0], bw[r * 3 + sx][1][1]);
            }
          }
        }
      }
    const int img = tile / per_img, rem = tile - img * per_img, ty = rem / tiles_x, tx = rem - ty * tiles_x;
    __half* out = a.out + (size_t)img * a.OH * a.OW * a.out_ld;
#pragma unroll
    for (int y = 0; y < HP_ROWS; ++y) {
      const int oy = ty * HP_TH + warp * HP_ROWS + y;
      if (oy < a.OH)
        hp_store_row(ost + warp * 32 * HP_OPITCH, acc[y], sc, bi, a.relu, out + ((size_t)oy * a.OW + tx * HP_TW) * a.out_ld, a.out_ld,
                     tx * HP_TW, a.OW, lane);
    }
  }
}

// level1 (16 -> 32) and level2.tree1.conv1 (32 -> 64): 3x3, pad 1, STRIDE 2.  Adjacent output rows share one input row in
// three, so there is no fragment reuse to gain; what the persistent form removes is the per-CTA weight staging and the B-operand
// ldmatrix traffic (2 of the 3 shared-memory instructions per MMA pair): weights as register-resident B fragments (72 / 144
// registers; for 64 output channels two warps split them), double-buffered halo, per-warp result staging.  Tile = (8 / NW) output
// rows x 32 columns, warp = (row, 32-channel slice).  Same accumulation order as conv3x3_hires_kernel: bit-identical.
template <int CIN, int COUT>
struct S2Persist {
  static constexpr int NW = COUT / 32;                 // warps along the output channels
  static constexpr int TH = 8 / NW, TW = 32;
  static constexpr int IH = (TH - 1) * 2 + 3, IW = (TW - 1) * 2 + 3;
  static constexpr int PITCH = CIN * 2 + 16;           // bytes per halo pixel
  static constexpr int HALO = ((IH * IW * PITCH + 127) / 128) * 128;
  static constexpr int OPITCH = 40;                    // halves per staged pixel of a warp's 32-channel slice
  static constexpr int SMEM = 2 * HALO + 8 * 32 * OPITCH * 2;
  static constexpr int KC = CIN / 16;
  static_assert(COUT == 32 || COUT == 64, "32-channel slices");
};

template <int CIN, int COUT>
__global__ void __launch_bounds__(256, 1) conv3x3_s2_persist_kernel(const HiresArgs a, int tiles_x, int tiles_y, int ntiles) {
  using C = S2Persist<CIN, COUT>;
  extern __shared__ __align__(128) unsigned char hp_raw[];
  unsigned char* halo = hp_raw;
  __half* ost = reinterpret_cast<__half*>(hp_raw + 2 * C::HALO);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int oy_l = warp / C::NW, nw = warp % C::NW;   // output row of the tile, 32-channel slice
  pdl_launch_dependents();
  uint32_t bw[9][C::KC][4][2];
#pragma unroll
  for (int tap = 0; tap < 9; ++tap)
#pragma unroll
    for (int kc = 0; kc < C::KC; ++kc)
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
          bw[tap][kc][j][hh] =
              *reinterpret_cast<const uint32_t*>(a.wt + ((size_t)(nw * 32 + j * 8 + g) * 9 + tap) * CIN + kc * 16 + hh * 8 + 2 * t);
  float sc[8], bi[8];
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int n = nw * 32 + j * 8 + 2 * t + e;
      sc[j * 2 + e] = a.scale ? a.scale[n] : 1.f, bi[j * 2 + e] = a.bias ? a.bias[n] : 0.f;
    }
  pdl_wait();
  const int per_img = tiles_x * tiles_y;
  auto load_halo = [&](int tile, int buf) {
    const int img = tile / per_img, rem = tile - img * per_img, ty = rem / tiles_x, tx = rem - ty * tiles_x;
    const __half* in = a.in + (size_t)img * a.H * a.W * a.in_ld;
    const int iy0 = ty * C::TH * 2 - 1, ix0 = tx * C::TW * 2 - 1;
    unsigned char* dst = halo + buf * C::HALO;
    constexpr int PCH = CIN / 8;
    for (int i = tid; i < C::IH * C::IW * PCH; i += 256) {
      const int p = i / PCH, q = i - p * PCH;
      const int py = p / C::IW, px = p - py * C::IW;
      const int gy = iy0 + py, gx = ix0 + px;
      const bool ok = gy >= 0 && gy < a.H && gx >= 0 && gx < a.W;
      cp_async16(dst + p * C::PITCH + q * 16, ok ? in + ((size_t)gy * a.W + gx) * a.in_ld + q * 8 : in, ok);
    }
  };
  const int a_row = (lane & 7) + ((lane >> 3) & 1) * 8, a_kh = lane >> 4;
  __half* ost_w = ost + warp * 32 * C::OPITCH;
  int tile = blockIdx.x, cur = 0;
  if (tile < ntiles) load_halo(tile, 0);
  for (; tile < ntiles; tile += gridDim.x, cur ^= 1) {
    cp_async_wait_all();
    __syncthreads();
    if (tile + (int)gridDim.x < ntiles) load_halo(tile + gridDim.x, cur ^ 1);
    const uint32_t halo_s = hs_smem(halo + cur * C::HALO);
    float acc[2][4][4];
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[m][j][e] = 0.f;
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int sx = 0; sx < 3; ++sx)
#pragma unroll
        for (int kc = 0; kc < C::KC; ++kc) {
          uint32_t af[2][4];
#pragma unroll
          for (int m = 0; m < 2; ++m)
            ldmatrix_x4(halo_s + ((oy_l * 2 + r) * C::IW + (m * 16 + a_row) * 2 + sx) * C::PITCH + kc * 32 + a_kh * 16, af[m][0], af[m][1],
                        af[m][2], af[m][3]);
#pragma unroll
          for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int m = 0; m < 2; ++m) mma_16816(acc[m][j], af[m], bw[r * 3 + sx][kc][j][0], bw[r * 3 + sx][kc][j][1]);
        }
    const int img = tile / per_img, rem = tile - img * per_img, ty = rem / tiles_x, tx = rem - ty * tiles_x;
    const int oy = ty * C::TH + oy_l, ox0 = tx * C::TW;
    if (oy < a.OH) {
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float v0 = __fadd_rn(__fmul_rn(acc[m][j][2 * h], sc[j * 2]), bi[j * 2]);
            float v1 = __fadd_rn(__fmul_rn(acc[m][j][2 * h + 1], sc[j * 2 + 1]), bi[j * 2 + 1]);
            if (a.relu) v0 = fmaxf(v0, 0.f), v1 = fmaxf(v1, 0.f);
            *reinterpret_cast<__half2*>(ost_w + (m * 16 + g + h * 8) * C::OPITCH + j * 8 + 2 * t) = __floats2half2_rn(v0, v1);
          }
      __syncwarp();
      __half* out_row = a.out + (((size_t)img * a.OH + oy) * a.OW + ox0) * a.out_ld + nw * 32;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int c = i * 32 + lane, px = c >> 2, q = c & 3;
        if (ox0 + px < a.OW)
          *reinterpret_cast<uint4*>(out_row + (size_t)px * a.out_ld + q * 8) = *reinterpret_cast<const uint4*>(ost_w + px * C::OPITCH + q * 8);
      }
      __syncwarp();
    }
  }
}

// ---- dispatch ---------------------------------------------------------------------------------
static bool common_ok(const smot_conv_desc* d) {
  return d->in_dtype == SMOT_F16 && d->out_dtype == SMOT_F16 && !d->residual && d->out_ld % 8 == 0 &&
         (((uintptr_t)d->in | (uintptr_t)d->weight | (uintptr_t)d->out) & 15) == 0;
}

bool conv2d_hires_supported(const smot_conv_desc* d) {
  if (!common_ok(d)) return false;
  if (d->KH == 7 && d->KW == 7 && d->stride == 1 && d->pad == 3 && d->Cin == 3 && d->in_ld == 4 && d->Cout == 16) return true;
  if (d->KH == 3 && d->KW == 3 && d->pad == 1 && d->in_ld % 8 == 0) {
    if (d->stride == 1 && d->Cin == 16 && d->Cout == 16) return true;
    if (d->stride == 2 && d->Cin == 16 && d->Cout == 32 && d->H % 2 == 0 && d->W % 2 == 0) return true;
    if (d->stride == 2 && d->Cin == 32 && d->Cout == 64 && d->H % 2 == 0 && d->W % 2 == 0) return true;
  }
  return false;
}

template <int CIN, int COUT, int STRIDE>
static int launch3(const HiresArgs& a, int batch, cudaStream_t st) {
  using C = Hires3<CIN, COUT, STRIDE>;
  SMOT_ENSURE_SMEM((conv3x3_hires_kernel<CIN, COUT, STRIDE>), C::SMEM, "smot_conv2d(hires)");
  dim3 grid(ceil_div(a.OW, C::TW), ceil_div(a.OH, C::TH), batch);
  launch_pdl(conv3x3_hires_kernel<CIN, COUT, STRIDE>, grid, dim3(256), C::SMEM, st, a);
  SMOT_CHECK_LAUNCH("smot_conv2d(hires)");
  return SMOT_OK;
}

int conv2d_hires(const smot_conv_desc* d, cudaStream_t st) {
  HiresArgs a;
  a.in = (const __half*)d->in, a.wt = (const __half*)d->weight, a.scale = d->scale, a.bias = d->bias, a.out = (__half*)d->out;
  a.H = d->H, a.W = d->W, a.in_ld = d->in_ld, a.OH = d->OH, a.OW = d->OW, a.out_ld = d->out_ld, a.relu = d->relu;
  if (d->batch == 0) return SMOT_OK;
  // persistent forms (stride-1 layers): when there is at least one 32x32 tile per SM.  SMOT_HIRES_PERSIST=0 keeps the
  // per-tile kernels (A/B; the results are the same bits), =2 takes the persistent ones whatever the size (tests).
  const bool stem = d->KH == 7, c16 = d->KH == 3 && d->stride == 1 && d->Cin == 16 && d->Cout == 16;
  if (stem || c16) {
    const char* e = getenv("SMOT_HIRES_PERSIST");
    const int mode = e ? atoi(e) : 1;
    const int tx = ceil_div(a.OW, HP_TW), ty = ceil_div(a.OH, HP_TH), ntiles = tx * ty * d->batch, sms = sm_count();
    if (mode != 0 && (mode == 2 || ntiles >= sms) && (!stem || a.W % 2 == 0)) {
      const int grid = ntiles < sms ? ntiles : sms;
      if (stem) {
        launch_pdl(stem7x7_persist_kernel, dim3(grid), dim3(256), SP_SMEM, st, a, tx, ty, ntiles);
      } else {
        SMOT_ENSURE_SMEM(conv3x3_c16_persist_kernel, L0_SMEM, "smot_conv2d(hires)");
        launch_pdl(conv3x3_c16_persist_kernel, dim3(grid), dim3(256), L0_SMEM, st, a, tx, ty, ntiles);
      }
      SMOT_CHECK_LAUNCH("smot_conv2d(hires, persistent)");
      return SMOT_OK;
    }
  }
  if (d->KH == 3 && d->stride == 2) {
    const char* e = getenv("SMOT_HIRES_PERSIST");
    const int mode = e ? atoi(e) : 1;
    const bool small = d->Cin == 16;   // 16 -> 32, else 32 -> 64
    const int th = small ? S2Persist<16, 32>::TH : S2Persist<32, 64>::TH;
    const int tx = ceil_div(a.OW, 32), ty = ceil_div(a.OH, th), ntiles = tx * ty * d->batch, sms = sm_count();
    if (mode != 0 && (mode == 2 || ntiles >= sms)) {
      const int grid = ntiles < sms ? ntiles : sms;
      if (small) {
        SMOT_ENSURE_SMEM((conv3x3_s2_persist_kernel<16, 32>), (S2Persist<16, 32>::SMEM), "smot_conv2d(hires)");
        launch_pdl(conv3x3_s2_persist_kernel<16, 32>, dim3(grid), dim3(256), S2Persist<16, 32>::SMEM, st, a, tx, ty, ntiles);
      } else {
        SMOT_ENSURE_SMEM((conv3x3_s2_persist_kernel<32, 64>), (S2Persist<32, 64>::SMEM), "smot_conv2d(hires)");
        launch_pdl(conv3x3_s2_persist_kernel<32, 64>, dim3(grid), dim3(256), S2Persist<32, 64>::SMEM, st, a, tx, ty, ntiles);
      }
      SMOT_CHECK_LAUNCH("smot_conv2d(hires, persistent)");
      return SMOT_OK;
    }
  }
  if (d->KH == 7) {
    dim3 grid(ceil_div(a.OW, ST_TW), ceil_div(a.OH, ST_TH), d->batch);
    launch_pdl(stem7x7_hires_kernel, grid, dim3(256), 0, st, a);
    SMOT_CHECK_LAUNCH("smot_conv2d(stem)");
    return SMOT_OK;
  }
  if (d->Cin == 16 && d->Cout == 16) return launch3<16, 16, 1>(a, d->batch, st);
  if (d->Cin == 16 && d->Cout == 32) return launch3<16, 32, 2>(a, d->batch, st);
  return launch3<32, 64, 2>(a, d->batch, st);
}

}  // namespace smot
