// wgmma / TMA implicit-GEMM convolution for sm_90a (fp16 operands, fp32 accumulation in registers).
//
// GEMM view as in conv_simt.cu: M = output pixels, N = Cout, K = taps * Cin.  One CTA produces a
// 128 (pixels) x BN (channels) output tile; the 128 pixels are a TILE_W x TILE_H patch of one image
// (16x8 for feature maps, 128x1 for matrices), so that for filter tap (r,s) the A operand of the
// tile is ONE 4-D TMA box of the NHWC input at offset (s-pad, r-pad): im2col is never built, and
// the zero padding of the convolution is TMA's out-of-bounds fill.  K advances over
// taps x (Cin/64): each step stages a 128x64 A box and a BNx64 weight box (both 128B-swizzled,
// K-major) in a shared-memory ring fed by one TMA-producer thread.  Two consumer warpgroups own
// 64 rows of the tile each: per step each issues 4 x wgmma.mma_async (M=64, N=BN, K=16) into its
// register accumulator and releases the ring slot of the previous step once that step's wgmma
// group has retired (one group stays in flight).  The same warpgroups then apply
// scale/bias (+residual) (+ReLU) and store fp16 NHWC with an arbitrary channel pitch (so DLA roots
// still read their children without a concat).
//
// Warp roles (288 threads): warps 0..3 and 4..7 = consumer warpgroups 0 and 1 (tile rows 0..63 / 64..127; a
// warpgroup must start at a warp index that is a multiple of 4), warp 8 = TMA producer.
#include <cuda.h>
#include <cudaTypedefs.h>

#include <stdlib.h>
#include <mutex>
#include <string>
#include <unordered_map>

#include "common.cuh"

namespace smot {

constexpr int TC_BM = 128;
constexpr int TC_BK = 64;  // fp16 elements = 128 bytes = one swizzle row
constexpr int TC_CONSUMERS = 256;
constexpr int TC_THREADS = TC_CONSUMERS + 32;
constexpr int TC_PRODUCER_WARP = TC_CONSUMERS / 32;

struct TcArgs {
  const float* scale;
  const float* bias;
  const __half* res;
  __half* out;
  int H, W;          // output (= input, stride 1) spatial size
  int Cin, Cout, out_ld, res_ld, relu;
  int taps, KW, pad, cin_chunks, stride;
  int tiles_w, tiles_h, tile_w, tile_h;
  // split-K (gridDim.z > 1): fp32 partial tiles [z][tile][128][Cout], summed by splitk_reduce_kernel
  int splits, chunks_per_split, num_tiles;
  int cluster_reduce;   // 1: the `splits` CTAs of a tile are one thread-block cluster and finish the tile themselves (no reduce kernel)
  // in-CTA K slices (splits == 1, slices > 1): ONE CTA runs all `slices` K ranges of `chunks_per_split` chunks, each into a
  // fresh register accumulator that is added to a running sum in slice order when the range ends -- the bits of the
  // split-K path without its partial tiles, its reduce kernel and its 8x CTA count
  int slices;
  float* partial;
  unsigned long long* dbg;  // developer timing probe (SMOT_TC_DEBUG): 8 timestamps of CTA (0,0,0), else null
};

// ---- PTX wrappers ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// bounded wait: a mis-programmed pipeline must fail the launch, never hang the GPU.  No printf here: a function call
// inside the consumer loop would make ptxas serialize every wgmma of the kernel.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  for (uint32_t spin = 0; !mbar_try_wait(bar, parity); ++spin)
    if (spin > (1u << 26)) __trap();
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ unsigned long long gtimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
#define TC_STAMP(i)                                                                                   \
  do {                                                                                                \
    if (a.dbg && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) a.dbg[i] = gtimer();          \
  } while (0)

// SM90 shared-memory matrix descriptor: K-major, 128B swizzle, 8-row groups `sbo_bytes` apart (1024 B = dense atoms)
__device__ __forceinline__ uint64_t gmma_desc_sw128(const void* smem, uint32_t sbo_bytes = 1024u, uint32_t base_offset = 0u) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_u32(smem) & 0x3FFFF) >> 4);  // start address
  d |= (uint64_t)1 << 16;                            // leading byte offset (unused: one atom along K)
  d |= (uint64_t)(sbo_bytes >> 4) << 32;             // stride byte offset
  d |= (uint64_t)(base_offset & 7u) << 49;           // swizzle phase of the start address
  d |= (uint64_t)1 << 62;                            // layout type: SWIZZLE_128B
  return d;
}

// wgmma.mma_async m64nNk16, D(f32, registers) = A(f16, smem) * B(f16, smem) (+ D when accum != 0); both operands K-major
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t ad, uint64_t bd, uint32_t accum) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(ad), "l"(bd), "r"(accum));
}
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t ad, uint64_t bd, uint32_t accum) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
      "}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(ad), "l"(bd), "r"(accum));
}
__device__ __forceinline__ void wgmma_n256(float (&d)[128], uint64_t ad, uint64_t bd, uint32_t accum) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
      "}, %128, %129, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(ad), "l"(bd), "r"(accum));
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keep the compiler from moving accumulator reads / writes across a wgmma fence or wait
template <int R>
__device__ __forceinline__ void wg_fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// one 64-channel K chunk: 4 x K=16 steps, +32 bytes (2 x 16B units) per step inside the swizzle atom
template <int BN>
__device__ __forceinline__ void wgmma_chunk(float (&d)[BN / 2], uint64_t ad, uint64_t bd, bool accumulate) {
#pragma unroll
  for (int k = 0; k < TC_BK / 16; ++k) {
    const uint32_t acc = (accumulate || k != 0) ? 1u : 0u;
    if constexpr (BN == 64) wgmma_n64(d, ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), acc);
    else if constexpr (BN == 128) wgmma_n128(d, ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), acc);
    else wgmma_n256(d, ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), acc);
  }
}

// consumer threads park this N-tile's scale / bias in shared memory, then meet (named barrier 1, consumers only)
template <int BN>
__device__ __forceinline__ void tc_stage_scale_bias(const TcArgs& a, float* s_scale, float* s_bias, int n0) {
  for (int i = threadIdx.x; i < BN; i += TC_CONSUMERS) {
    s_scale[i] = a.scale ? __ldg(a.scale + n0 + i) : 1.f;
    s_bias[i] = a.bias ? __ldg(a.bias + n0 + i) : 0.f;
  }
  asm volatile("bar.sync 1, %0;" ::"n"(TC_CONSUMERS) : "memory");
}

// ---- epilogue of one consumer warpgroup: registers -> scale / bias (+residual) (+ReLU) -> fp16 NHWC, or the raw fp32
// partial tile when K is split.  wgmma's accumulator layout: thread (warp w, lane l) of the warpgroup holds rows
// 16w + l/4 and 16w + l/4 + 8 of its 64, columns 8j + 2(l%4) and +1 in d[4j + 2h], d[4j + 2h + 1] (h = row half).
template <int BN>
__device__ __forceinline__ void tc_epilogue(const TcArgs& a, const float (&d)[BN / 2], const float* s_scale, const float* s_bias,
                                            int img, int h0, int w0, int n0) {
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127, warp = t >> 5, lane = t & 31;
  const int cl = 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = wg * 64 + warp * 16 + (lane >> 2) + 8 * h;
    if (a.splits > 1) {
      // ---- split-K: park the raw fp32 partial tile [split][tile][128][Cout]; splitk_reduce_kernel finishes the layer
      float* mine = a.partial + (((size_t)blockIdx.z * a.num_tiles + blockIdx.x) * TC_BM + row) * a.Cout + n0 + cl;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) *reinterpret_cast<float2*>(mine + 8 * j) = make_float2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
      continue;
    }
    const int oh = h0 + row / a.tile_w, ow = w0 + row % a.tile_w;
    if (oh >= a.H || ow >= a.W) continue;
    const size_t pix = ((size_t)img * a.H + oh) * a.W + ow;
    const __half* rp = a.res ? a.res + pix * a.res_ld + n0 + cl : nullptr;
    __half* op = a.out + pix * a.out_ld + n0 + cl;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int c = 8 * j + cl;
      float v0 = d[4 * j + 2 * h], v1 = d[4 * j + 2 * h + 1];
      if (a.scale) {
        const float2 sc = *reinterpret_cast<const float2*>(s_scale + c);
        v0 = __fmul_rn(v0, sc.x), v1 = __fmul_rn(v1, sc.y);
      }
      if (a.bias) {
        const float2 bi = *reinterpret_cast<const float2*>(s_bias + c);
        v0 = __fadd_rn(v0, bi.x), v1 = __fadd_rn(v1, bi.y);
      }
      if (rp) {
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(rp + 8 * j));
        v0 += f.x, v1 += f.y;
      }
      if (a.relu) v0 = fmaxf(v0, 0.f), v1 = fmaxf(v1, 0.f);
      *reinterpret_cast<__half2*>(op + 8 * j) = __floats2half2_rn(v0, v1);
    }
  }
}

// ---- split-K finish inside the cluster (developer switch SMOT_TC_CLUSTER, replaces splitk_reduce_kernel).
// The `splits` CTAs of an output tile are launched as ONE thread-block cluster (1,1,splits): they are co-scheduled by the
// hardware, so after parking their raw fp32 partial tiles in the L2-resident workspace they can meet at a cluster barrier and
// each finish 128/splits rows of the tile: sum the partials in split order (deterministic, the same order and the same
// fp32 operations as splitk_reduce_kernel, so the results are bit-identical to it), scale / bias / residual / ReLU, fp16 store.
template <int BN>
__device__ __forceinline__ void tc_splitk_finish(const TcArgs& a, const float* s_scale, const float* s_bias, int img, int h0, int w0,
                                                 int n0) {
  // all warps take part; every thread has FIN_ITEMS float4 positions x up to 8 partials in flight before it sums
  constexpr int FIN_ITEMS = 3, MAXS = 8;
  const int tid = (int)threadIdx.x;
  const int rows_per = (TC_BM + a.splits - 1) / a.splits;
  const int r_lo = (int)blockIdx.z * rows_per;
  const int r_hi = min(TC_BM, r_lo + rows_per);
  constexpr int C4 = BN / 4;
  const int n_items = (r_hi - r_lo) * C4;
  const size_t zstride = (size_t)a.num_tiles * TC_BM * a.Cout;
  const float* tile = a.partial + (size_t)blockIdx.x * TC_BM * a.Cout + n0;
  for (int base = tid; base < n_items; base += TC_THREADS * FIN_ITEMS) {
    float4 v[FIN_ITEMS][MAXS];
    int row[FIN_ITEMS], col[FIN_ITEMS];
    bool ok[FIN_ITEMS];
#pragma unroll
    for (int it = 0; it < FIN_ITEMS; ++it) {
      const int idx = base + it * TC_THREADS;
      row[it] = r_lo + idx / C4, col[it] = (idx % C4) * 4;
      const int oh = h0 + row[it] / a.tile_w, ow = w0 + row[it] % a.tile_w;
      ok[it] = idx < n_items && oh < a.H && ow < a.W;
      const float* p = tile + (size_t)row[it] * a.Cout + col[it];
#pragma unroll
      for (int z = 0; z < MAXS; ++z)
        if (ok[it] && z < a.splits) v[it][z] = __ldcg(reinterpret_cast<const float4*>(p + (size_t)z * zstride));
    }
#pragma unroll
    for (int it = 0; it < FIN_ITEMS; ++it) {
      if (!ok[it]) continue;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int z = 0; z < MAXS; ++z)
        if (z < a.splits) acc.x += v[it][z].x, acc.y += v[it][z].y, acc.z += v[it][z].z, acc.w += v[it][z].w;   // split order
      float o[4] = {acc.x, acc.y, acc.z, acc.w};
      const int c = col[it];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (a.scale) o[j] = __fmul_rn(o[j], s_scale[c + j]);
        if (a.bias) o[j] = __fadd_rn(o[j], s_bias[c + j]);
      }
      const int oh = h0 + row[it] / a.tile_w, ow = w0 + row[it] % a.tile_w;
      const size_t pix = ((size_t)img * a.H + oh) * a.W + ow;
      if (a.res) {
        const float4 r = ld4(a.res + pix * a.res_ld + n0 + c);
        o[0] += r.x, o[1] += r.y, o[2] += r.z, o[3] += r.w;
      }
      if (a.relu) {
#pragma unroll
        for (int j = 0; j < 4; ++j) o[j] = fmaxf(o[j], 0.f);
      }
      st4(a.out + pix * a.out_ld + n0 + c, make_float4(o[0], o[1], o[2], o[3]));
    }
  }
}

template <int BN, int STAGES>
struct TcSmem {
  static constexpr int A_BYTES = TC_BM * TC_BK * 2;
  static constexpr int B_BYTES = BN * TC_BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int TOTAL = STAGES * STAGE_BYTES + 1024 /*alignment slack*/ + 256 /*barriers*/ + BN * 8 /*scale, bias*/;
};

// K slices keep a second register accumulator (the running sum): only the variants whose two accumulators fit carry them
template <int BN, int STAGES>
constexpr bool tc_has_slices() { return STAGES > 2 && BN <= 128; }

// the 2-stage variants (many short tiles) run 2 CTAs per SM: cap their registers accordingly
template <int BN, int STAGES>
__global__ void __launch_bounds__(TC_THREADS, STAGES == 2 ? 2 : 1) conv_tc_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                                  const __grid_constant__ CUtensorMap tmB,
                                                                                  const TcArgs a) {
  using S = TcSmem<BN, STAGES>;
  constexpr bool SLICES = tc_has_slices<BN, STAGES>();
  extern __shared__ uint8_t tc_smem_raw[];
  // 128B-swizzled tiles need 1024B-aligned bases
  uint8_t* smem = tc_smem_raw + ((1024u - (smem_u32(tc_smem_raw) & 1023u)) & 1023u);
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * S::A_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * S::STAGE_BYTES);
  uint64_t* full = bars;
  uint64_t* empty = bars + STAGES;
  float* s_scale = reinterpret_cast<float*>(smem + STAGES * S::STAGE_BYTES + 256);  // [BN] scale, then [BN] bias
  float* s_bias = s_scale + BN;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  pdl_launch_dependents();
  if (threadIdx.x == 0) TC_STAMP(0);
  // tile coordinates
  int t = blockIdx.x;
  const int tw = t % a.tiles_w;
  t /= a.tiles_w;
  const int th = t % a.tiles_h;
  const int img = t / a.tiles_h;
  const int w0 = tw * a.tile_w, h0 = th * a.tile_h;
  const int n0 = blockIdx.y * BN;
  const int all_chunks = a.taps * a.cin_chunks;
  const bool sliced = SLICES && a.slices > 1;                             // all K slices in this CTA, one running sum
  const int it0 = sliced ? 0 : (int)blockIdx.z * a.chunks_per_split;    // this CTA's K range [it0, it0 + total)
  const int total = sliced ? all_chunks : min(a.chunks_per_split, all_chunks - it0);

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 2);  // one arrival per consumer warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();  // everything above overlapped the previous kernel; its outputs are read (and buffers rewritten) from here on
  if (threadIdx.x == 0) TC_STAMP(1);

  if (warp == TC_PRODUCER_WARP) {
    if (lane == 0) {  // ===== TMA producer =====
      for (int it = 0; it < total; ++it) {
        const int s = it % STAGES;
        const uint32_t ph = (uint32_t)(it / STAGES) & 1u;
        mbar_wait(&empty[s], ph ^ 1u);
        mbar_expect_tx(&full[s], (uint32_t)S::STAGE_BYTES);
        const int tap = (it0 + it) / a.cin_chunks, cc = (it0 + it) - tap * a.cin_chunks;
        const int r = tap / a.KW, sx = tap - r * a.KW;
        tma_load_4d(sA + s * S::A_BYTES, &tmA, &full[s], cc * TC_BK, w0 * a.stride + sx - a.pad, h0 * a.stride + r - a.pad, img);
        tma_load_2d(sB + s * S::B_BYTES, &tmB, &full[s], tap * a.Cin + cc * TC_BK, n0);
      }
    }
  } else {  // ===== consumer warpgroups: wgmma main loop, then the epilogue of their 64 rows =====
    tc_stage_scale_bias<BN>(a, s_scale, s_bias, n0);
    const int wg = threadIdx.x >> 7;
    const bool leader = (threadIdx.x & 127) == 0;
    float acc[BN / 2];
    float sum[SLICES ? BN / 2 : 1];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    if constexpr (SLICES) {
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) sum[i] = 0.f;
    }
    for (int it = 0; it < total; ++it) {
      const int s = it % STAGES;
      mbar_wait(&full[s], (uint32_t)(it / STAGES) & 1u);
      if (it == 0 && threadIdx.x == 0) TC_STAMP(2);
      const int itl = sliced ? it % a.chunks_per_split : it;   // chunk inside this CTA's (or this slice's) K range
      const uint64_t ad = gmma_desc_sw128(sA + s * S::A_BYTES + wg * (64 * TC_BK * 2));
      const uint64_t bd = gmma_desc_sw128(sB + s * S::B_BYTES);
      wg_fence_acc(acc);
      wg_fence();
      wgmma_chunk<BN>(acc, ad, bd, itl != 0);
      wg_commit();
      wg_wait<1>();                                     // the previous chunk's wgmma group has read its slot
      wg_fence_acc(acc);
      if (it > 0 && leader) mbar_arrive(&empty[(it - 1) % STAGES]);
      if constexpr (SLICES) {
        if (sliced && (itl == a.chunks_per_split - 1 || it == total - 1)) {
          // a K slice is complete: add it to the running sum in slice order from 0.f -- splitk_reduce_kernel's operations
          wg_wait<0>();
          wg_fence_acc(acc);
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) sum[i] += acc[i];
        }
      }
    }
    wg_wait<0>();
    wg_fence_acc(acc);
    if (threadIdx.x == 0) TC_STAMP(3);
    if constexpr (SLICES) {
      if (sliced) {
        tc_epilogue<BN>(a, sum, s_scale, s_bias, img, h0, w0, n0);
      } else {
        tc_epilogue<BN>(a, acc, s_scale, s_bias, img, h0, w0, n0);
      }
    } else {
      tc_epilogue<BN>(a, acc, s_scale, s_bias, img, h0, w0, n0);
    }
    if (threadIdx.x == 0) TC_STAMP(4);
  }
  if constexpr (STAGES > 2)   // the 2-stage variants run 2 CTAs per SM on full-GPU layers: they never split K, keep their registers low
  if (a.cluster_reduce) {
    // every CTA of the tile's cluster has parked its partial: publish (gpu scope), meet, finish 128 / splits rows each
    __threadfence();
    __syncwarp();
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
    tc_splitk_finish<BN>(a, s_scale, s_bias, img, h0, w0, n0);
  }
  if (threadIdx.x == 0) TC_STAMP(5);
}

// ---------------------------------------------------------------------------------------------
// 3x3 / stride 1 with a shared-memory resident input halo (developer switch SMOT_TC_HALO).
// conv_tc_kernel re-reads the A operand once per filter tap: 9 x 16 KB per 64-channel chunk and CTA.  Here the
// (8+2) x (16+2) pixel halo of an 8 x 16 output tile is loaded ONCE per channel chunk (one 4-D TMA box, PW pixels per
// patch row, 128B-swizzled, zero fill = conv padding) and the nine taps are nine shifted views of it: row m = y*8 + x of
// tap (r, s) is patch pixel (y + r, x + s), i.e. the wgmma descriptor of consumer warpgroup g (rows y = 8g..8g+7) starts
// ((8g + r)*PW + s) * 128 B into the patch and steps PW * 128 B between its 8-row groups.  Only the weights still stream
// per tap (their own ring).  K order: channel chunk outermost, taps inside.
// ---------------------------------------------------------------------------------------------
constexpr int HALO_TW = 8, HALO_TH = 16, HALO_SA = 2;

template <int BN, int PW, int SB>
struct HaloSmem {
  static constexpr int A_BOX_BYTES = (HALO_TH + 2) * PW * TC_BK * 2;              // bytes one TMA patch delivers
  static constexpr int A_BYTES = ((A_BOX_BYTES + 1023) / 1024) * 1024;
  static constexpr int B_BYTES = BN * TC_BK * 2;
  static constexpr int RING = HALO_SA * A_BYTES + SB * B_BYTES;
  static constexpr int TOTAL = RING + 1024 /*alignment slack*/ + 256 /*barriers*/ + BN * 8 /*scale, bias*/;
  static_assert((2 * HALO_SA + 2 * SB) * 8 <= 256, "barrier block");
};

template <int BN, int PW, int SB>
__global__ void __launch_bounds__(TC_THREADS) conv3x3_halo_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                  const __grid_constant__ CUtensorMap tmB, const TcArgs a,
                                                                  const int bo_mode) {
  using S = HaloSmem<BN, PW, SB>;
  extern __shared__ uint8_t tc_smem_raw[];
  uint8_t* smem = tc_smem_raw + ((1024u - (smem_u32(tc_smem_raw) & 1023u)) & 1023u);
  uint8_t* sA = smem;
  uint8_t* sB = smem + HALO_SA * S::A_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S::RING);
  uint64_t* fullA = bars;
  uint64_t* emptyA = fullA + HALO_SA;
  uint64_t* fullB = emptyA + HALO_SA;
  uint64_t* emptyB = fullB + SB;
  float* s_scale = reinterpret_cast<float*>(smem + S::RING + 256);
  float* s_bias = s_scale + BN;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  pdl_launch_dependents();
  int t = blockIdx.x;
  const int tw = t % a.tiles_w;
  t /= a.tiles_w;
  const int th = t % a.tiles_h;
  const int img = t / a.tiles_h;
  const int w0 = tw * HALO_TW, h0 = th * HALO_TH;
  const int n0 = blockIdx.y * BN;
  const int cc0 = (int)blockIdx.z * a.chunks_per_split;                  // this CTA's channel chunks [cc0, cc0 + ncc)
  const int ncc = min(a.chunks_per_split, a.cin_chunks - cc0);

  if (threadIdx.x == 0) {
    for (int i = 0; i < HALO_SA; ++i) mbar_init(&fullA[i], 1), mbar_init(&emptyA[i], 2);
    for (int i = 0; i < SB; ++i) mbar_init(&fullB[i], 1), mbar_init(&emptyB[i], 2);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();

  // developer probes (timing only, results are garbage): 256 = no MMAs, 512 = no weight loads, 1024 = no patch loads
  const bool no_mma = bo_mode & 256, no_b = bo_mode & 512, no_a = bo_mode & 1024;
  if (warp == TC_PRODUCER_WARP) {
    if (lane == 0) {  // ===== TMA producer: one halo patch per channel chunk, one weight tile per tap =====
      int ib = 0;
      for (int ic = 0; ic < ncc; ++ic) {
        const int sa = ic % HALO_SA;
        if (!no_a) {
          mbar_wait(&emptyA[sa], ((uint32_t)(ic / HALO_SA) & 1u) ^ 1u);
          mbar_expect_tx(&fullA[sa], (uint32_t)S::A_BOX_BYTES);
          tma_load_4d(sA + sa * S::A_BYTES, &tmA, &fullA[sa], (cc0 + ic) * TC_BK, w0 - 1, h0 - 1, img);
        }
        for (int tap = 0; tap < 9 && !no_b; ++tap, ++ib) {
          const int sb = ib % SB;
          mbar_wait(&emptyB[sb], ((uint32_t)(ib / SB) & 1u) ^ 1u);
          mbar_expect_tx(&fullB[sb], (uint32_t)S::B_BYTES);
          tma_load_2d(sB + sb * S::B_BYTES, &tmB, &fullB[sb], tap * a.Cin + (cc0 + ic) * TC_BK, n0);
        }
      }
    }
  } else {  // ===== consumer warpgroups =====
    tc_stage_scale_bias<BN>(a, s_scale, s_bias, n0);
    const int wg = threadIdx.x >> 7;
    const bool leader = (threadIdx.x & 127) == 0;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int ib = 0;
    for (int ic = 0; ic < ncc; ++ic) {
      const int sa = ic % HALO_SA;
      if (!no_a) mbar_wait(&fullA[sa], (uint32_t)(ic / HALO_SA) & 1u);
      const uint8_t* patch = sA + sa * S::A_BYTES;
      for (int tap = 0; tap < 9; ++tap, ++ib) {
        const int sb = ib % SB;
        if (!no_b) mbar_wait(&fullB[sb], (uint32_t)(ib / SB) & 1u);
        const int r = tap / 3, sx = tap - 3 * r;
        const uint32_t first_row = (uint32_t)((8 * wg + r) * PW + sx);   // patch pixel of this warpgroup's row 0 for this tap
        const uint64_t ad = gmma_desc_sw128(patch + first_row * 128u, (uint32_t)PW * 128u, (bo_mode & 1) ? first_row : 0u);
        const uint64_t bd = gmma_desc_sw128(sB + sb * S::B_BYTES);
        if (!no_mma) {
          wg_fence_acc(acc);
          wg_fence();
          wgmma_chunk<BN>(acc, ad, bd, (ic | tap) != 0);
          wg_commit();
          wg_wait<1>();                                   // the previous tap's wgmma group is done with its slots
          wg_fence_acc(acc);
        }
        if (ib > 0 && leader) {
          if (!no_b) mbar_arrive(&emptyB[(ib - 1) % SB]);
          if (tap == 0 && !no_a) mbar_arrive(&emptyA[(ic - 1) % HALO_SA]);   // all nine taps of the previous patch are read
        }
      }
    }
    wg_wait<0>();
    wg_fence_acc(acc);
    tc_epilogue<BN>(a, acc, s_scale, s_bias, img, h0, w0, n0);
  }
}

// Deterministic split-K finish: out[pixel][n] = act((sum_z partial[z]) * scale + bias + residual), summed in split order.
// One thread per 4 output channels of one pixel; tiles map back to pixels exactly as in conv_tc_kernel.
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const TcArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  const int c4 = a.Cout / 4;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)a.num_tiles * TC_BM * c4;
  if (idx >= total) return;
  const int n = (int)(idx % c4) * 4;
  const size_t rowg = idx / c4;  // tile * 128 + row
  const int row = (int)(rowg % TC_BM);
  int t = (int)(rowg / TC_BM);
  const int tw = t % a.tiles_w;
  t /= a.tiles_w;
  const int th = t % a.tiles_h;
  const int img = t / a.tiles_h;
  const int oh = th * a.tile_h + row / a.tile_w, ow = tw * a.tile_w + row % a.tile_w;
  if (oh >= a.H || ow >= a.W) return;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int z = 0; z < a.splits; ++z) {
    const float4 p = *reinterpret_cast<const float4*>(a.partial + ((size_t)z * a.num_tiles * TC_BM + rowg) * a.Cout + n);
    acc.x += p.x, acc.y += p.y, acc.z += p.z, acc.w += p.w;
  }
  float v[4] = {acc.x, acc.y, acc.z, acc.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (a.scale) v[j] = __fmul_rn(v[j], a.scale[n + j]);
    if (a.bias) v[j] = __fadd_rn(v[j], a.bias[n + j]);
  }
  const size_t pix = ((size_t)img * a.H + oh) * a.W + ow;
  if (a.res) {
    const float4 r = ld4(a.res + pix * a.res_ld + n);
    v[0] += r.x, v[1] += r.y, v[2] += r.z, v[3] += r.w;
  }
  if (a.relu) {
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = fmaxf(v[j], 0.f);
  }
  st4(a.out + pix * a.out_ld + n, make_float4(v[0], v[1], v[2], v[3]));
}

// ---- host side ------------------------------------------------------------------------------
constexpr int SMOT_TC_DEFAULT_MAXSPLIT = 8;
// The split factor of a layer fixes the order in which its fp32 partial sums are added, so it is a function of the layer
// alone and not of the device it runs on: the same weights and frames give the same bits on any GPU.  The basis is a
// CTA budget of 148 (a little more than the 132 SMs of an H100: the split CTAs of few-tile layers fill one wave either way).
constexpr int SMOT_TC_SPLIT_BASIS = 148;
static PFN_cuTensorMapEncodeTiled get_encode() {
  static PFN_cuTensorMapEncodeTiled fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled>(p);
  }
  return fn;
}

static bool encode_map(CUtensorMap* tm, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                       const uint32_t* box, const uint32_t* estr_in = nullptr) {
  PFN_cuTensorMapEncodeTiled enc = get_encode();
  if (!enc) {
    set_error("smot_conv2d(wgmma): cuTensorMapEncodeTiled entry point not available");
    return false;
  }
  uint32_t estr[4] = {1, 1, 1, 1};
  if (estr_in)
    for (int i = 0; i < rank; ++i) estr[i] = estr_in[i];
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(base), dims, strides_bytes, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("smot_conv2d(wgmma): cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
    return false;
  }
  return true;
}

// Widest split of the K loop of a few-tile layer (levels 4 / 5, FC layers), finished by splitk_reduce_kernel.
// SMOT_TC_MAXSPLIT=1..8 (SMOT_TC_NOSPLIT=1 is MAXSPLIT=1).  A wider split makes a layer alone faster, but 8 CTAs per
// tile plus a reduce kernel per layer occupy SMs that the detection tail and the track stage of the neighbouring frames
// would otherwise use.
static int tc_max_split() {
  static const int v = [] {
    if (getenv("SMOT_TC_NOSPLIT")) return 1;
    const char* e = getenv("SMOT_TC_MAXSPLIT");
    const int m = e ? atoi(e) : SMOT_TC_DEFAULT_MAXSPLIT;
    return m < 1 ? 1 : (m > 8 ? 8 : m);
  }();
  return v;
}

bool conv2d_tc_supported(const smot_conv_desc* d) {
  if (d->in_dtype != SMOT_F16 || d->out_dtype != SMOT_F16) return false;
  if (d->KH != d->KW || (d->KH != 1 && d->KH != 3) || d->pad != d->KH / 2) return false;
  if (d->stride != 1 && !(d->stride == 2 && d->KH == 3 && d->H % 2 == 0 && d->W % 2 == 0 && d->H > 1)) return false;
  if (d->Cin % TC_BK != 0 || d->Cout % 64 != 0) return false;
  if (d->in_ld % 8 != 0 || d->out_ld % 8 != 0 || (d->residual && d->res_ld % 8 != 0)) return false;
  if (((uintptr_t)d->in | (uintptr_t)d->weight | (uintptr_t)d->out | (uintptr_t)d->residual) & 15) return false;
  if (d->batch < 1 || d->OH != d->H / d->stride || d->OW != d->W / d->stride) return false;
  if ((long long)d->batch * d->OH * d->OW < 16) return false;  // not worth a 128-row tile
  return true;
}

// launch attributes: programmatic dependent launch always; a (1,1,cluster_z) thread-block cluster when the CTAs of a tile
// finish their split-K sum themselves
template <int BN, int STAGES>
static cudaError_t launch_tc_ex(const CUtensorMap& tmA, const CUtensorMap& tmB, const TcArgs& a, dim3 grid, int cluster_z,
                                cudaStream_t st) {
  using S = TcSmem<BN, STAGES>;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid, cfg.blockDim = dim3(TC_THREADS), cfg.dynamicSmemBytes = S::TOTAL, cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  cfg.attrs = attr, cfg.numAttrs = 1;
  if (cluster_z > 1) {
    attr[1].id = cudaLaunchAttributeClusterDimension;
    attr[1].val.clusterDim.x = 1, attr[1].val.clusterDim.y = 1, attr[1].val.clusterDim.z = (unsigned)cluster_z;
    cfg.numAttrs = 2;
  }
  return cudaLaunchKernelEx(&cfg, conv_tc_kernel<BN, STAGES>, tmA, tmB, a);
}

template <int BN, int STAGES>
static int launch_tc(const CUtensorMap& tmA, const CUtensorMap& tmB, const TcArgs& a, dim3 grid, cudaStream_t st) {
  using S = TcSmem<BN, STAGES>;
  SMOT_ENSURE_SMEM((conv_tc_kernel<BN, STAGES>), S::TOTAL, "smot_conv2d(wgmma)");
  cudaError_t e = launch_tc_ex<BN, STAGES>(tmA, tmB, a, grid, a.cluster_reduce ? a.splits : 1, st);
  if (e != cudaSuccess) {
    set_error("smot_conv2d(wgmma): launch failed: %s", cudaGetErrorString(e));
    return SMOT_ERR_CUDA;
  }
  SMOT_CHECK_LAUNCH("smot_conv2d(wgmma)");
  return SMOT_OK;
}

// How many (1,1,cz) clusters of this kernel variant the device can hold at once (a cluster lives inside one GPC, so this is
// NOT sm_count() / cz: a GPC holds only a few clusters of 8).  Queried once per (variant, cz); 0 = query failed.
template <int BN, int STAGES>
static int tc_max_clusters(int cz) {
  static std::mutex mu;
  static int cache[9] = {-1, -1, -1, -1, -1, -1, -1, -1, -1};
  if (cz < 2 || cz > 8) return 0;
  std::lock_guard<std::mutex> lock(mu);
  if (cache[cz] >= 0) return cache[cz];
  using S = TcSmem<BN, STAGES>;
  int n = 0;
  if (cudaFuncSetAttribute(conv_tc_kernel<BN, STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, S::TOTAL) == cudaSuccess) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(1, 1, (unsigned)cz), cfg.blockDim = dim3(TC_THREADS), cfg.dynamicSmemBytes = S::TOTAL;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 1, attr[0].val.clusterDim.y = 1, attr[0].val.clusterDim.z = (unsigned)cz;
    cfg.attrs = attr, cfg.numAttrs = 1;
    if (cudaOccupancyMaxActiveClusters(&n, conv_tc_kernel<BN, STAGES>, &cfg) != cudaSuccess) n = 0;
  }
  (void)cudaGetLastError();
  cache[cz] = n;
  return n;
}

// ring depth of the generic kernel for a given tile width / CTA population / K length (measured choices, see conv2d_tc)
static int tc_stages(int BN, bool solo, bool shallow, int my_chunks, int forced) {
  if (BN == 256) return (forced ? forced >= 4 : (solo && my_chunks >= 4)) ? 4 : 3;
  const bool deep = forced ? forced >= 6 : (solo && my_chunks >= 6);
  if (BN == 128) return shallow ? 2 : (deep ? 6 : 3);
  return deep ? 8 : (shallow ? 2 : 4);
}

#define SMOT_TC_DISPATCH(BN_, ST_, EXPR)                                                       \
  ((BN_) == 256 ? ((ST_) == 4 ? EXPR(256, 4) : EXPR(256, 3))                                    \
   : (BN_) == 128 ? ((ST_) == 2 ? EXPR(128, 2) : ((ST_) == 6 ? EXPR(128, 6) : EXPR(128, 3)))   \
                  : ((ST_) == 8 ? EXPR(64, 8) : ((ST_) == 2 ? EXPR(64, 2) : EXPR(64, 4))))

template <int BN, int PW, int SB>
static int launch_halo(const CUtensorMap& tmA, const CUtensorMap& tmB, const TcArgs& a, dim3 grid, int bo_mode, cudaStream_t st) {
  using S = HaloSmem<BN, PW, SB>;
  SMOT_ENSURE_SMEM((conv3x3_halo_kernel<BN, PW, SB>), S::TOTAL, "smot_conv2d(wgmma halo)");
  launch_pdl(conv3x3_halo_kernel<BN, PW, SB>, grid, dim3(TC_THREADS), S::TOTAL, st, tmA, tmB, a, bo_mode);
  SMOT_CHECK_LAUNCH("smot_conv2d(wgmma halo)");
  return SMOT_OK;
}

static int halo_mode() {  // developer switch SMOT_TC_HALO: 0 = off, 16 / 10 = patch width, +100 = descriptor base offset mode
  const char* e = getenv("SMOT_TC_HALO");
  return e ? atoi(e) : 0;
}

static int conv2d_tc_halo(const smot_conv_desc* d, int mode, cudaStream_t st) {
  TcArgs a;
  a.scale = d->scale, a.bias = d->bias, a.res = (const __half*)d->residual, a.out = (__half*)d->out;
  a.H = d->OH, a.W = d->OW, a.stride = 1, a.Cin = d->Cin, a.Cout = d->Cout, a.out_ld = d->out_ld, a.res_ld = d->res_ld, a.relu = d->relu;
  a.taps = 9, a.KW = 3, a.pad = 1, a.cin_chunks = d->Cin / TC_BK;
  a.tile_w = HALO_TW, a.tile_h = HALO_TH;
  a.tiles_w = ceil_div(d->OW, HALO_TW), a.tiles_h = ceil_div(d->OH, HALO_TH);
  const long long tiles = (long long)a.tiles_w * a.tiles_h * d->batch;
  const int pw = mode % 100;
  int bo_mode = (mode / 100) & 1;
  if (const char* e = getenv("SMOT_TC_PROBE")) bo_mode |= atoi(e);
  int BN = 64;
  if (d->Cout % 256 == 0 && tiles * (d->Cout / 256) >= 96) BN = 256;
  else if (d->Cout % 128 == 0 && tiles * (d->Cout / 128) >= 96) BN = 128;
  int splits = 1;
  {
    const int bw = d->Cout % 256 == 0 ? 256 : (d->Cout % 128 == 0 ? 128 : 64);
    const long long cw = tiles * (d->Cout / bw);
    if (d->workspace && cw <= 40 && a.cin_chunks >= 2 && tc_max_split() > 1) {
      int sp = (int)(SMOT_TC_SPLIT_BASIS / cw);
      if (sp > tc_max_split()) sp = tc_max_split();
      if (sp > a.cin_chunks) sp = a.cin_chunks;
      const size_t need = (size_t)SMOT_CONV_WS_COUNTER_BYTES + (size_t)sp * tiles * TC_BM * d->Cout * sizeof(float);
      if (sp >= 2 && need <= d->workspace_bytes) splits = sp, BN = bw;
    }
  }
  CUtensorMap tmA, tmB;
  {
    uint64_t dims[4] = {(uint64_t)d->Cin, (uint64_t)d->W, (uint64_t)d->H, (uint64_t)d->batch};
    uint64_t str[3] = {(uint64_t)d->in_ld * 2, (uint64_t)d->W * d->in_ld * 2, (uint64_t)d->H * d->W * d->in_ld * 2};
    uint32_t box[4] = {(uint32_t)TC_BK, (uint32_t)pw, (uint32_t)(HALO_TH + 2), 1u};
    if (!encode_map(&tmA, d->in, 4, dims, str, box)) return SMOT_ERR_CUDA;
  }
  {
    const uint64_t K = (uint64_t)9 * d->Cin;
    uint64_t dims[2] = {K, (uint64_t)d->Cout};
    uint64_t str[1] = {K * 2};
    uint32_t box[2] = {(uint32_t)TC_BK, (uint32_t)BN};
    if (!encode_map(&tmB, d->weight, 2, dims, str, box)) return SMOT_ERR_CUDA;
  }
  a.chunks_per_split = (a.cin_chunks + splits - 1) / splits;
  a.splits = (a.cin_chunks + a.chunks_per_split - 1) / a.chunks_per_split;
  a.num_tiles = (int)tiles;
  a.cluster_reduce = 0;
  a.slices = 1;
  a.dbg = nullptr;
  a.partial = d->workspace ? (float*)((char*)d->workspace + SMOT_CONV_WS_COUNTER_BYTES) : nullptr;
  dim3 grid((unsigned)tiles, (unsigned)(d->Cout / BN), (unsigned)a.splits);
  const bool crowded = (long long)grid.x * grid.y * grid.z > sm_count();   // several CTAs per SM: shallow weight ring, 2 CTAs / SM
  int rc;
#define SMOT_HALO(BN_, SB_) (pw == 10 ? launch_halo<BN_, 10, SB_>(tmA, tmB, a, grid, bo_mode, st) : launch_halo<BN_, 16, SB_>(tmA, tmB, a, grid, bo_mode, st))
  if (BN == 256) rc = SMOT_HALO(256, 4);
  else if (BN == 128) rc = crowded ? SMOT_HALO(128, 2) : SMOT_HALO(128, 6);
  else rc = crowded ? SMOT_HALO(64, 4) : SMOT_HALO(64, 8);
#undef SMOT_HALO
  if (rc != SMOT_OK || a.splits == 1) return rc;
  const size_t total_out = (size_t)a.num_tiles * TC_BM * (d->Cout / 4);
  launch_pdl(splitk_reduce_kernel, dim3((unsigned)((total_out + 255) / 256)), dim3(256), 0, st, a);
  SMOT_CHECK_LAUNCH("smot_conv2d(split-K reduce)");
  return SMOT_OK;
}

int conv2d_tc(const smot_conv_desc* d, cudaStream_t st) {
  if (d->KH == 3 && d->stride == 1 && d->H > 1 && (halo_mode() % 100 == 16 || halo_mode() % 100 == 10))
    return conv2d_tc_halo(d, halo_mode(), st);
  TcArgs a;
  a.scale = d->scale, a.bias = d->bias, a.res = (const __half*)d->residual, a.out = (__half*)d->out;
  a.H = d->OH, a.W = d->OW, a.stride = d->stride, a.Cin = d->Cin, a.Cout = d->Cout, a.out_ld = d->out_ld, a.res_ld = d->res_ld, a.relu = d->relu;
  a.taps = d->KH * d->KW, a.KW = d->KW, a.pad = d->pad, a.cin_chunks = d->Cin / TC_BK;
  if (d->H == 1) {
    a.tile_w = 128, a.tile_h = 1;
  } else {
    a.tile_w = 16, a.tile_h = 8;
  }
  a.tiles_w = ceil_div(d->OW, a.tile_w), a.tiles_h = ceil_div(d->OH, a.tile_h);
  const long long tiles = (long long)a.tiles_w * a.tiles_h * d->batch;
  // Tile shape.  Most of these layers are short, so per-kernel / per-CTA fixed cost (launch, prologue, epilogue) is a large
  // share of a layer.  Hence: (a) the widest N that still leaves ~100 CTAs; (b) layers with only a handful of output tiles
  // (levels 4-5, FC layers) take the widest BN AND split K over up to 8 CTAs, finished by splitk_reduce_kernel.
  const int all_chunks = a.taps * a.cin_chunks;
  static const int min_ctas = getenv("SMOT_TC_MINCTAS") ? atoi(getenv("SMOT_TC_MINCTAS")) : 96;   // developer override
  int BN = 64;
  if (d->Cout % 256 == 0 && tiles * (d->Cout / 256) >= min_ctas) BN = 256;
  else if (d->Cout % 128 == 0 && tiles * (d->Cout / 128) >= min_ctas) BN = 128;
  const char* force = getenv("SMOT_TC_STAGES");  // developer override: ring depth
  const int fs = force ? atoi(force) : 0;
  // developer switch SMOT_TC_CLUSTER=1: the split CTAs of a tile form a cluster and finish the tile themselves (tc_splitk_finish).
  // Bit-identical to the reduce kernel, but the serial store -> fence -> cluster barrier -> 128 KB read-back of one CTA
  // competes with a reduce grid that spreads over all SMs and overlaps the next layer's prologue through PDL.
  static const bool cluster_ok = getenv("SMOT_TC_CLUSTER") && atoi(getenv("SMOT_TC_CLUSTER")) == 1;
  int splits = 1, cluster_reduce = 0;
  {
    const int bw = d->Cout % 256 == 0 ? 256 : (d->Cout % 128 == 0 ? 128 : 64);
    // The split factor is a function of the tiles of ONE image: a batch-2 backbone pass (Engine.pair_plan) must sum every
    // output element in exactly the order a single-frame pass does, so that clip results equal frame-by-frame results bit
    // for bit.  (With two images the split layers then run two half-length waves instead of one: the same time.)
    const long long tiles_img = tiles / (d->batch > 0 ? d->batch : 1);
    const long long cw = tiles_img * (d->Cout / bw);
    if (d->workspace && cw <= 40 && all_chunks >= 16 && tc_max_split() > 1) {
      int sp = (int)(SMOT_TC_SPLIT_BASIS / cw);
      if (sp > tc_max_split()) sp = tc_max_split();
      if (sp > all_chunks / 4) sp = all_chunks / 4;
      const size_t need = (size_t)SMOT_CONV_WS_COUNTER_BYTES + (size_t)sp * tiles * TC_BM * d->Cout * sizeof(float);
      if (sp >= 2 && need <= d->workspace_bytes) {
        // preferred: the split CTAs of a tile form a cluster and finish the tile themselves; take the widest split whose
        // clusters are all resident at once (the cluster barrier needs co-residency only inside a cluster, but a second wave
        // would double the layer's time)
        for (int cz = cluster_ok ? sp : 0; cz >= 2; --cz) {
          const int cps = (all_chunks + cz - 1) / cz;
          const int real = (all_chunks + cps - 1) / cps;                       // no empty split
          if (real != cz) continue;
          const int stg = tc_stages(bw, true, false, cps, fs);
#define SMOT_TC_MAXC(BN_, ST_) tc_max_clusters<BN_, ST_>(cz)
          const int fit = SMOT_TC_DISPATCH(bw, stg, SMOT_TC_MAXC);
#undef SMOT_TC_MAXC
          if (fit >= cw) {   // (per image: a batch of two takes two waves of clusters)
            splits = cz, BN = bw, cluster_reduce = 1;
            break;
          }
        }
        if (!cluster_reduce) splits = sp, BN = bw;                             // fallback: partials + splitk_reduce_kernel
      }
    }
  }
  // In-CTA K slices (developer switch SMOT_TC_SLICED=1 | 128 = N tile; default off): the SAME K ranges, summed in the SAME
  // order -- bit-identical results (test_conv2d_tcgen05_k_slices_equal_split_k) -- but by one CTA that adds each range's
  // register accumulator to a running sum, no partial tiles, no reduce kernel.  The accumulator and the sum must both fit in
  // registers, so N tiles stop at 128.  The split's extra CTAs fill the GPU where the neighbouring stages leave room and
  // crowd it where they do not, so the split path stays the default.
  bool sliced = false;
  static const int slice_min = getenv("SMOT_TC_SLICED_MIN") ? atoi(getenv("SMOT_TC_SLICED_MIN")) : 2;
  if (splits >= slice_min && splits > 1 && !cluster_reduce) {
    const char* e = getenv("SMOT_TC_SLICED");
    if (e && e[0] != '0') {
      const int want = atoi(e) == 128 ? 128 : 64;
      const int bn = BN < want ? BN : want;
      if (bn >= 64) sliced = true, BN = bn;
    }
  }
  CUtensorMap tmA, tmB;
  {
    uint64_t dims[4] = {(uint64_t)d->Cin, (uint64_t)d->W, (uint64_t)d->H, (uint64_t)d->batch};
    uint64_t str[3] = {(uint64_t)d->in_ld * 2, (uint64_t)d->W * d->in_ld * 2, (uint64_t)d->H * d->W * d->in_ld * 2};
    // stride-2 convs: the box is traversed with element stride 2 and still lands as tile_w x tile_h pixels
    uint32_t box[4] = {(uint32_t)TC_BK, (uint32_t)(a.tile_w * d->stride), (uint32_t)(a.tile_h * d->stride), 1u};
    uint32_t estr[4] = {1u, (uint32_t)d->stride, (uint32_t)d->stride, 1u};
    if (!encode_map(&tmA, d->in, 4, dims, str, box, estr)) return SMOT_ERR_CUDA;
  }
  {
    const uint64_t K = (uint64_t)a.taps * d->Cin;
    uint64_t dims[2] = {K, (uint64_t)d->Cout};
    uint64_t str[1] = {K * 2};
    uint32_t box[2] = {(uint32_t)TC_BK, (uint32_t)BN};
    if (!encode_map(&tmB, d->weight, 2, dims, str, box)) return SMOT_ERR_CUDA;
  }
  a.splits = splits;
  a.chunks_per_split = (all_chunks + splits - 1) / splits;
  a.splits = (all_chunks + a.chunks_per_split - 1) / a.chunks_per_split;  // no empty split
  a.cluster_reduce = (cluster_reduce && a.splits == splits) ? 1 : 0;
  a.slices = 1;
  if (sliced) {
    a.slices = a.splits, a.splits = 1;
  }
  a.num_tiles = (int)tiles;
  {
    const char* dbg = getenv("SMOT_TC_DEBUG");  // hex device pointer to 8 x u64
    a.dbg = dbg ? (unsigned long long*)strtoull(dbg, nullptr, 16) : nullptr;
  }
  a.partial = d->workspace ? (float*)((char*)d->workspace + SMOT_CONV_WS_COUNTER_BYTES) : nullptr;
  dim3 grid((unsigned)tiles, (unsigned)(d->Cout / BN), (unsigned)a.splits);
  // many short tiles: 2-stage rings let 2 CTAs share an SM, so one CTA's prologue / epilogue overlaps the
  // main loops of the others (the same bytes in flight per SM as one CTA with 4 stages)
  const bool shallow = fs ? fs == 2 : (tiles * (d->Cout / BN) >= 296 && all_chunks <= 36);
  // at most one CTA per SM: nothing else hides the TMA round trip (the loop then advances `ring depth` chunks
  // per round trip), so use the whole shared memory for the ring: 8 x 24 KB, 6 x 32 KB, 4 x 48 KB
  const bool solo = (long long)grid.x * grid.y * grid.z <= sm_count();
  int stages = tc_stages(BN, solo, shallow, sliced ? all_chunks : a.chunks_per_split, fs);
  if (sliced && stages == 2) stages = BN == 128 ? 3 : 4;   // the 2-stage variants carry no slice code
#define SMOT_TC_LAUNCH(BN_, ST_) launch_tc<BN_, ST_>(tmA, tmB, a, grid, st)
  const int rc = SMOT_TC_DISPATCH(BN, stages, SMOT_TC_LAUNCH);
#undef SMOT_TC_LAUNCH
  if (rc != SMOT_OK || a.splits == 1 || a.cluster_reduce) return rc;
  const size_t total_out = (size_t)a.num_tiles * TC_BM * (d->Cout / 4);
  launch_pdl(splitk_reduce_kernel, dim3((unsigned)((total_out + 255) / 256)), dim3(256), 0, st, a);
  SMOT_CHECK_LAUNCH("smot_conv2d(split-K reduce)");
  return SMOT_OK;
}

}  // namespace smot
