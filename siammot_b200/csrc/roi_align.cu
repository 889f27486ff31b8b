// Legacy (non-aligned) ROIAlign over an FPN pyramid, NHWC, one warp per output bin.
//
// Replaces three things of the reference at once:
//   * maskrcnn_benchmark _C.roi_align_forward (upstream csrc/cuda/ROIAlign_cuda.cu: one thread per
//     output element, 16 scalar loads each) -- here lanes own 4 channels each, so every corner read
//     of a warp is one contiguous 16B/8B-per-lane vector load;
//   * LevelMapper + the per-level nonzero/index_put loop of sr_pool.py:74-89 -- level chosen in-kernel;
//   * TrackUtils.pad_feature (track_utils.py:87-107), 170 MB of zero-padded copies per frame at 720p --
//     emulated: coordinates are evaluated in the padded frame exactly as the reference does, and
//     corner reads that fall into the padding return 0.
#include <stdlib.h>

#include "common.cuh"

namespace smot {

struct RoiArgs {
  smot_pyramid pyr;
  const float* rois;
  const float* level_boxes;
  const int* count;      // [batch]
  int max_rois, channels, res, sampling;
  // smot_roi_align_batched (the kernels' BATCHED instantiations): `batch` images, ROI row r belongs to image r / max_rois and
  // samples level l of that image at pyr.feat[l] + image * img_stride[l] (elements); count[image] bounds the image's segment.
  // The single-image instantiations never read these two fields, and compile to the code they had before batching existed.
  int batch = 1;
  long long img_stride[SMOT_MAX_LEVELS];
};

template <typename T, bool BATCHED = false>
__global__ void roi_align_kernel(const RoiArgs a, T* __restrict__ out) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int bins = a.res * a.res;
  if (warp >= (BATCHED ? a.batch * a.max_rois : a.max_rois) * bins) return;
  const int r = warp / bins;
  const int bin = warp - r * bins;
  const int ph = bin / a.res, pw = bin - ph * a.res;
  T* dst = out + (size_t)warp * a.channels;
  const int img = BATCHED ? r / a.max_rois : 0;
  const int n = a.count ? min(a.count[img], a.max_rois) : a.max_rois;
  if (r - img * a.max_rois >= n) {
    for (int c = lane * 4; c < a.channels; c += 128) st4(dst + c, make_float4(0.f, 0.f, 0.f, 0.f));
    return;
  }
  // ---- level (LevelMapper: floor(4 + log2(sqrt(area)/224 + 1e-6)), clamp, - k_min)
  const float* lb = (a.level_boxes ? a.level_boxes : a.rois) + 4 * r;
  const float area = (lb[2] - lb[0] + 1.f) * (lb[3] - lb[1] + 1.f);
  float lv = floorf(4.f + log2f(__fdiv_rn(__fsqrt_rn(area), 224.f) + 1e-6f));
  const float kmin = (float)a.pyr.k_min, kmax = (float)(a.pyr.k_min + a.pyr.num_levels - 1);
  lv = fminf(fmaxf(lv, kmin), kmax);
  const int l = (int)lv - a.pyr.k_min;

  const T* __restrict__ feat = reinterpret_cast<const T*>(a.pyr.feat[l]) + (BATCHED ? img * a.img_stride[l] : 0);
  const int H = a.pyr.H[l], W = a.pyr.W[l], ld = a.pyr.ld[l], pad = a.pyr.pad[l];
  const int Hp = H + 2 * pad, Wp = W + 2 * pad;  // size of the (virtual) padded map
  const float sc = a.pyr.scale[l];
  const float* roi = a.rois + 4 * r;
  const float x1 = roi[0] * sc, y1 = roi[1] * sc, x2 = roi[2] * sc, y2 = roi[3] * sc;
  const float rw = fmaxf(x2 - x1, 1.f), rh = fmaxf(y2 - y1, 1.f);
  const float bin_h = __fdiv_rn(rh, (float)a.res), bin_w = __fdiv_rn(rw, (float)a.res);
  const int gh = a.sampling > 0 ? a.sampling : (int)ceilf(__fdiv_rn(rh, (float)a.res));
  const int gw = a.sampling > 0 ? a.sampling : (int)ceilf(__fdiv_rn(rw, (float)a.res));
  const float cnt = (float)(gh * gw);

  for (int c = lane * 4; c < a.channels; c += 128) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int iy = 0; iy < gh; ++iy) {
      float y = y1 + (float)ph * bin_h + __fdiv_rn(((float)iy + .5f) * bin_h, (float)gh);
      for (int ix = 0; ix < gw; ++ix) {
        float x = x1 + (float)pw * bin_w + __fdiv_rn(((float)ix + .5f) * bin_w, (float)gw);
        if (y < -1.f || y > (float)Hp || x < -1.f || x > (float)Wp) continue;
        float yy = y <= 0.f ? 0.f : y, xx = x <= 0.f ? 0.f : x;
        int yl = (int)yy, xl = (int)xx, yh, xh;
        if (yl >= Hp - 1) { yh = yl = Hp - 1; yy = (float)yl; } else yh = yl + 1;
        if (xl >= Wp - 1) { xh = xl = Wp - 1; xx = (float)xl; } else xh = xl + 1;
        const float ly = yy - (float)yl, lx = xx - (float)xl, hy = 1.f - ly, hx = 1.f - lx;
        const float w1 = hy * hx, w2 = hy * lx, w3 = ly * hx, w4 = ly * lx;
        // to the real (unpadded) map; reads inside the padding are zeros
        const int ryl = yl - pad, ryh = yh - pad, rxl = xl - pad, rxh = xh - pad;
        const bool oyl = ryl >= 0 && ryl < H, oyh = ryh >= 0 && ryh < H;
        const bool oxl = rxl >= 0 && rxl < W, oxh = rxh >= 0 && rxh < W;
        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
        float4 v1 = (oyl && oxl) ? ld4(feat + ((size_t)ryl * W + rxl) * ld + c) : z;
        float4 v2 = (oyl && oxh) ? ld4(feat + ((size_t)ryl * W + rxh) * ld + c) : z;
        float4 v3 = (oyh && oxl) ? ld4(feat + ((size_t)ryh * W + rxl) * ld + c) : z;
        float4 v4 = (oyh && oxh) ? ld4(feat + ((size_t)ryh * W + rxh) * ld + c) : z;
        acc.x += w1 * v1.x + w2 * v2.x + w3 * v3.x + w4 * v4.x;
        acc.y += w1 * v1.y + w2 * v2.y + w3 * v3.y + w4 * v4.y;
        acc.z += w1 * v1.z + w2 * v2.z + w3 * v3.z + w4 * v4.z;
        acc.w += w1 * v1.w + w2 * v2.w + w3 * v3.w + w4 * v4.w;
      }
    }
    acc.x = __fdiv_rn(acc.x, cnt), acc.y = __fdiv_rn(acc.y, cnt), acc.z = __fdiv_rn(acc.z, cnt), acc.w = __fdiv_rn(acc.w, cnt);
    st4(dst + c, acc);
  }
}

// ---------------------------------------------------------------------------------------------
// Channel-planar variant: out[(roi * C + c) * plane_pitch + ph * row_pitch + pw].
//
// Producer side of smot_xcorr_planar: the EMM correlation runs per (track, channel) on the tensor cores with the window
// COLUMN as the contraction index, i.e. it wants every channel's res x res window as a dense 2-D plane.  Writing the
// search windows in that layout here (row pitch 40 halves, plane 1208 halves = exactly the shared-memory image the MMA
// phase reads) turns the consumer's staging -- 16-byte gathers at a 256-byte stride and 2-byte transposing stores --
// into one bulk copy per CTA.  The columns res .. row_pitch-1 are never written: the caller zero-fills the buffer once.
//
// grid (res rows, rois): a CTA produces one window row for all channels.  Its 8 warps compute the row's bins with the
// same arithmetic (operation for operation) as roi_align_kernel -- lanes own 4 channels, corner reads are contiguous
// 8/16-byte-per-lane loads -- and park the values in a shared-memory tile [C][res]; the tile is then written out as one
// contiguous run per channel.  (The bin arithmetic is restated rather than shared with roi_align_kernel so that the
// validated kernel stays byte-identical; unify once this variant has been through the GPU tests.)
// ---------------------------------------------------------------------------------------------
constexpr int RAP_TP = 33;  // tile pitch in elements: odd -> the 4-channels-per-lane stores are at most 2-way conflicted

template <typename T>
__global__ void __launch_bounds__(256) roi_align_planar_kernel(const RoiArgs a, T* __restrict__ out, int row_pitch,
                                                               int plane_pitch) {
  extern __shared__ __align__(16) unsigned char rap_raw[];
  T* tile = reinterpret_cast<T*>(rap_raw);  // [channels][RAP_TP]
  pdl_launch_dependents();                  // the correlation kernel may start its (input-independent) prologue now
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int ph = blockIdx.x, r = blockIdx.y;
  const int n = a.count ? min(*a.count, a.max_rois) : a.max_rois;
  T* dst = out + (size_t)r * a.channels * plane_pitch + (size_t)ph * row_pitch;
  if (r >= n) {  // rows past the count are zero, as in roi_align_kernel
    for (int i = threadIdx.x; i < a.channels * a.res; i += blockDim.x) {
      const int c = i / a.res, pw = i - c * a.res;
      dst[(size_t)c * plane_pitch + pw] = from_f<T>(0.f);
    }
    return;
  }
  const float* lb = (a.level_boxes ? a.level_boxes : a.rois) + 4 * r;
  const float area = (lb[2] - lb[0] + 1.f) * (lb[3] - lb[1] + 1.f);
  float lv = floorf(4.f + log2f(__fdiv_rn(__fsqrt_rn(area), 224.f) + 1e-6f));
  const float kmin = (float)a.pyr.k_min, kmax = (float)(a.pyr.k_min + a.pyr.num_levels - 1);
  lv = fminf(fmaxf(lv, kmin), kmax);
  const int l = (int)lv - a.pyr.k_min;

  const T* __restrict__ feat = reinterpret_cast<const T*>(a.pyr.feat[l]);
  const int H = a.pyr.H[l], W = a.pyr.W[l], ld = a.pyr.ld[l], pad = a.pyr.pad[l];
  const int Hp = H + 2 * pad, Wp = W + 2 * pad;
  const float sc = a.pyr.scale[l];
  const float* roi = a.rois + 4 * r;
  const float x1 = roi[0] * sc, y1 = roi[1] * sc, x2 = roi[2] * sc, y2 = roi[3] * sc;
  const float rw = fmaxf(x2 - x1, 1.f), rh = fmaxf(y2 - y1, 1.f);
  const float bin_h = __fdiv_rn(rh, (float)a.res), bin_w = __fdiv_rn(rw, (float)a.res);
  const int gh = a.sampling > 0 ? a.sampling : (int)ceilf(__fdiv_rn(rh, (float)a.res));
  const int gw = a.sampling > 0 ? a.sampling : (int)ceilf(__fdiv_rn(rw, (float)a.res));
  const float cnt = (float)(gh * gw);

  for (int pw = wid; pw < a.res; pw += 8) {
    for (int c = lane * 4; c < a.channels; c += 128) {
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int iy = 0; iy < gh; ++iy) {
        float y = y1 + (float)ph * bin_h + __fdiv_rn(((float)iy + .5f) * bin_h, (float)gh);
        for (int ix = 0; ix < gw; ++ix) {
          float x = x1 + (float)pw * bin_w + __fdiv_rn(((float)ix + .5f) * bin_w, (float)gw);
          if (y < -1.f || y > (float)Hp || x < -1.f || x > (float)Wp) continue;
          float yy = y <= 0.f ? 0.f : y, xx = x <= 0.f ? 0.f : x;
          int yl = (int)yy, xl = (int)xx, yh, xh;
          if (yl >= Hp - 1) { yh = yl = Hp - 1; yy = (float)yl; } else yh = yl + 1;
          if (xl >= Wp - 1) { xh = xl = Wp - 1; xx = (float)xl; } else xh = xl + 1;
          const float ly = yy - (float)yl, lx = xx - (float)xl, hy = 1.f - ly, hx = 1.f - lx;
          const float w1 = hy * hx, w2 = hy * lx, w3 = ly * hx, w4 = ly * lx;
          const int ryl = yl - pad, ryh = yh - pad, rxl = xl - pad, rxh = xh - pad;
          const bool oyl = ryl >= 0 && ryl < H, oyh = ryh >= 0 && ryh < H;
          const bool oxl = rxl >= 0 && rxl < W, oxh = rxh >= 0 && rxh < W;
          const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
          float4 v1 = (oyl && oxl) ? ld4(feat + ((size_t)ryl * W + rxl) * ld + c) : z;
          float4 v2 = (oyl && oxh) ? ld4(feat + ((size_t)ryl * W + rxh) * ld + c) : z;
          float4 v3 = (oyh && oxl) ? ld4(feat + ((size_t)ryh * W + rxl) * ld + c) : z;
          float4 v4 = (oyh && oxh) ? ld4(feat + ((size_t)ryh * W + rxh) * ld + c) : z;
          acc.x += w1 * v1.x + w2 * v2.x + w3 * v3.x + w4 * v4.x;
          acc.y += w1 * v1.y + w2 * v2.y + w3 * v3.y + w4 * v4.y;
          acc.z += w1 * v1.z + w2 * v2.z + w3 * v3.z + w4 * v4.z;
          acc.w += w1 * v1.w + w2 * v2.w + w3 * v3.w + w4 * v4.w;
        }
      }
      T* tp = tile + (size_t)c * RAP_TP + pw;
      tp[0] = from_f<T>(__fdiv_rn(acc.x, cnt));
      tp[RAP_TP] = from_f<T>(__fdiv_rn(acc.y, cnt));
      tp[2 * RAP_TP] = from_f<T>(__fdiv_rn(acc.z, cnt));
      tp[3 * RAP_TP] = from_f<T>(__fdiv_rn(acc.w, cnt));
    }
  }
  __syncthreads();
  // one contiguous run of `res` elements per channel
  for (int i = threadIdx.x; i < a.channels * a.res; i += blockDim.x) {
    const int c = i / a.res, pw = i - c * a.res;
    dst[(size_t)c * plane_pitch + pw] = tile[(size_t)c * RAP_TP + pw];
  }
}

// ---------------------------------------------------------------------------------------------
// Row-wise ROIAlign with separable sample tables (round 2).
//
// ncu on the kernels above: 27 M warp instructions for 27 000 bins, issue slots 75 %
// busy, L1 hit rate 80 %, DRAM 2 % -- they are INSTRUCTION bound: every warp re-derives the level (log2 / sqrt / IEEE
// division), the bin geometry (4 divisions) and, per sample, two IEEE divisions plus ~40 instructions of clamping and
// bounds logic, ~1000 instructions per bin of which ~150 are loads and multiply-adds.
// The sample coordinates are separable (x depends on (pw, ix) only, y on (ph, iy) only), as are the clamps, the corner
// indices, the interpolation weights and the "inside the padded map / inside the real map" predicates.  So: grid (bin row,
// roi); the CTA derives the roi's geometry once, thread j fills entry j of a shared-memory table of the row's res * gw x-samples
// (and the first gh threads the y-samples) with EXACTLY the operations of roi_align_kernel; the warps then walk the bins
// reading two table entries per sample: what is left per sample is 4 weight products, 4 vector loads and the 16
// multiply-add pairs, in the same order and rounding as before -- the outputs are bit-identical to roi_align_kernel's
// (tests/test_kernels_on_cpu.py runs both sources on the host; tests/test_ops_gpu.py on the GPU).
// PLANAR: results leave through the [C][res] shared-memory tile as one contiguous run per channel (see above); otherwise
// NHWC rows (roi, ph, pw, C).
// ---------------------------------------------------------------------------------------------
constexpr int RAR_MAX_SAMPLES = 512;   // res * gw x-entries per CTA
constexpr int RAR_MAX_YS = 128;        // rows_per_cta * gh y-entries per CTA

struct RarSample {   // one axis of one sample
  int lo, hi;        // corner indices in the REAL (unpadded) map
  float l, h;        // interpolation weights (l towards hi, h = 1 - l towards lo)
  int flags;         // bit 0: sample inside the padded map (else skipped); bit 1 / 2: lo / hi inside the real map
};

__device__ __forceinline__ RarSample rar_sample(float v, int size_padded, int size_real, int pad) {
  RarSample s;
  s.flags = (v < -1.f || v > (float)size_padded) ? 0 : 1;
  float vv = v <= 0.f ? 0.f : v;
  int lo = (int)vv, hi;
  if (lo >= size_padded - 1) { hi = lo = size_padded - 1; vv = (float)lo; } else hi = lo + 1;
  s.l = vv - (float)lo;
  s.h = 1.f - s.l;
  s.lo = lo - pad, s.hi = hi - pad;
  if (s.lo >= 0 && s.lo < size_real) s.flags |= 2;
  if (s.hi >= 0 && s.hi < size_real) s.flags |= 4;
  return s;
}

// One axis of one sample as the inner loop wants it (16 bytes = one shared-memory load): ELEMENT OFFSETS of the two corners and
// their weights.  A corner outside the real map (the virtual zero padding) or a sample outside the padded map gets weight 0 and
// the offset of a corner that exists, so the loop has no predicates, no flags and no 64-bit index arithmetic: 0 * value adds
// +-0 where roi_align_kernel adds w * 0 or skips the sample -- the same sums, bit for bit (feature maps are finite).
struct __align__(16) RarTap {
  int lo, hi;        // element offsets (index * stride) of the corners
  float h, l;        // weight of the lo / hi corner
};

__device__ __forceinline__ RarTap rar_tap(float v, int size_padded, int size_real, int pad, int stride) {
  const RarSample s = rar_sample(v, size_padded, size_real, pad);
  const bool valid = s.flags & 1, in_lo = s.flags & 2, in_hi = s.flags & 4;
  RarTap t;
  t.h = (valid && in_lo) ? s.h : 0.f;
  t.l = (valid && in_hi) ? s.l : 0.f;
  t.lo = in_lo ? s.lo * stride : (in_hi ? s.hi * stride : 0);
  t.hi = in_hi ? s.hi * stride : t.lo;
  return t;
}

// four channels as they sit in memory (fp16: 8 bytes = 2 registers), converted only when they are consumed
template <typename T> struct Raw4;
template <> struct Raw4<float> { float4 v; };
template <> struct Raw4<__half> { uint2 v; };
__device__ __forceinline__ Raw4<float> ld4raw(const float* p) { Raw4<float> r; r.v = *reinterpret_cast<const float4*>(p); return r; }
__device__ __forceinline__ Raw4<__half> ld4raw(const __half* p) { Raw4<__half> r; r.v = *reinterpret_cast<const uint2*>(p); return r; }
__device__ __forceinline__ float4 raw_to_f4(const Raw4<float>& r) { return r.v; }
__device__ __forceinline__ float4 raw_to_f4(const Raw4<__half>& r) {
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&r.v.x));
  const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&r.v.y));
  return make_float4(a.x, a.y, b.x, b.y);
}

// SAMP: compile-time sampling ratio (2 = every shipped configuration; the sample loops unroll and the 16 corner loads of a bin
// are independent) or 0 = run time.
// Round-2 instruction diet: ncu counted 818 warp instructions per bin (4 samples) in the previous form -- 64-bit index products
// per corner, five-word table entries, per-corner predicates.  Now per sample: one 16-byte table load, 4 weight products, 4 adds +
// 4 address computations + 4 loads, the conversions and the 32 multiply / add of the reference's summation order.
template <typename T, bool PLANAR, int SAMP, bool BATCHED = false>
__global__ void __launch_bounds__(256) roi_align_rows_kernel(const RoiArgs a, T* __restrict__ out, int row_pitch, int plane_pitch) {
  extern __shared__ __align__(16) unsigned char rar_raw[];
  __shared__ RarTap xs[RAR_MAX_SAMPLES];
  __shared__ RarTap ys[RAR_MAX_YS];
  T* tile = reinterpret_cast<T*>(rar_raw);  // PLANAR only: [channels][RAP_TP]
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  // the CTA owns bin rows [ph0, ph1) of roi r (PLANAR: exactly one row, the tile holds one row; NHWC: rows_per_cta rows, so
  // that the roi's geometry and the sample tables are amortised over ~64+ bins even at 7 x 7)
  const int ph0 = PLANAR ? (int)blockIdx.x : (int)blockIdx.x * row_pitch, r = blockIdx.y;
  const int ph1 = PLANAR ? ph0 + 1 : min(a.res, ph0 + row_pitch);
  const int img = BATCHED ? r / a.max_rois : 0;   // the image of row r
  const int n = a.count ? min(a.count[img], a.max_rois) : a.max_rois;
  if (r - img * a.max_rois >= n) {   // rows past the image's count are zero
    if (PLANAR) {
      T* dst = out + (size_t)r * a.channels * plane_pitch + (size_t)ph0 * row_pitch;
      for (int i = threadIdx.x; i < a.channels * a.res; i += blockDim.x) {
        const int c = i / a.res, pw = i - c * a.res;
        dst[(size_t)c * plane_pitch + pw] = from_f<T>(0.f);
      }
    } else {
      T* dst = out + ((size_t)r * a.res + ph0) * a.res * a.channels;
      for (int i = threadIdx.x * 4; i < (ph1 - ph0) * a.res * a.channels; i += blockDim.x * 4) st4(dst + i, make_float4(0.f, 0.f, 0.f, 0.f));
    }
    return;
  }
  // ---- the roi's geometry: the operations of roi_align_kernel, once per thread instead of once per sample
  const float* lb = (a.level_boxes ? a.level_boxes : a.rois) + 4 * r;
  const float area = (lb[2] - lb[0] + 1.f) * (lb[3] - lb[1] + 1.f);
  float lv = floorf(4.f + log2f(__fdiv_rn(__fsqrt_rn(area), 224.f) + 1e-6f));
  const float kmin = (float)a.pyr.k_min, kmax = (float)(a.pyr.k_min + a.pyr.num_levels - 1);
  lv = fminf(fmaxf(lv, kmin), kmax);
  const int l = (int)lv - a.pyr.k_min;
  const T* __restrict__ feat = reinterpret_cast<const T*>(a.pyr.feat[l]) + (BATCHED ? img * a.img_stride[l] : 0);
  const int H = a.pyr.H[l], W = a.pyr.W[l], ld = a.pyr.ld[l], pad = a.pyr.pad[l];
  const int Hp = H + 2 * pad, Wp = W + 2 * pad;
  const float sc = a.pyr.scale[l];
  const float* roi = a.rois + 4 * r;
  const float x1 = roi[0] * sc, y1 = roi[1] * sc, x2 = roi[2] * sc, y2 = roi[3] * sc;
  const float rw = fmaxf(x2 - x1, 1.f), rh = fmaxf(y2 - y1, 1.f);
  const float bin_h = __fdiv_rn(rh, (float)a.res), bin_w = __fdiv_rn(rw, (float)a.res);
  const int gh = SAMP > 0 ? SAMP : a.sampling, gw = gh;    // the host routes adaptive sampling (<= 0) to roi_align_kernel
  const float cnt = (float)(gh * gw);
  for (int j = threadIdx.x; j < a.res * gw; j += blockDim.x) {
    const int pw = j / gw, ix = j - pw * gw;
    const float x = x1 + (float)pw * bin_w + __fdiv_rn(((float)ix + .5f) * bin_w, (float)gw);
    xs[j] = rar_tap(x, Wp, W, pad, ld);
  }
  if ((int)threadIdx.x < (ph1 - ph0) * gh) {
    const int pr = (int)threadIdx.x / gh, iy = (int)threadIdx.x - pr * gh;
    const float y = y1 + (float)(ph0 + pr) * bin_h + __fdiv_rn(((float)iy + .5f) * bin_h, (float)gh);
    ys[threadIdx.x] = rar_tap(y, Hp, H, pad, W * ld);
  }
  __syncthreads();
  const int4* xs4 = reinterpret_cast<const int4*>(xs);
  const int4* ys4 = reinterpret_cast<const int4*>(ys);
  for (int bin = wid; bin < (ph1 - ph0) * a.res; bin += 8) {
    const int pr = bin / a.res, pw = bin - pr * a.res, ph = ph0 + pr;
    for (int c = lane * 4; c < a.channels; c += 128) {
      const T* __restrict__ base = feat + c;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int iy = 0; iy < gh; ++iy) {
        const int4 ty = ys4[pr * gh + iy];
        const float yh = __int_as_float(ty.z), yl = __int_as_float(ty.w);
#pragma unroll
        for (int ix = 0; ix < gw; ++ix) {
          const int4 tx = xs4[pw * gw + ix];
          const float xh = __int_as_float(tx.z), xl = __int_as_float(tx.w);
          const float w1 = yh * xh, w2 = yh * xl, w3 = yl * xh, w4 = yl * xl;
          const float4 v1 = raw_to_f4(ld4raw(base + (ty.x + tx.x))), v2 = raw_to_f4(ld4raw(base + (ty.x + tx.y)));
          const float4 v3 = raw_to_f4(ld4raw(base + (ty.y + tx.x))), v4 = raw_to_f4(ld4raw(base + (ty.y + tx.y)));
          acc.x += w1 * v1.x + w2 * v2.x + w3 * v3.x + w4 * v4.x;
          acc.y += w1 * v1.y + w2 * v2.y + w3 * v3.y + w4 * v4.y;
          acc.z += w1 * v1.z + w2 * v2.z + w3 * v3.z + w4 * v4.z;
          acc.w += w1 * v1.w + w2 * v2.w + w3 * v3.w + w4 * v4.w;
        }
      }
      acc.x = __fdiv_rn(acc.x, cnt), acc.y = __fdiv_rn(acc.y, cnt), acc.z = __fdiv_rn(acc.z, cnt), acc.w = __fdiv_rn(acc.w, cnt);
      if (PLANAR) {
        T* tp = tile + (size_t)c * RAP_TP + pw;
        tp[0] = from_f<T>(acc.x);
        tp[RAP_TP] = from_f<T>(acc.y);
        tp[2 * RAP_TP] = from_f<T>(acc.z);
        tp[3 * RAP_TP] = from_f<T>(acc.w);
      } else {
        st4(out + (((size_t)r * a.res + ph) * a.res + pw) * a.channels + c, acc);
      }
    }
  }
  if (PLANAR) {
    __syncthreads();
    // a warp per channel, a lane per bin of the row (res <= 32): no division per element, one contiguous run per store
    T* dst = out + (size_t)r * a.channels * plane_pitch + (size_t)ph0 * row_pitch;
    for (int c = wid; c < a.channels; c += 8)
      if (lane < a.res) dst[(size_t)c * plane_pitch + lane] = tile[(size_t)c * RAP_TP + lane];
  }
}

// developer switch SMOT_ROI_ROWS=0: the one-warp-per-bin kernels (A/B; results are bit-identical)
static bool roi_rows_enabled() {
  static const bool on = [] {
    const char* e = getenv("SMOT_ROI_ROWS");
    return !(e && e[0] == '0');
  }();
  return on;
}

// developer switch SMOT_ROI_UNROLL=1: the sampling-2 specialisation (sample loops unrolled at compile time).  With the round-2
// table format the body is the same either way; the earlier, heavier unrolled form (96 registers) measured slower (41.6 vs 33.0 us).
static bool roi_unroll_enabled() {
  static const bool on = [] {
    const char* e = getenv("SMOT_ROI_UNROLL");
    return e && e[0] == '1';
  }();
  return on;
}

}  // namespace smot

using namespace smot;

extern "C" int smot_roi_align_planar(const smot_pyramid* pyr, const float* rois, const float* level_boxes, const int* count,
                                     int max_rois, int channels, int res, int sampling_ratio, void* out, int row_pitch,
                                     int plane_pitch, int dtype, void* stream) {
  SMOT_CHECK_ARG(pyr && out && (rois || max_rois == 0), "smot_roi_align_planar: null argument");
  SMOT_CHECK_ARG(pyr->num_levels >= 1 && pyr->num_levels <= SMOT_MAX_LEVELS, "smot_roi_align_planar: num_levels %d", pyr->num_levels);
  SMOT_CHECK_ARG(channels > 0 && channels % 4 == 0 && res > 0 && res < RAP_TP && max_rois >= 0,
                 "smot_roi_align_planar: channels must be a multiple of 4 and res <= %d", RAP_TP - 1);
  SMOT_CHECK_ARG(row_pitch >= res && (long long)plane_pitch >= (long long)(res - 1) * row_pitch + res,
                 "smot_roi_align_planar: pitches %d / %d too small for res %d", row_pitch, plane_pitch, res);
  for (int l = 0; l < pyr->num_levels; ++l)
    SMOT_CHECK_ARG(pyr->feat[l] && pyr->ld[l] % 4 == 0 && pyr->H[l] > 0 && pyr->W[l] > 0 && pyr->pad[l] >= 0,
                   "smot_roi_align_planar: bad level %d", l);
  if (max_rois == 0) return SMOT_OK;
  RoiArgs a;
  a.pyr = *pyr, a.rois = rois, a.level_boxes = level_boxes, a.count = count;
  a.max_rois = max_rois, a.channels = channels, a.res = res, a.sampling = sampling_ratio;
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid((unsigned)res, (unsigned)max_rois);
  const bool rows = roi_rows_enabled() && sampling_ratio > 0 && sampling_ratio <= 16 && res * sampling_ratio <= RAR_MAX_SAMPLES;
  if (dtype == SMOT_F32) {
    const size_t smem = (size_t)channels * RAP_TP * sizeof(float);
    if (rows && sampling_ratio == 2 && roi_unroll_enabled()) {
      SMOT_ENSURE_SMEM((roi_align_rows_kernel<float, true, 2>), smem, "smot_roi_align_planar");
      roi_align_rows_kernel<float, true, 2><<<grid, 256, smem, st>>>(a, (float*)out, row_pitch, plane_pitch);
    } else if (rows) {
      SMOT_ENSURE_SMEM((roi_align_rows_kernel<float, true, 0>), smem, "smot_roi_align_planar");
      roi_align_rows_kernel<float, true, 0><<<grid, 256, smem, st>>>(a, (float*)out, row_pitch, plane_pitch);
    } else {
      SMOT_ENSURE_SMEM(roi_align_planar_kernel<float>, smem, "smot_roi_align_planar");
      roi_align_planar_kernel<float><<<grid, 256, smem, st>>>(a, (float*)out, row_pitch, plane_pitch);
    }
  } else if (dtype == SMOT_F16) {
    const size_t smem = (size_t)channels * RAP_TP * sizeof(__half);
    if (rows && sampling_ratio == 2 && roi_unroll_enabled()) {
      SMOT_ENSURE_SMEM((roi_align_rows_kernel<__half, true, 2>), smem, "smot_roi_align_planar");
      roi_align_rows_kernel<__half, true, 2><<<grid, 256, smem, st>>>(a, (__half*)out, row_pitch, plane_pitch);
    } else if (rows) {
      SMOT_ENSURE_SMEM((roi_align_rows_kernel<__half, true, 0>), smem, "smot_roi_align_planar");
      roi_align_rows_kernel<__half, true, 0><<<grid, 256, smem, st>>>(a, (__half*)out, row_pitch, plane_pitch);
    } else {
      SMOT_ENSURE_SMEM(roi_align_planar_kernel<__half>, smem, "smot_roi_align_planar");
      roi_align_planar_kernel<__half><<<grid, 256, smem, st>>>(a, (__half*)out, row_pitch, plane_pitch);
    }
  } else {
    SMOT_CHECK_ARG(false, "smot_roi_align_planar: bad dtype %d", dtype);
  }
  SMOT_CHECK_LAUNCH("smot_roi_align_planar");
  return SMOT_OK;
}

static int roi_align_nhwc(const char* who, const smot_pyramid* pyr, const long long* img_stride, int batch, const float* rois,
                          const float* level_boxes, const int* count, int max_rois, int channels, int res, int sampling_ratio,
                          void* out, int dtype, cudaStream_t st) {
  SMOT_CHECK_ARG(pyr && out && (rois || max_rois == 0), "%s: null argument", who);
  SMOT_CHECK_ARG(pyr->num_levels >= 1 && pyr->num_levels <= SMOT_MAX_LEVELS, "%s: num_levels %d", who, pyr->num_levels);
  SMOT_CHECK_ARG(channels > 0 && channels % 4 == 0 && res > 0 && max_rois >= 0, "%s: channels must be a multiple of 4", who);
  for (int l = 0; l < pyr->num_levels; ++l)
    SMOT_CHECK_ARG(pyr->feat[l] && pyr->ld[l] % 4 == 0 && pyr->H[l] > 0 && pyr->W[l] > 0 && pyr->pad[l] >= 0,
                   "%s: bad level %d", who, l);
  if (max_rois == 0 || batch == 0) return SMOT_OK;
  RoiArgs a;
  a.pyr = *pyr, a.rois = rois, a.level_boxes = level_boxes, a.count = count;
  a.max_rois = max_rois, a.channels = channels, a.res = res, a.sampling = sampling_ratio;
  a.batch = batch;
  for (int l = 0; l < SMOT_MAX_LEVELS; ++l) a.img_stride[l] = img_stride && l < pyr->num_levels ? img_stride[l] : 0;
  const long long rows_total = (long long)batch * max_rois;
  const long long warps = rows_total * res * res;
  const unsigned blocks = (unsigned)((warps * 32 + 255) / 256);
  const bool rows = roi_rows_enabled() && sampling_ratio > 0 && sampling_ratio <= 16 && res * sampling_ratio <= RAR_MAX_SAMPLES;
  // rows of bins per CTA: ~64+ bins, so that the per-CTA geometry + tables are amortised (7 x 7 -> the whole roi)
  int rpc = (64 + res - 1) / res;
  if (rpc > res) rpc = res;
  if (rpc * sampling_ratio > RAR_MAX_YS) rpc = RAR_MAX_YS / (sampling_ratio > 0 ? sampling_ratio : 1);
  const dim3 grid((unsigned)((res + rpc - 1) / rpc), (unsigned)rows_total);
  const bool unroll = roi_unroll_enabled() && sampling_ratio == 2;
  const bool batched = img_stride != nullptr;   // smot_roi_align_batched: the BATCHED instantiations
#define SMOT_ROI_LAUNCH(B_)                                                                                    \
  if (dtype == SMOT_F32 && rows && unroll)                                                                     \
    roi_align_rows_kernel<float, false, 2, B_><<<grid, 256, 0, st>>>(a, (float*)out, rpc, 0);                  \
  else if (dtype == SMOT_F16 && rows && unroll)                                                                \
    roi_align_rows_kernel<__half, false, 2, B_><<<grid, 256, 0, st>>>(a, (__half*)out, rpc, 0);                \
  else if (dtype == SMOT_F32 && rows)                                                                          \
    roi_align_rows_kernel<float, false, 0, B_><<<grid, 256, 0, st>>>(a, (float*)out, rpc, 0);                  \
  else if (dtype == SMOT_F16 && rows)                                                                          \
    roi_align_rows_kernel<__half, false, 0, B_><<<grid, 256, 0, st>>>(a, (__half*)out, rpc, 0);                \
  else if (dtype == SMOT_F32)                                                                                  \
    roi_align_kernel<float, B_><<<blocks, 256, 0, st>>>(a, (float*)out);                                       \
  else if (dtype == SMOT_F16)                                                                                  \
    roi_align_kernel<__half, B_><<<blocks, 256, 0, st>>>(a, (__half*)out);                                     \
  else                                                                                                         \
    SMOT_CHECK_ARG(false, "%s: bad dtype %d", who, dtype);
  if (batched) {
    SMOT_ROI_LAUNCH(true)
  } else {
    SMOT_ROI_LAUNCH(false)
  }
#undef SMOT_ROI_LAUNCH
  SMOT_CHECK_LAUNCH(who);
  return SMOT_OK;
}

extern "C" int smot_roi_align(const smot_pyramid* pyr, const float* rois, const float* level_boxes, const int* count,
                              int max_rois, int channels, int res, int sampling_ratio, void* out, int dtype,
                              void* stream) {
  return roi_align_nhwc("smot_roi_align", pyr, nullptr, 1, rois, level_boxes, count, max_rois, channels, res, sampling_ratio, out,
                        dtype, (cudaStream_t)stream);
}

extern "C" int smot_roi_align_batched(const smot_pyramid* pyr, const long long* image_stride, int batch, const float* rois,
                                      const int* count, int max_rois, int channels, int res, int sampling_ratio, void* out,
                                      int dtype, void* stream) {
  SMOT_CHECK_ARG(batch >= 0 && batch <= 65535 && image_stride && (count || batch <= 1),
                 "smot_roi_align_batched: batch %d needs image strides and per-image counts", batch);
  SMOT_CHECK_ARG((long long)batch * max_rois <= 65535, "smot_roi_align_batched: %d x %d rows exceed the grid", batch, max_rois);
  return roi_align_nhwc("smot_roi_align_batched", pyr, image_stride, batch, rois, nullptr, count, max_rois, channels, res,
                        sampling_ratio, out, dtype, (cudaStream_t)stream);
}
