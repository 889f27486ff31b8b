// FP32-FMA implicit-GEMM convolution (NHWC), the exact-arithmetic member of the conv family.
//
// GEMM view: M = batch*OH*OW output pixels, N = Cout, K = KH*KW*Cin (k = (r*KW + s)*Cin + c).
// A is gathered on the fly from the NHWC input (im2col never materialised), B is the
// [Cout][KH][KW][Cin] weight.  Block tile BM x BN x 16 staged in shared memory (register
// prefetch double buffering), TM x TN accumulators per thread, fp32 accumulation in k order.
// Epilogue fuses FrozenBN scale/bias (or conv bias), residual add and ReLU
// (reference: siammot/modelling/backbone/dla.py:43-57,181-189).
//
// This kernel is what SMOT_F32 runs end to end (bit-for-bit IEEE fp32 multiply-adds, no tensor
// cores), and in SMOT_F16 it covers the layers the wgmma kernel does not take (Cin % 64 != 0,
// strided, tiny Cout).
#include "common.cuh"

namespace smot {

struct ConvArgs {
  const void* in;
  const void* wt;
  const float* scale;
  const float* bias;
  const void* res;
  void* out;
  int batch, H, W, Cin, in_ld;
  int OH, OW, Cout, out_ld, res_ld;
  int KH, KW, stride, pad, relu;
  int M, K;
};

constexpr int BK = 16;

template <typename TI, typename TO, int BM, int BN, int TM, int TN, bool VEC>
__global__ void __launch_bounds__((BM / TM) * (BN / TN)) conv_simt_kernel(const ConvArgs p) {
  constexpr int NT = (BM / TM) * (BN / TN);
  constexpr int EA = BM * BK / NT;  // A elements per thread per k-tile (contiguous in k)
  constexpr int EB = BN * BK / NT;  // B elements per thread per k-tile (contiguous in k)
  static_assert(EA >= 1 && EB >= 1 && BK % EA == 0 && BK % EB == 0, "tile shape");
  static_assert(TM % 4 == 0 && (TN % 4 == 0), "micro tile must be float4 friendly");
  __shared__ __align__(16) float As[2][BK][BM];
  __shared__ __align__(16) float Bs[2][BK][BN];

  const TI* __restrict__ in = reinterpret_cast<const TI*>(p.in);
  const TI* __restrict__ wt = reinterpret_cast<const TI*>(p.wt);
  const int tid = threadIdx.x;
  const int m0 = blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;

  // ---- A loader coordinates: this thread always loads pixel a_m, k offsets [a_k, a_k+EA)
  const int a_ml = tid % BM;
  const int a_k = (tid / BM) * EA;
  const int a_m = m0 + a_ml;
  const bool a_ok = a_m < p.M;
  int ih0 = 0, iw0 = 0;
  const TI* a_img = in;
  if (a_ok) {
    int n_img = a_m / (p.OH * p.OW);
    int rem = a_m - n_img * (p.OH * p.OW);
    int oh = rem / p.OW, ow = rem - oh * p.OW;
    ih0 = oh * p.stride - p.pad;
    iw0 = ow * p.stride - p.pad;
    a_img = in + (size_t)n_img * p.H * p.W * p.in_ld;
  }
  // ---- B loader coordinates
  const int b_nl = tid / (BK / EB);
  const int b_k = (tid % (BK / EB)) * EB;
  const int b_n = n0 + b_nl;
  const bool b_ok = b_n < p.Cout;
  const TI* b_row = wt + (size_t)(b_ok ? b_n : 0) * p.K;

  float ra[EA], rb[EB];
  auto load_tile = [&](int kt) {
    const int k0 = kt * BK;
    if constexpr (VEC) {
      // Cin % BK == 0: the whole k-tile sits inside one filter tap
      const int tap = k0 / p.Cin;
      const int c0 = k0 - tap * p.Cin;
      const int r = tap / p.KW, s = tap - r * p.KW;
      const int ih = ih0 + r, iw = iw0 + s;
      const bool ok = a_ok && ih >= 0 && ih < p.H && iw >= 0 && iw < p.W;
      if (ok) {
        const TI* src = a_img + ((size_t)ih * p.W + iw) * p.in_ld + c0 + a_k;
#pragma unroll
        for (int e = 0; e < EA; e += 4) {
          float4 v = ld4(src + e);
          ra[e] = v.x, ra[e + 1] = v.y, ra[e + 2] = v.z, ra[e + 3] = v.w;
        }
      } else {
#pragma unroll
        for (int e = 0; e < EA; ++e) ra[e] = 0.f;
      }
      if constexpr (EB % 4 == 0) {
        if (b_ok) {
#pragma unroll
          for (int e = 0; e < EB; e += 4) {
            float4 v = ld4(b_row + k0 + b_k + e);
            rb[e] = v.x, rb[e + 1] = v.y, rb[e + 2] = v.z, rb[e + 3] = v.w;
          }
        } else {
#pragma unroll
          for (int e = 0; e < EB; ++e) rb[e] = 0.f;
        }
      } else {
#pragma unroll
        for (int e = 0; e < EB; ++e) rb[e] = b_ok ? to_f(b_row[k0 + b_k + e]) : 0.f;
      }
    } else {
#pragma unroll
      for (int e = 0; e < EA; ++e) {
        const int k = k0 + a_k + e;
        float v = 0.f;
        if (a_ok && k < p.K) {
          const int tap = k / p.Cin;
          const int c = k - tap * p.Cin;
          const int r = tap / p.KW, s = tap - r * p.KW;
          const int ih = ih0 + r, iw = iw0 + s;
          if (ih >= 0 && ih < p.H && iw >= 0 && iw < p.W) v = to_f(a_img[((size_t)ih * p.W + iw) * p.in_ld + c]);
        }
        ra[e] = v;
      }
#pragma unroll
      for (int e = 0; e < EB; ++e) {
        const int k = k0 + b_k + e;
        rb[e] = (b_ok && k < p.K) ? to_f(b_row[k]) : 0.f;
      }
    }
  };
  auto store_tile = [&](int buf) {
#pragma unroll
    for (int e = 0; e < EA; ++e) As[buf][a_k + e][a_ml] = ra[e];
#pragma unroll
    for (int e = 0; e < EB; ++e) Bs[buf][b_k + e][b_nl] = rb[e];
  };

  const int tx = tid % (BN / TN);
  const int ty = tid / (BN / TN);
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  const int nkt = (p.K + BK - 1) / BK;
  load_tile(0);
  store_tile(0);
  __syncthreads();
  for (int kt = 0; kt < nkt; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nkt) load_tile(kt + 1);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; i += 4) {
        float4 v = *reinterpret_cast<const float4*>(&As[buf][k][ty * TM + i]);
        a[i] = v.x, a[i + 1] = v.y, a[i + 2] = v.z, a[i + 3] = v.w;
      }
#pragma unroll
      for (int j = 0; j < TN; j += 4) {
        float4 v = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * TN + j]);
        b[j] = v.x, b[j + 1] = v.y, b[j + 2] = v.z, b[j + 3] = v.w;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nkt) {
      store_tile(buf ^ 1);
      __syncthreads();
    }
  }

  // ---- epilogue: scale/bias (unfused mul+add like FrozenBatchNorm2d), residual, ReLU
  TO* __restrict__ out = reinterpret_cast<TO*>(p.out);
  const TI* __restrict__ res = reinterpret_cast<const TI*>(p.res);
  const int nb = n0 + tx * TN;
  const bool vec_out = (p.Cout % 4 == 0) && (p.out_ld % 4 == 0) && (res == nullptr || p.res_ld % 4 == 0) &&
                       ((reinterpret_cast<uintptr_t>(out) & 15) == 0) &&
                       (res == nullptr || (reinterpret_cast<uintptr_t>(res) & 15) == 0);
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int m = m0 + ty * TM + i;
    if (m >= p.M) continue;
#pragma unroll
    for (int j0 = 0; j0 < TN; j0 += 4) {
      const int n = nb + j0;
      if (n >= p.Cout) continue;
      float v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int nn = n + j;
        float y = acc[i][j0 + j];
        if (nn < p.Cout) {
          if (p.scale) y = __fmul_rn(y, p.scale[nn]);
          if (p.bias) y = __fadd_rn(y, p.bias[nn]);
        }
        v[j] = y;
      }
      if (vec_out) {
        if (res) {
          float4 r = ld4(res + (size_t)m * p.res_ld + n);
          v[0] += r.x, v[1] += r.y, v[2] += r.z, v[3] += r.w;
        }
        if (p.relu) {
#pragma unroll
          for (int j = 0; j < 4; ++j) v[j] = fmaxf(v[j], 0.f);
        }
        st4(out + (size_t)m * p.out_ld + n, make_float4(v[0], v[1], v[2], v[3]));
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int nn = n + j;
          if (nn >= p.Cout) continue;
          float y = v[j];
          if (res) y += to_f(res[(size_t)m * p.res_ld + nn]);
          if (p.relu) y = fmaxf(y, 0.f);
          out[(size_t)m * p.out_ld + nn] = from_f<TO>(y);
        }
      }
    }
  }
}

template <typename TI, typename TO, int BM, int BN, int TM, int TN>
static void launch_cfg(const ConvArgs& a, bool vec, cudaStream_t st) {
  dim3 grid(ceil_div(a.M, BM), ceil_div(a.Cout, BN));
  dim3 block((BM / TM) * (BN / TN));
  if (vec)
    conv_simt_kernel<TI, TO, BM, BN, TM, TN, true><<<grid, block, 0, st>>>(a);
  else
    conv_simt_kernel<TI, TO, BM, BN, TM, TN, false><<<grid, block, 0, st>>>(a);
}

template <typename TI, typename TO>
static void launch_typed(const ConvArgs& a, cudaStream_t st) {
  // vector path: k-tiles never straddle a tap and all 16B/8B loads are aligned
  const bool vec = (a.Cin % BK == 0) && (a.in_ld % 4 == 0) &&
                   ((reinterpret_cast<uintptr_t>(a.in) & 15) == 0) && ((reinterpret_cast<uintptr_t>(a.wt) & 15) == 0);
  if (a.Cout <= 16)
    launch_cfg<TI, TO, 256, 16, 4, 4>(a, vec, st);
  else if (a.M >= 8192)
    launch_cfg<TI, TO, 128, 64, 8, 4>(a, vec, st);
  else
    launch_cfg<TI, TO, 64, 64, 4, 4>(a, vec, st);
}

int conv2d_simt(const smot_conv_desc* d, cudaStream_t st) {
  ConvArgs a;
  a.in = d->in, a.wt = d->weight, a.scale = d->scale, a.bias = d->bias, a.res = d->residual, a.out = d->out;
  a.batch = d->batch, a.H = d->H, a.W = d->W, a.Cin = d->Cin, a.in_ld = d->in_ld;
  a.OH = d->OH, a.OW = d->OW, a.Cout = d->Cout, a.out_ld = d->out_ld, a.res_ld = d->res_ld;
  a.KH = d->KH, a.KW = d->KW, a.stride = d->stride, a.pad = d->pad, a.relu = d->relu;
  a.M = d->batch * d->OH * d->OW;
  a.K = d->KH * d->KW * d->Cin;
  if (a.M == 0) return SMOT_OK;
  if (d->in_dtype == SMOT_F32 && d->out_dtype == SMOT_F32)
    launch_typed<float, float>(a, st);
  else if (d->in_dtype == SMOT_F16 && d->out_dtype == SMOT_F16)
    launch_typed<__half, __half>(a, st);
  else if (d->in_dtype == SMOT_F16 && d->out_dtype == SMOT_F32)
    launch_typed<__half, float>(a, st);
  else {
    set_error("smot_conv2d: unsupported dtype combination in=%d out=%d", d->in_dtype, d->out_dtype);
    return SMOT_ERR_UNSUPPORTED;
  }
  SMOT_CHECK_LAUNCH("smot_conv2d(simt)");
  return SMOT_OK;
}

}  // namespace smot
