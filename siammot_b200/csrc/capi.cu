// C-ABI glue: error reporting, conv dispatch (SIMT vs wgmma).
#include <stdarg.h>
#include <string.h>

#include <stdlib.h>

#include "common.cuh"

namespace smot {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int conv2d_simt(const smot_conv_desc* d, cudaStream_t st);
int conv2d_tc(const smot_conv_desc* d, cudaStream_t st);
bool conv2d_tc_supported(const smot_conv_desc* d);
int conv2d_hires(const smot_conv_desc* d, cudaStream_t st);
bool conv2d_hires_supported(const smot_conv_desc* d);
int conv2d_smalln(const smot_conv_desc* d, cudaStream_t st);
bool conv2d_smalln_supported(const smot_conv_desc* d);

}  // namespace smot

using namespace smot;

namespace smot {
int sm_count() {
  static int cached[SMOT_MAX_DEVICES];
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= SMOT_MAX_DEVICES) return 132;
  if (!cached[dev]) {
    int n = 0;
    cached[dev] = (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0) ? n : 132;
  }
  return cached[dev];
}

bool pdl_enabled() {
  static const bool on = [] {
    const char* e = getenv("SMOT_PDL");
    return !(e && e[0] == '0');
  }();
  return on;
}
}  // namespace smot

extern "C" int smot_abi_version(void) { return SMOT_ABI_VERSION; }
extern "C" const char* smot_last_error(void) { return g_err; }

static int check_conv(const smot_conv_desc* d) {
  SMOT_CHECK_ARG(d, "smot_conv2d: null descriptor");
  SMOT_CHECK_ARG(d->in && d->weight && d->out, "smot_conv2d: null tensor pointer");
  SMOT_CHECK_ARG(d->batch >= 0 && d->H > 0 && d->W > 0 && d->Cin > 0 && d->Cout > 0 && d->KH > 0 && d->KW > 0 &&
                     d->stride > 0 && d->pad >= 0,
                 "smot_conv2d: bad geometry");
  SMOT_CHECK_ARG(d->in_ld >= d->Cin && d->out_ld >= d->Cout, "smot_conv2d: pitch smaller than channel count");
  SMOT_CHECK_ARG(d->OH == (d->H + 2 * d->pad - d->KH) / d->stride + 1 && d->OW == (d->W + 2 * d->pad - d->KW) / d->stride + 1,
                 "smot_conv2d: OHxOW %dx%d inconsistent with input %dx%d k=%d s=%d p=%d", d->OH, d->OW, d->H, d->W, d->KH,
                 d->stride, d->pad);
  SMOT_CHECK_ARG(!d->residual || d->res_ld >= d->Cout, "smot_conv2d: residual pitch");
  SMOT_CHECK_ARG((d->in_dtype == SMOT_F32 || d->in_dtype == SMOT_F16) && (d->out_dtype == SMOT_F32 || d->out_dtype == SMOT_F16),
                 "smot_conv2d: bad dtype");
  return SMOT_OK;
}

extern "C" int smot_conv2d_algo(const smot_conv_desc* d) {
  if (check_conv(d)) return -1;
  return conv2d_tc_supported(d) ? SMOT_CONV_TCGEN05 : SMOT_CONV_SIMT;
}

extern "C" int smot_conv2d(const smot_conv_desc* d, void* stream) {
  int rc = check_conv(d);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  int algo = d->algo;
  if (algo == SMOT_CONV_AUTO) algo = conv2d_tc_supported(d) ? SMOT_CONV_TCGEN05 : SMOT_CONV_SIMT;
  if (algo == SMOT_CONV_TCGEN05) {
    SMOT_CHECK_ARG(conv2d_tc_supported(d), "smot_conv2d: tensor-core (wgmma) path does not support this descriptor");
    return conv2d_tc(d, st);
  }
  if (d->algo == SMOT_CONV_AUTO && conv2d_hires_supported(d)) return conv2d_hires(d, st);  // DLA stem / levels 0-1
  // SIMT family: warp-per-pixel kernel for Cout <= 16, register-tiled implicit GEMM otherwise
  if (d->algo == SMOT_CONV_AUTO && conv2d_smalln_supported(d)) return conv2d_smalln(d, st);
  return conv2d_simt(d, st);
}
