"""Builds tests/cpu_cuda/_kernels_cpu.so: the source text of selected libsmot kernels compiled by g++ over shim.h.
TEST INFRASTRUCTURE; see shim.h."""
import os
import re
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(REPO, "siammot_b200", "csrc")
OUT = os.path.join(HERE, "_kernels_cpu.so")


def _function_text(src, signature_regex):
    """Text of the top-level definition whose header matches: from the header to the first line that is a lone '}'."""
    m = re.search(signature_regex, src)
    assert m, signature_regex
    start = src.rfind("\n", 0, m.start()) + 1
    # include a preceding `template <...>` line
    prev = src.rfind("\n", 0, start - 1) + 1
    if src[prev:start].lstrip().startswith("template"):
        start = prev
    end = src.index("\n}\n", m.end()) + 3
    return src[start:end]


def _rows_kernel_text(roi, fp16=False):
    """roi_align_rows_kernel + its helpers (sample struct / function) for the host build: the dynamic shared memory is the
    shim's buffer, the static __shared__ tables become per-block arrays (the shim runs one block at a time)."""
    helpers = roi[roi.index("constexpr int RAR_MAX_SAMPLES"):roi.index("// SAMP: compile-time sampling ratio")]
    if not fp16:
        helpers = re.sub(r"template <> struct Raw4<__half>.*?\n", "", helpers)
        helpers = re.sub(r"__device__ __forceinline__ Raw4<__half> ld4raw.*?\n", "", helpers)
        helpers = re.sub(r"__device__ __forceinline__ float4 raw_to_f4\(const Raw4<__half>& r\) \{.*?\n\}\n", "", helpers, flags=re.S)
        helpers = re.sub(r"template <> __device__ __forceinline__ Raw4<__half> raw_zero<__half>\(\).*?\n", "", helpers)
    k = _function_text(roi, r"__global__ void __launch_bounds__\(256\) roi_align_rows_kernel")
    k = k.replace("extern __shared__ __align__(16) unsigned char rar_raw[];", "unsigned char* rar_raw = cpu_dynamic_smem;")
    k = k.replace("__shared__ RarTap xs[RAR_MAX_SAMPLES];", "static RarTap xs[RAR_MAX_SAMPLES];")
    k = k.replace("__shared__ RarTap ys[RAR_MAX_YS];", "static RarTap ys[RAR_MAX_YS];")
    return helpers + k


def generate():
    roi = open(os.path.join(CSRC, "roi_align.cu")).read()
    elt = open(os.path.join(CSRC, "elementwise.cu")).read()
    sel = open(os.path.join(CSRC, "select_nms.cu")).read()
    header = open(os.path.join(REPO, "include", "smot.h")).read()
    pyramid = re.search(r"typedef struct \{\s*const void\* feat\[SMOT_MAX_LEVELS\];.*?\} smot_pyramid;", header, re.S).group(0)
    parts = ['#include "shim.h"', "#define SMOT_MAX_LEVELS 5", pyramid, "namespace smot {",
             re.search(r"struct RoiArgs \{.*?\};", roi, re.S).group(0),
             re.search(r"constexpr int RAP_TP = \d+;[^\n]*", roi).group(0),
             _function_text(roi, r"__global__ void roi_align_kernel"),     # GPU-validated: validates the shim itself
             # the kernel declares its dynamic shared memory as an extern array: bind that name to the shim's buffer
             _function_text(roi, r"__global__ void __launch_bounds__\(256\) roi_align_planar_kernel")
             .replace("extern __shared__ __align__(16) unsigned char rap_raw[];", "unsigned char* rap_raw = cpu_dynamic_smem;"),
             _rows_kernel_text(roi),
             _function_text(elt, r"__global__ void maxpool3x3s2_kernel"),
             _function_text(elt, r"__global__ void deform_im2col3x3_kernel"),
             _function_text(sel, r"__global__ void track_combine_grouped_kernel"),
             "}  // namespace smot", """
using namespace smot;
extern "C" void cpu_roi_align_planar(const smot_pyramid* pyr, const float* rois, const float* level_boxes, const int* count,
                                     int max_rois, int channels, int res, int sampling, float* out, int row_pitch, int plane_pitch) {
  RoiArgs a;
  a.pyr = *pyr, a.rois = rois, a.level_boxes = level_boxes, a.count = count;
  a.max_rois = max_rois, a.channels = channels, a.res = res, a.sampling = sampling;
  cpu_launch(dim3(res, max_rois), dim3(256), [&] { roi_align_planar_kernel<float>(a, out, row_pitch, plane_pitch); });
}
extern "C" void cpu_roi_align_rows(const smot_pyramid* pyr, const float* rois, const float* level_boxes, const int* count, int max_rois,
                                   int channels, int res, int sampling, float* out, int row_pitch, int plane_pitch, int planar) {
  RoiArgs a;
  a.pyr = *pyr, a.rois = rois, a.level_boxes = level_boxes, a.count = count;
  a.max_rois = max_rois, a.channels = channels, a.res = res, a.sampling = sampling;
  // `planar`: 1 = planar rows; 0 = NHWC with the product's rows-per-CTA rule; 2 = NHWC, unrolled sampling-2 specialisation
  int rpc = (64 + res - 1) / res;
  if (rpc > res) rpc = res;
  if (planar == 1)
    cpu_launch(dim3(res, max_rois), dim3(256), [&] { roi_align_rows_kernel<float, true, 0>(a, out, row_pitch, plane_pitch); });
  else if (planar == 2)
    cpu_launch(dim3((res + rpc - 1) / rpc, max_rois), dim3(256), [&] { roi_align_rows_kernel<float, false, 2>(a, out, rpc, 0); });
  else
    cpu_launch(dim3((res + rpc - 1) / rpc, max_rois), dim3(256), [&] { roi_align_rows_kernel<float, false, 0>(a, out, rpc, 0); });
}
extern "C" void cpu_roi_align(const smot_pyramid* pyr, const float* rois, const float* level_boxes, const int* count, int max_rois,
                              int channels, int res, int sampling, float* out) {
  RoiArgs a;
  a.pyr = *pyr, a.rois = rois, a.level_boxes = level_boxes, a.count = count;
  a.max_rois = max_rois, a.channels = channels, a.res = res, a.sampling = sampling;
  const long long warps = (long long)max_rois * res * res;
  cpu_launch(dim3((unsigned)((warps * 32 + 255) / 256)), dim3(256), [&] { roi_align_kernel<float>(a, out); });
}
extern "C" void cpu_maxpool3x3s2(const float* in, float* out, int batch, int H, int W, int C, int in_ld, int out_ld) {
  const size_t total = (size_t)batch * ((H - 1) / 2 + 1) * ((W - 1) / 2 + 1) * (C / 4);
  cpu_launch(dim3((unsigned)((total + 63) / 64)), dim3(64), [&] { maxpool3x3s2_kernel<float>(in, out, batch, H, W, C, in_ld, out_ld); });
}
extern "C" void cpu_deform_im2col3x3(const float* in, const float* off, float* cols, int H, int W, int C, int in_ld, int off_ld,
                                     int OH, int OW, int out_ld, int stride) {
  const size_t total = (size_t)OH * OW * 9 * (C / 4);
  cpu_launch(dim3((unsigned)((total + 63) / 64)), dim3(64),
             [&] { deform_im2col3x3_kernel<float>(in, off, cols, H, W, C, in_ld, off_ld, OH, OW, out_ld, stride); });
}
extern "C" void cpu_track_combine_grouped(const float* det_boxes, const float* det_scores, int ncap, const float* dec_boxes,
                                          const float* dec_scores, int ncls, const int* labels, const float* conf, const int* valid,
                                          const float* active, int n, int tracktor, float* cat_boxes, float* cat_scores,
                                          int* zero_count, int* perm) {
  const int total = ncap + n;
  cpu_launch(dim3((total + 1 + 31) / 32), dim3(32), [&] {
    track_combine_grouped_kernel(det_boxes, det_scores, ncap, dec_boxes, dec_scores, ncls, labels, conf, valid, active, n, tracktor,
                                 cat_boxes, cat_scores, zero_count, perm);
  });
}
"""]
    path = os.path.join(HERE, "_kernels_cpu.cpp")
    with open(path, "w") as f:
        f.write("// GENERATED by tests/cpu_cuda/cpu_cuda_build.py from siammot_b200/csrc/*.cu -- do not edit\n" + "\n".join(parts) + "\n")
    return path


def _compile(src, out, extra=()):
    cmd = ["g++", "-std=c++20", "-O1", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-I", HERE] + list(extra) + [src, "-o", out]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("g++ failed:\n" + r.stdout[-4000:])
    return out


def build():
    return _compile(generate(), OUT)


OUT_TC = os.path.join(HERE, "_xcorr_cpu.so")
CUDA_INCLUDE = os.environ.get("CUDA_INCLUDE", "/usr/local/cuda/include")


def generate_xcorr():
    """xcorr_mma_kernel (GPU-validated) and xcorr_planar_kernel from csrc/emm.cu over shim_tc.h.  The inline-PTX wrappers are
    replaced by the shim's emulations (same names); the remaining asm statements in the kernel bodies (proxy fences, the
    %globaltimer read of the bounded wait) have no host meaning and are dropped."""
    emm = open(os.path.join(CSRC, "emm.cu")).read()
    consts_mma = emm[emm.index("constexpr int XM_CG = 16;"):emm.index("__device__ __forceinline__ void xm_ldmatrix_x4")]
    consts_planar = emm[emm.index("template <int CG>\nstruct XpGeom"):emm.index("__device__ __forceinline__ void xp_mbar_init")]
    k_mma = _function_text(emm, r"__global__ void __launch_bounds__\(XM_WARPS \* 32\) xcorr_mma_kernel")
    k_planar = _function_text(emm, r"__global__ void __launch_bounds__\(XpGeom<CG>::THREADS\) xcorr_planar_kernel")
    assert k_planar.lstrip().startswith("template <int MMA_MODE, int CG>")
    k_planar = _function_text(emm, r"__device__ __forceinline__ void xp_plane_mma") + k_planar
    consts_flat = emm[emm.index("constexpr int XF_MAX_UNITS"):emm.index("template <int MMA_MODE>\n__global__ void __launch_bounds__(XF_THREADS, 1) xcorr_flat_kernel")]
    k_flat = _function_text(emm, r"__global__ void __launch_bounds__\(XF_THREADS, 1\) xcorr_flat_kernel")
    k_planar += consts_flat + k_flat
    k_planar = re.sub(r"XP_STAMP\(\d\);", ";", k_planar)
    k_mma = k_mma.replace("extern __shared__ __align__(16) unsigned char xm_raw[];", "unsigned char* xm_raw = cpu_dynamic_smem;")
    k_planar = k_planar.replace("extern __shared__ __align__(128) unsigned char xp_raw[];", "unsigned char* xp_raw = cpu_dynamic_smem;")
    k_planar = re.sub(r'asm volatile\("fence[^"]*" ::: "memory"\);', ";", k_planar)
    k_planar = re.sub(r'asm volatile\("mov\.u64 %0, %globaltimer;" : "=l"\(now\)\);', "now = 0;", k_planar)
    assert "asm" not in k_planar and "asm" not in k_mma and "extern __shared__" not in k_planar + k_mma
    # the fp16 instantiations of the simple kernels ride in this translation unit (it has __half)
    roi = open(os.path.join(CSRC, "roi_align.cu")).read()
    elt = open(os.path.join(CSRC, "elementwise.cu")).read()
    header = open(os.path.join(REPO, "include", "smot.h")).read()
    pyramid = re.search(r"typedef struct \{\s*const void\* feat\[SMOT_MAX_LEVELS\];.*?\} smot_pyramid;", header, re.S).group(0)
    simple = ["#define SMOT_MAX_LEVELS 5", pyramid, "namespace smot {", re.search(r"struct RoiArgs \{.*?\};", roi, re.S).group(0),
              re.search(r"constexpr int RAP_TP = \d+;[^\n]*", roi).group(0),
              _function_text(roi, r"__global__ void roi_align_kernel"),
              _function_text(roi, r"__global__ void __launch_bounds__\(256\) roi_align_planar_kernel")
              .replace("extern __shared__ __align__(16) unsigned char rap_raw[];", "unsigned char* rap_raw = cpu_dynamic_smem;"),
              _rows_kernel_text(roi, fp16=True),
              _function_text(elt, r"__global__ void maxpool3x3s2_kernel"),
              _function_text(elt, r"__global__ void deform_im2col3x3_kernel"), "}  // namespace smot", """
extern "C" void cpu_roi_align_rows_h(const smot_pyramid* pyr, const float* rois, const float* level_boxes, const int* count, int max_rois,
                                     int channels, int res, int sampling, void* out, int row_pitch, int plane_pitch, int planar) {
  smot::RoiArgs a;
  a.pyr = *pyr, a.rois = rois, a.level_boxes = level_boxes, a.count = count;
  a.max_rois = max_rois, a.channels = channels, a.res = res, a.sampling = sampling;
  int rpc = (64 + res - 1) / res;
  if (rpc > res) rpc = res;
  if (planar == 1)
    cpu_launch(dim3(res, max_rois), dim3(256), [&] { smot::roi_align_rows_kernel<__half, true, 0>(a, (__half*)out, row_pitch, plane_pitch); });
  else if (planar == 2)
    cpu_launch(dim3((res + rpc - 1) / rpc, max_rois), dim3(256), [&] { smot::roi_align_rows_kernel<__half, false, 2>(a, (__half*)out, rpc, 0); });
  else
    cpu_launch(dim3((res + rpc - 1) / rpc, max_rois), dim3(256), [&] { smot::roi_align_rows_kernel<__half, false, 0>(a, (__half*)out, rpc, 0); });
}
extern "C" void cpu_deform_im2col3x3_h(const void* in, const float* off, void* cols, int H, int W, int C, int in_ld, int off_ld,
                                       int OH, int OW, int out_ld, int stride) {
  const size_t total = (size_t)OH * OW * 9 * (C / 4);
  cpu_launch(dim3((unsigned)((total + 63) / 64)), dim3(64), [&] {
    smot::deform_im2col3x3_kernel<__half>((const __half*)in, off, (__half*)cols, H, W, C, in_ld, off_ld, OH, OW, out_ld, stride);
  });
}
extern "C" void cpu_roi_align_h(const smot_pyramid* pyr, const float* rois, const float* level_boxes, const int* count, int max_rois,
                                int channels, int res, int sampling, void* out) {
  smot::RoiArgs a;
  a.pyr = *pyr, a.rois = rois, a.level_boxes = level_boxes, a.count = count;
  a.max_rois = max_rois, a.channels = channels, a.res = res, a.sampling = sampling;
  const long long warps = (long long)max_rois * res * res;
  cpu_launch(dim3((unsigned)((warps * 32 + 255) / 256)), dim3(256), [&] { smot::roi_align_kernel<__half>(a, (__half*)out); });
}
extern "C" void cpu_roi_align_planar_h(const smot_pyramid* pyr, const float* rois, const float* level_boxes, const int* count,
                                       int max_rois, int channels, int res, int sampling, void* out, int row_pitch, int plane_pitch) {
  smot::RoiArgs a;
  a.pyr = *pyr, a.rois = rois, a.level_boxes = level_boxes, a.count = count;
  a.max_rois = max_rois, a.channels = channels, a.res = res, a.sampling = sampling;
  cpu_launch(dim3(res, max_rois), dim3(256), [&] { smot::roi_align_planar_kernel<__half>(a, (__half*)out, row_pitch, plane_pitch); });
}
extern "C" void cpu_maxpool3x3s2_h(const void* in, void* out, int batch, int H, int W, int C, int in_ld, int out_ld) {
  const size_t total = (size_t)batch * ((H - 1) / 2 + 1) * ((W - 1) / 2 + 1) * (C / 4);
  cpu_launch(dim3((unsigned)((total + 63) / 64)), dim3(64),
             [&] { smot::maxpool3x3s2_kernel<__half>((const __half*)in, (__half*)out, batch, H, W, C, in_ld, out_ld); });
}
"""]
    parts = ['#include "shim_tc.h"'] + simple + ["namespace smot {", consts_mma, k_mma, consts_planar, k_planar, "}  // namespace smot", """
using namespace smot;
extern "C" void cpu_xcorr_mma(const void* x, const void* k, void* out, int n, int C) {
  cpu_launch_warps(dim3(C / XM_CG, n), dim3(XM_WARPS * 32), [&] { xcorr_mma_kernel((const __half*)x, (const __half*)k, (__half*)out, C); });
}
template <int MODE, int CG>
static void cpu_xcorr_planar_launch(const void* xp, const void* k, void* out, int n, int C) {
  cpu_launch_warps(dim3(C / CG, n), dim3(XpGeom<CG>::THREADS), [&] { xcorr_planar_kernel<MODE, CG>((const __half*)xp, (const __half*)k, (__half*)out, C); });
}
extern "C" int cpu_xcorr_planar_cfg(const void* xp, const void* k, void* out, int n, int C, int mode, int cg) {
  switch (mode * 32 + cg) {
    case 2: cpu_xcorr_planar_launch<0, 2>(xp, k, out, n, C); break;
    case 4: cpu_xcorr_planar_launch<0, 4>(xp, k, out, n, C); break;
    case 8: cpu_xcorr_planar_launch<0, 8>(xp, k, out, n, C); break;
    case 16: cpu_xcorr_planar_launch<0, 16>(xp, k, out, n, C); break;
    case 34: cpu_xcorr_planar_launch<1, 2>(xp, k, out, n, C); break;
    case 36: cpu_xcorr_planar_launch<1, 4>(xp, k, out, n, C); break;
    case 40: cpu_xcorr_planar_launch<1, 8>(xp, k, out, n, C); break;
    case 48: cpu_xcorr_planar_launch<1, 16>(xp, k, out, n, C); break;
    default: return 1;
  }
  return 0;
}
extern "C" void cpu_xcorr_planar(const void* xp, const void* k, void* out, int n, int C, int mode) {
  cpu_xcorr_planar_cfg(xp, k, out, n, C, mode, 16);
}
extern "C" int cpu_xcorr_flat(const void* xp, const void* k, void* out, int n, int C, int mode, int grid) {
  const int units = n * C / 4;
  if (C % 4 || (units + grid - 1) / grid > XF_MAX_UNITS) return 1;
  if (mode == 0)
    cpu_launch_warps(dim3(grid), dim3(XF_THREADS), [&] { xcorr_flat_kernel<0>((const __half*)xp, (const __half*)k, (__half*)out, C, units); });
  else
    cpu_launch_warps(dim3(grid), dim3(XF_THREADS), [&] { xcorr_flat_kernel<1>((const __half*)xp, (const __half*)k, (__half*)out, C, units); });
  return 0;
}
extern "C" int cpu_xcorr_plane_halves() { return XM_CSTRIDE; }
"""]
    path = os.path.join(HERE, "_xcorr_cpu.cpp")
    with open(path, "w") as f:
        f.write("// GENERATED by tests/cpu_cuda/cpu_cuda_build.py from siammot_b200/csrc/emm.cu -- do not edit\n" + "\n".join(parts) + "\n")
    return path


def build_xcorr():
    return _compile(generate_xcorr(), OUT_TC, ["-I", CUDA_INCLUDE])


if __name__ == "__main__":
    print(build())


OUT_HIRES = os.path.join(HERE, "_hires_cpu.so")


def generate_hires():
    """csrc/conv_hires.cu: the per-tile kernels of the stem / level0 (validated on the GPU against the oracle) and their
    persistent forms, over shim_tc.h (cp.async = immediate copy or zero fill, ldmatrix / mma.sync emulated).  The persistent
    kernels must reproduce the per-tile ones bit for bit."""
    src = open(os.path.join(CSRC, "conv_hires.cu")).read()
    body = src[src.index("template <int CIN, int COUT, int STRIDE>\nstruct Hires3"):src.index("// ---- dispatch")]
    args = re.search(r"struct HiresArgs \{.*?\};", src, re.S).group(0)
    body = body.replace("extern __shared__ __align__(128) unsigned char hs_raw[];", "unsigned char* hs_raw = cpu_dynamic_smem;")
    body = body.replace("extern __shared__ __align__(128) unsigned char hp_raw[];", "unsigned char* hp_raw = cpu_dynamic_smem;")
    body = body.replace("__shared__ __align__(16) __half ", "alignas(16) static __half ")
    assert "asm" not in body and "extern __shared__" not in body
    parts = ['#include "shim_tc.h"', "namespace smot {", args, """
inline float __fadd_rn(float a, float b) { return a + b; }   // -ffp-contract=off: plain IEEE operations
inline float __fmul_rn(float a, float b) { return a * b; }
inline uint32_t hs_smem(const void* p) { return cpu_smem_offset(p); }
inline void cp_async16(void* dst, const void* src, bool valid) { if (valid) std::memcpy(dst, src, 16); else std::memset(dst, 0, 16); }
inline void cp_async8(void* dst, const void* src, bool valid) { if (valid) std::memcpy(dst, src, 8); else std::memset(dst, 0, 8); }
inline void cp_async_wait_all() {}
inline void ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) { xm_ldmatrix_x4(addr, r0, r1, r2, r3); }
inline void mma_16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) { xm_mma(c, a, b0, b1); }
""", body, "}  // namespace smot", """
using namespace smot;
static HiresArgs hires_args(const void* in, const void* wt, const float* scale, const float* bias, void* out, int H, int W, int in_ld,
                            int out_ld, int relu) {
  HiresArgs a;
  a.in = (const __half*)in, a.wt = (const __half*)wt, a.scale = scale, a.bias = bias, a.out = (__half*)out;
  a.H = H, a.W = W, a.in_ld = in_ld, a.OH = H, a.OW = W, a.out_ld = out_ld, a.relu = relu;
  return a;
}
extern "C" void cpu_stem(const void* in, const void* wt, const float* scale, const float* bias, void* out, int batch, int H, int W,
                         int out_ld, int relu, int persistent_ctas) {
  const HiresArgs a = hires_args(in, wt, scale, bias, out, H, W, 4, out_ld, relu);
  if (persistent_ctas > 0) {
    const int tx = (W + HP_TW - 1) / HP_TW, ty = (H + HP_TH - 1) / HP_TH;
    cpu_launch_warps(dim3(persistent_ctas), dim3(256), [&] { stem7x7_persist_kernel(a, tx, ty, tx * ty * batch); });
  } else {
    cpu_launch_warps(dim3((W + ST_TW - 1) / ST_TW, (H + ST_TH - 1) / ST_TH, batch), dim3(256), [&] { stem7x7_hires_kernel(a); });
  }
}
extern "C" void cpu_conv3x3_c16(const void* in, const void* wt, const float* scale, const float* bias, void* out, int batch, int H,
                                int W, int in_ld, int out_ld, int relu, int persistent_ctas) {
  const HiresArgs a = hires_args(in, wt, scale, bias, out, H, W, in_ld, out_ld, relu);
  if (persistent_ctas > 0) {
    const int tx = (W + HP_TW - 1) / HP_TW, ty = (H + HP_TH - 1) / HP_TH;
    cpu_launch_warps(dim3(persistent_ctas), dim3(256), [&] { conv3x3_c16_persist_kernel(a, tx, ty, tx * ty * batch); });
  } else {
    using C = Hires3<16, 16, 1>;
    cpu_launch_warps(dim3((W + C::TW - 1) / C::TW, (H + C::TH - 1) / C::TH, batch), dim3(256), [&] { conv3x3_hires_kernel<16, 16, 1>(a); });
  }
}
extern "C" void cpu_conv3x3_s2(const void* in, const void* wt, const float* scale, const float* bias, void* out, int batch, int H,
                               int W, int cin, int in_ld, int out_ld, int relu, int persistent_ctas) {
  HiresArgs a = hires_args(in, wt, scale, bias, out, H, W, in_ld, out_ld, relu);
  a.OH = H / 2, a.OW = W / 2;
  if (persistent_ctas > 0) {
    if (cin == 16) {
      using P = S2Persist<16, 32>;
      const int tx = (a.OW + 31) / 32, ty = (a.OH + P::TH - 1) / P::TH;
      cpu_launch_warps(dim3(persistent_ctas), dim3(256), [&] { conv3x3_s2_persist_kernel<16, 32>(a, tx, ty, tx * ty * batch); });
    } else {
      using P = S2Persist<32, 64>;
      const int tx = (a.OW + 31) / 32, ty = (a.OH + P::TH - 1) / P::TH;
      cpu_launch_warps(dim3(persistent_ctas), dim3(256), [&] { conv3x3_s2_persist_kernel<32, 64>(a, tx, ty, tx * ty * batch); });
    }
  } else if (cin == 16) {
    using C = Hires3<16, 32, 2>;
    cpu_launch_warps(dim3((a.OW + C::TW - 1) / C::TW, (a.OH + C::TH - 1) / C::TH, batch), dim3(256), [&] { conv3x3_hires_kernel<16, 32, 2>(a); });
  } else {
    using C = Hires3<32, 64, 2>;
    cpu_launch_warps(dim3((a.OW + C::TW - 1) / C::TW, (a.OH + C::TH - 1) / C::TH, batch), dim3(256), [&] { conv3x3_hires_kernel<32, 64, 2>(a); });
  }
}
"""]
    path = os.path.join(HERE, "_hires_cpu.cpp")
    with open(path, "w") as f:
        f.write("// GENERATED by tests/cpu_cuda/cpu_cuda_build.py from siammot_b200/csrc/conv_hires.cu -- do not edit\n" + "\n".join(parts) + "\n")
    return path


def build_hires():
    return _compile(generate_hires(), OUT_HIRES, ["-I", CUDA_INCLUDE])


# ---- proposal selection / NMS (csrc/select_nms.cu) -------------------------------------------------------------------------
def _split_top_level(text):
    """Split a launch configuration `grid, block, smem, stream` at the commas outside parentheses."""
    parts, depth, cur = [], 0, ""
    for ch in text:
        depth += ch == "("
        depth -= ch == ")"
        if ch == "," and depth == 0:
            parts.append(cur.strip())
            cur = ""
        else:
            cur += ch
    return parts + [cur.strip()]


def _host_launches(text):
    """`kernel<<<grid, block, smem, st>>>(args);` -> a synchronous shim launch of the same grid (the host code around the
    launches -- argument checks, workspace carving, the shared-memory decision -- is the library's own text)."""
    def sub(m):
        kern, cfg, args = m.groups()
        c = _split_top_level(cfg)
        smem = c[2] if len(c) > 2 else "0"
        return "cpu_launch_smem(dim3(%s), dim3(%s), (size_t)(%s), [&] { %s(%s); });" % (c[0], c[1], smem, kern, args)
    out, n = re.subn(r"(\w+(?:<\w+>)?)<<<(.*?)>>>\((.*?)\);", sub, text, flags=re.S)
    assert n > 0 and "<<<" not in out
    return out


def generate_select(path, mutation=None):
    """csrc/select_nms.cu from its first constant to its end -- the sort / NMS, RPN, box-decode and scatter kernels AND the
    extern "C" entry points that size, carve and launch them -- plus float_key / iou_plus1 of csrc/common.cuh, over
    shim_warp.h.  `mutation` = (old, new[, old2, new2 ...]) textual substitutions applied to select_nms.cu first (each `old`
    must occur)."""
    sel = open(os.path.join(CSRC, "select_nms.cu")).read()
    common = open(os.path.join(CSRC, "common.cuh")).read()
    if mutation:
        for old, new in zip(mutation[0::2], mutation[1::2]):
            assert old in sel, old
            sel = sel.replace(old, new)
    body = sel[sel.index("constexpr int SN_THREADS"):]
    body = body.replace("extern __shared__ __align__(16) unsigned char smem_raw[];", "unsigned char* smem_raw = cpu_dynamic_smem;")
    body = re.sub(r"(?<!extern )__shared__ ", "static ", body)   # one block runs at a time: a block's statics are its shared memory
    body = _host_launches(body)
    assert "__shared__" not in body
    helpers = (_function_text(common, r"__device__ __forceinline__ uint32_t float_key") +
               _function_text(common, r"__device__ __forceinline__ float iou_plus1"))
    parts = ['#include "shim_warp.h"', '#include "smot.h"', r"""
#include <cstdarg>
typedef void* cudaStream_t;
static char cpu_error[512];
namespace smot {
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  std::vsnprintf(cpu_error, sizeof cpu_error, fmt, ap);
  va_end(ap);
}
}  // namespace smot
extern "C" const char* cpu_last_error() { return cpu_error; }
static int cpu_launches = 0;
extern "C" int cpu_launch_count() { return cpu_launches; }
#define SMOT_CHECK_ARG(cond, ...)   \
  do {                              \
    if (!(cond)) {                  \
      ::smot::set_error(__VA_ARGS__); \
      return SMOT_ERR_INVALID;      \
    }                               \
  } while (0)
#define SMOT_CHECK_LAUNCH(name) \
  do {                          \
  } while (0)
// the opt-in grant: the largest dynamic shared memory the kernel may be launched with (checked again at every launch)
#define SMOT_ENSURE_SMEM(kernel, bytes, what)                                                 \
  do {                                                                                        \
    if ((size_t)(bytes) > sizeof cpu_dynamic_smem) {                                          \
      ::smot::set_error("%s: %zu bytes of shared memory", what, (size_t)(bytes));             \
      return SMOT_ERR_CUDA;                                                                   \
    }                                                                                         \
  } while (0)
static void cpu_launch_smem(dim3 grid, dim3 block, size_t smem, const std::function<void()>& body) {
  if (smem > sizeof cpu_dynamic_smem) {
    std::fprintf(stderr, "launch with %zu bytes of dynamic shared memory\n", smem);
    std::abort();
  }
  ++cpu_launches;
  cpu_launch_warps(grid, block, body);
}
namespace smot {""", helpers, body]
    with open(path, "w") as f:
        f.write("// GENERATED by tests/cpu_cuda/cpu_cuda_build.py from siammot_b200/csrc/select_nms.cu -- do not edit\n" +
                "\n".join(parts) + "\n")
    return path


def build_select(out, mutation=None):
    """Compile generate_select's text into the shared library `out` (its .cpp is written beside it)."""
    return _compile(generate_select(os.path.splitext(out)[0] + ".cpp", mutation), out, ["-I", os.path.join(REPO, "include")])
