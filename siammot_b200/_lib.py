"""ctypes binding of libsmot.so (include/smot.h).  There is NO fallback: if the CUDA library is
missing or an entry point fails, a RuntimeError is raised -- the product never computes on the CPU."""
import ctypes as C
import os

import torch  # noqa: F401  (loads libcudart / creates the CUDA context owner before libsmot.so)

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsmot.so")

F32, F16 = 0, 1
CONV_AUTO, CONV_SIMT, CONV_TCGEN05 = 0, 1, 2
MAX_LEVELS, MAX_ANCHORS = 5, 16
ABI_VERSION = 5
CONV_WS_COUNTER_BYTES = 65536
XCORR_ROW_PITCH, XCORR_PLANE = 40, 1208   # SMOT_XCORR_ROW_PITCH / SMOT_XCORR_PLANE: the channel-planar search-window layout


class ConvDesc(C.Structure):
    _fields_ = [("inp", C.c_void_p), ("weight", C.c_void_p), ("scale", C.c_void_p), ("bias", C.c_void_p),
                ("residual", C.c_void_p), ("out", C.c_void_p),
                ("batch", C.c_int), ("H", C.c_int), ("W", C.c_int), ("Cin", C.c_int), ("in_ld", C.c_int),
                ("OH", C.c_int), ("OW", C.c_int), ("Cout", C.c_int), ("out_ld", C.c_int), ("res_ld", C.c_int),
                ("KH", C.c_int), ("KW", C.c_int), ("stride", C.c_int), ("pad", C.c_int),
                ("relu", C.c_int), ("in_dtype", C.c_int), ("out_dtype", C.c_int), ("algo", C.c_int),
                ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t)]


class Pyramid(C.Structure):
    _fields_ = [("feat", C.c_void_p * MAX_LEVELS), ("H", C.c_int * MAX_LEVELS), ("W", C.c_int * MAX_LEVELS),
                ("ld", C.c_int * MAX_LEVELS), ("scale", C.c_float * MAX_LEVELS), ("pad", C.c_int * MAX_LEVELS),
                ("num_levels", C.c_int), ("k_min", C.c_int)]


class RpnLevel(C.Structure):
    _fields_ = [("head", C.c_void_p), ("head_ld", C.c_int), ("H", C.c_int), ("W", C.c_int), ("A", C.c_int),
                ("stride", C.c_int), ("cell_anchors", C.c_float * (MAX_ANCHORS * 4))]


_lib = None

# kernels launched by one call of each entry point (memsets not counted); used for bench.py's gpu_launches
KERNELS_PER_CALL = {"smot_conv2d": 1, "smot_image_to_nhwc": 1, "smot_maxpool2x2": 1, "smot_maxpool3x3s2": 1, "smot_deform_im2col3x3": 1, "smot_upsample_add": 1,
                    "smot_subsample2": 1, "smot_groupnorm_relu": 1, "smot_roi_align": 1, "smot_rpn_select": 6,
                    "smot_sort_nms": 3, "smot_box_decode": 1, "smot_track_combine": 1, "smot_track_combine_grouped": 1, "smot_xcorr": 1, "smot_emm_decode": 2,
                    "smot_roi_align_planar": 1, "smot_xcorr_planar": 1,
                    "smot_roi_align_batched": 1, "smot_rpn_select_batched": 6, "smot_box_decode_batched": 1, "smot_sort_nms_segmented": 4, "smot_xcorr_planar_mode": 1, "smot_xcorr_planar_cfg": 1,
                    "smot_resample_h_u8": 1, "smot_resample_v_normalize": 1}


def _declare(lib):
    vp, i, f, d, sz = C.c_void_p, C.c_int, C.c_float, C.c_double, C.c_size_t
    lib.smot_abi_version.restype = i
    lib.smot_last_error.restype = C.c_char_p
    sigs = {
        "smot_conv2d": [C.POINTER(ConvDesc), vp],
        "smot_conv2d_algo": [C.POINTER(ConvDesc)],
        "smot_image_to_nhwc": [vp, vp, i, i, i, i, i, vp],
        "smot_maxpool2x2": [vp, vp, i, i, i, i, i, i, i, vp],
        "smot_maxpool3x3s2": [vp, vp, i, i, i, i, i, i, i, vp],
        "smot_deform_im2col3x3": [vp, vp, vp, i, i, i, i, i, i, i, i, i, i, vp],
        "smot_upsample_add": [vp, i, i, i, vp, i, i, i, i, i, vp],
        "smot_subsample2": [vp, vp, i, i, i, i, i, i, vp],
        "smot_groupnorm_relu": [vp, vp, vp, i, i, i, i, i, f, i, i, vp],
        "smot_roi_align": [C.POINTER(Pyramid), vp, vp, vp, i, i, i, i, vp, i, vp],
        "smot_rpn_select": [C.POINTER(RpnLevel), i, i, i, f, f, i, i, i, i, vp, vp, vp, vp, sz, vp],
        "smot_sort_nms": [vp, i, vp, i, vp, i, f, f, i, i, vp, vp, vp, vp, vp, vp, sz, vp],
        "smot_box_decode": [vp, i, vp, vp, i, i, C.POINTER(C.c_float * 4), i, i, i, vp, vp, vp, vp],
        "smot_roi_align_batched": [C.POINTER(Pyramid), vp, i, vp, vp, i, i, i, i, vp, i, vp],
        "smot_rpn_select_batched": [C.POINTER(RpnLevel), vp, i, i, i, i, f, f, i, i, i, i, vp, vp, vp, vp, sz, vp],
        "smot_box_decode_batched": [vp, i, vp, vp, i, i, i, C.POINTER(C.c_float * 4), i, i, i, vp, vp, vp],
        "smot_sort_nms_segmented": [vp, vp, vp, i, i, i, f, f, i, i, vp, vp, vp, vp, sz, vp],
        "smot_track_combine": [vp, vp, i, vp, vp, i, vp, vp, vp, vp, i, i, vp, vp, vp, vp],
        "smot_track_combine_grouped": [vp, vp, i, vp, vp, i, vp, vp, vp, vp, i, i, vp, vp, vp, vp, vp],
        "smot_xcorr": [vp, vp, vp, i, i, i, i, i, vp],
        "smot_roi_align_planar": [C.POINTER(Pyramid), vp, vp, vp, i, i, i, i, vp, i, i, i, vp],
        "smot_xcorr_planar": [vp, vp, vp, i, i, vp],
        "smot_xcorr_planar_mode": [vp, vp, vp, i, i, i, vp],
        "smot_xcorr_planar_cfg": [vp, vp, vp, i, i, i, i, vp],
        "smot_emm_decode": [vp, i, i, i, i, i, vp, vp, vp, f, i, d, i, i, i, vp, vp, vp, vp, vp],
        "smot_resample_coeffs": [i, i, vp, vp],
        "smot_resample_h_u8": [vp, i, i, i, vp, vp, i, i, vp, i, vp],
        "smot_resample_v_normalize": [vp, i, i, i, vp, vp, i, i, C.POINTER(C.c_float * 3), C.POINTER(C.c_float * 3), i, vp, vp],
    }
    for name, args in sigs.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = i
    lib.smot_rpn_select_workspace.argtypes = [i, i]
    lib.smot_rpn_select_workspace.restype = sz
    lib.smot_sort_nms_workspace.argtypes = [i]
    lib.smot_sort_nms_workspace.restype = sz
    lib.smot_rpn_select_batched_workspace.argtypes = [i, i, i]
    lib.smot_rpn_select_batched_workspace.restype = sz
    lib.smot_sort_nms_segmented_workspace.argtypes = [i, i, i]
    lib.smot_sort_nms_segmented_workspace.restype = sz
    lib.smot_resample_ksize.argtypes = [i, i]
    lib.smot_resample_ksize.restype = i


def lib():
    """The loaded library; raises RuntimeError (never falls back) when it cannot be used."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("libsmot.so not built: run `python -m siammot_b200.build` "
                               "(or __graft_entry__.build()); there is no CPU / PyTorch fallback")
        try:
            l = C.CDLL(LIB_PATH)
        except OSError as e:
            raise RuntimeError("cannot load %s: %s" % (LIB_PATH, e))
        _declare(l)
        if l.smot_abi_version() != ABI_VERSION:
            raise RuntimeError("libsmot.so ABI version %d != binding %d: rebuild" % (l.smot_abi_version(), ABI_VERSION))
        _lib = l
    return _lib


def check(rc, what=""):
    if rc != 0:
        msg = lib().smot_last_error().decode("utf-8", "replace")
        raise RuntimeError("libsmot %s failed (code %d): %s" % (what, rc, msg))


def dtype_code(t):
    if t == torch.float32:
        return F32
    if t == torch.float16:
        return F16
    raise TypeError("unsupported activation dtype %s (float32 / float16 only)" % t)


def stream_ptr():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)
