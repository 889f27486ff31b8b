"""Tensor-level wrappers over the C ABI (include/smot.h).

PyTorch is used for what it is here for: device memory, streams.  Every function launches
hand-written sm_90a kernels from libsmot.so on the current CUDA stream and raises RuntimeError on
failure; none has a CPU or torch-op fallback.

Activations are NHWC tensors (B, H, W, C); a channel slice ``buf[..., a:b]`` of a wider buffer is a
valid operand (its pixel pitch ``stride(-2)`` is passed as ``ld``), which is how the DLA roots read
their children without a concat (dla.py:183).
"""
import ctypes as C

import torch

from . import _lib
from ._lib import ConvDesc, Pyramid, RpnLevel, check, dtype_code, lib, stream_ptr


def _require_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("libsmot operands must be CUDA tensors (no CPU fallback)")


def _nhwc(t):
    """(B, H, W, C, ld) of an NHWC tensor/view whose pixels are laid out densely with pitch ld.
    A matrix of n rows is passed as shape (1, 1, n, C)."""
    if t.dim() != 4 or (t.shape[3] > 1 and t.stride(3) != 1):
        raise ValueError("expected an NHWC tensor with unit channel stride, got shape %s strides %s"
                         % (tuple(t.shape), t.stride()))
    B, H, W, Cc = t.shape
    ld = t.stride(2) if W > 1 else Cc
    if (H > 1 and t.stride(1) != W * ld) or (B > 1 and t.stride(0) != H * W * ld):
        raise ValueError("NHWC view is not pixel-dense: shape %s strides %s" % (tuple(t.shape), t.stride()))
    return B, H, W, Cc, ld


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def conv_workspace(device, nbytes=48 << 20):
    """Zeroed scratch for split-K convolutions (fp32 partial tiles + self-resetting arrival counters)."""
    return torch.zeros((nbytes,), dtype=torch.uint8, device=device)


def conv_desc(x, weight, out, scale=None, bias=None, residual=None, stride=1, pad=0, relu=False, algo=_lib.CONV_AUTO,
              workspace=None):
    """Build the smot_conv_desc for out = act(conv(x, weight)*scale + bias + residual)."""
    _require_cuda(x, weight, out, scale, bias, residual)
    B, H, W, Cin, in_ld = _nhwc(x)
    Bo, OH, OW, Cout, out_ld = _nhwc(out)
    if weight.dim() != 4 or not weight.is_contiguous() or weight.shape[0] != Cout or weight.shape[3] != Cin:
        raise ValueError("weight must be contiguous [Cout][KH][KW][Cin]; got %s for Cin=%d Cout=%d"
                         % (tuple(weight.shape), Cin, Cout))
    if weight.dtype != x.dtype or (residual is not None and residual.dtype != x.dtype):
        raise TypeError("weight / residual dtype must equal the input dtype")
    d = ConvDesc()
    d.inp, d.weight, d.scale, d.bias, d.residual, d.out = (x.data_ptr(), weight.data_ptr(),
                                                           scale.data_ptr() if scale is not None else None,
                                                           bias.data_ptr() if bias is not None else None,
                                                           residual.data_ptr() if residual is not None else None,
                                                           out.data_ptr())
    for t in (scale, bias):
        if t is not None and (t.dtype != torch.float32 or t.numel() != Cout or not t.is_contiguous()):
            raise ValueError("scale / bias must be contiguous fp32 [Cout]")
    d.batch, d.H, d.W, d.Cin, d.in_ld = B, H, W, Cin, in_ld
    d.OH, d.OW, d.Cout, d.out_ld = OH, OW, Cout, out_ld
    d.res_ld = _nhwc(residual)[4] if residual is not None else 0
    d.KH, d.KW, d.stride, d.pad = weight.shape[1], weight.shape[2], stride, pad
    d.relu = int(bool(relu))
    d.in_dtype, d.out_dtype, d.algo = dtype_code(x.dtype), dtype_code(out.dtype), algo
    d.workspace = workspace.data_ptr() if workspace is not None else None
    d.workspace_bytes = workspace.numel() * workspace.element_size() if workspace is not None else 0
    if Bo != B:
        raise ValueError("batch mismatch")
    return d


def conv2d(x, weight, scale=None, bias=None, residual=None, stride=1, pad=0, relu=False, out=None, out_dtype=None,
           algo=_lib.CONV_AUTO, workspace=None):
    B, H, W, _, _ = _nhwc(x)
    KH, KW = weight.shape[1], weight.shape[2]
    OH = (H + 2 * pad - KH) // stride + 1
    OW = (W + 2 * pad - KW) // stride + 1
    if out is None:
        out = torch.empty((B, OH, OW, weight.shape[0]), dtype=out_dtype or x.dtype, device=x.device)
    d = conv_desc(x, weight, out, scale, bias, residual, stride, pad, relu, algo, workspace)
    check(lib().smot_conv2d(C.byref(d), stream_ptr()), "smot_conv2d")
    return out


def conv2d_algo(x, weight, out, **kw):
    return lib().smot_conv2d_algo(C.byref(conv_desc(x, weight, out, **kw)))


def image_to_nhwc(chw, dtype, ld=4):
    _require_cuda(chw)
    Cc, H, W = chw.shape
    chw = chw.contiguous().float()
    out = torch.empty((1, H, W, ld), dtype=dtype, device=chw.device)
    check(lib().smot_image_to_nhwc(_ptr(chw), _ptr(out), Cc, H, W, ld, dtype_code(dtype), stream_ptr()), "smot_image_to_nhwc")
    return out[..., :Cc]


def maxpool2x2(x, out=None):
    _require_cuda(x)
    B, H, W, Cc, ld = _nhwc(x)
    if out is None:
        out = torch.empty((B, H // 2, W // 2, Cc), dtype=x.dtype, device=x.device)
    check(lib().smot_maxpool2x2(_ptr(x), _ptr(out), B, H, W, Cc, ld, _nhwc(out)[4], dtype_code(x.dtype), stream_ptr()),
          "smot_maxpool2x2")
    return out


def maxpool3x3s2(x, out=None):
    """F.max_pool2d(x, 3, 2, 1) on an NHWC map (the ResNet stem pool)."""
    _require_cuda(x)
    B, H, W, Cc, ld = _nhwc(x)
    if out is None:
        out = torch.empty((B, (H - 1) // 2 + 1, (W - 1) // 2 + 1, Cc), dtype=x.dtype, device=x.device)
    check(lib().smot_maxpool3x3s2(_ptr(x), _ptr(out), B, H, W, Cc, ld, _nhwc(out)[4], dtype_code(x.dtype), stream_ptr()),
          "smot_maxpool3x3s2")
    return out


def deform_im2col3x3(x, offsets, stride=1, out=None):
    """x (1,H,W,C) NHWC, offsets fp32 (1,OH,OW,>=18) -> columns (1,OH,OW,9*C) of a deformable 3x3 / pad 1 convolution."""
    _require_cuda(x, offsets)
    B, H, W, Cc, ld = _nhwc(x)
    Bo, OH, OW, _, old = _nhwc(offsets)
    assert B == 1 and Bo == 1 and offsets.dtype == torch.float32
    if out is None:
        out = torch.empty((1, OH, OW, 9 * Cc), dtype=x.dtype, device=x.device)
    check(lib().smot_deform_im2col3x3(_ptr(x), _ptr(offsets), _ptr(out), H, W, Cc, ld, old, OH, OW, _nhwc(out)[4], stride,
                                      dtype_code(x.dtype), stream_ptr()), "smot_deform_im2col3x3")
    return out


def upsample_add_(lateral, top):
    _require_cuda(lateral, top)
    _, H, W, Cc, lld = _nhwc(lateral)
    _, Ht, Wt, Ct, tld = _nhwc(top)
    assert Cc == Ct and lateral.dtype == top.dtype
    check(lib().smot_upsample_add(_ptr(top), Ht, Wt, tld, _ptr(lateral), H, W, lld, Cc, dtype_code(top.dtype), stream_ptr()),
          "smot_upsample_add")
    return lateral


def subsample2(x, out=None):
    _require_cuda(x)
    _, H, W, Cc, ld = _nhwc(x)
    if out is None:
        out = torch.empty((1, (H - 1) // 2 + 1, (W - 1) // 2 + 1, Cc), dtype=x.dtype, device=x.device)
    check(lib().smot_subsample2(_ptr(x), _ptr(out), H, W, Cc, ld, _nhwc(out)[4], dtype_code(x.dtype), stream_ptr()),
          "smot_subsample2")
    return out


def groupnorm_relu_(x, gamma, beta, groups, eps=1e-5, relu=True):
    _require_cuda(x, gamma, beta)
    B, H, W, Cc, ld = _nhwc(x)
    check(lib().smot_groupnorm_relu(_ptr(x), _ptr(gamma), _ptr(beta), B, H * W, Cc, ld, groups, eps, int(relu),
                                    dtype_code(x.dtype), stream_ptr()), "smot_groupnorm_relu")
    return x


def make_pyramid(feats, scales, pads=None, k_min=2):
    """feats: list of NHWC level maps (batch 1)."""
    p = Pyramid()
    n = len(scales)
    p.num_levels, p.k_min = n, k_min
    for l in range(n):
        _, H, W, _, ld = _nhwc(feats[l])
        p.feat[l], p.H[l], p.W[l], p.ld[l] = feats[l].data_ptr(), H, W, ld
        p.scale[l] = scales[l]
        p.pad[l] = pads[l] if pads is not None else 0
    return p


def roi_align(feats, rois, scales, res, sampling, level_boxes=None, pads=None, count=None, out=None, pyramid=None):
    """rois (n,4) fp32 xyxy.  Returns (n, res, res, C) in the feature dtype."""
    _require_cuda(rois, level_boxes, count, *feats)
    n = rois.shape[0]
    Cc = feats[0].shape[3]
    if out is None:
        out = torch.empty((n, res, res, Cc), dtype=feats[0].dtype, device=feats[0].device)
    if n == 0:
        return out
    p = pyramid or make_pyramid(feats, scales, pads)
    assert rois.dtype == torch.float32 and rois.is_contiguous()
    assert level_boxes is None or (level_boxes.dtype == torch.float32 and level_boxes.is_contiguous())
    check(lib().smot_roi_align(C.byref(p), _ptr(rois), _ptr(level_boxes), _ptr(count), n, Cc, res, sampling, _ptr(out),
                               dtype_code(feats[0].dtype), stream_ptr()), "smot_roi_align")
    return out


def rpn_levels(heads, strides, cell_anchors):
    """heads: list of fp32 (1,H,W,ld) tensors ([0,A) logits, then 4A deltas); cell_anchors: list of (A,4) CPU tensors."""
    arr = (RpnLevel * len(heads))()
    for l, h in enumerate(heads):
        _, H, W, _, ld = _nhwc(h)
        A = cell_anchors[l].shape[0]
        arr[l].head, arr[l].head_ld, arr[l].H, arr[l].W, arr[l].A, arr[l].stride = h.data_ptr(), ld, H, W, A, strides[l]
        flat = cell_anchors[l].reshape(-1).tolist()
        for i, v in enumerate(flat):
            arr[l].cell_anchors[i] = v
    return arr


def rpn_select(levels, pre_nms_top_n, post_nms_top_n, nms_thresh, min_size, fpn_post_nms_top_n, img_w, img_h, amodal,
               out_boxes, out_scores, out_count, workspace):
    check(lib().smot_rpn_select(levels, len(levels), pre_nms_top_n, post_nms_top_n, nms_thresh, float(min_size),
                                fpn_post_nms_top_n, img_w, img_h, int(amodal), _ptr(out_boxes), _ptr(out_scores),
                                _ptr(out_count), _ptr(workspace), workspace.numel() * workspace.element_size(),
                                stream_ptr()), "smot_rpn_select")


def rpn_select_workspace(num_levels, pre_nms_top_n, device):
    nbytes = lib().smot_rpn_select_workspace(num_levels, pre_nms_top_n)
    return torch.empty((nbytes,), dtype=torch.uint8, device=device)


def sort_nms_workspace(n_max, device):
    return torch.empty((max(lib().smot_sort_nms_workspace(n_max), 8),), dtype=torch.uint8, device=device)


def sort_nms(boxes, scores, out_count, n_max=None, count=None, min_score=-1e30, thresh=0.5, max_keep=None, tag=0,
             out_index=None, out_boxes=None, out_scores=None, out_tag=None, workspace=None, box_stride=4, score_stride=1):
    """Appends survivors at *out_count (device int32 scalar).  See smot.h."""
    _require_cuda(boxes, scores, out_count)
    if n_max is None:
        n_max = scores.shape[0]
    if max_keep is None:
        max_keep = n_max
    if workspace is None:
        workspace = sort_nms_workspace(n_max, boxes.device)
    check(lib().smot_sort_nms(_ptr(boxes), box_stride, _ptr(scores), score_stride, _ptr(count), n_max, min_score, thresh,
                              max_keep, tag, _ptr(out_index), _ptr(out_boxes), _ptr(out_scores), _ptr(out_tag),
                              _ptr(out_count), _ptr(workspace), workspace.numel(), stream_ptr()), "smot_sort_nms")


def box_decode(head, rois, ncls, weights, img_w, img_h, amodal, count=None, track_labels=None, out_boxes=None,
               out_scores=None):
    """head: fp32 (n, ld) [logits | per-class deltas]; returns boxes (n, ncls, 4), scores (n, ncls)."""
    _require_cuda(head, rois)
    n = rois.shape[0]
    if out_boxes is None:
        out_boxes = torch.empty((n, ncls, 4), dtype=torch.float32, device=head.device)
        out_scores = torch.empty((n, ncls), dtype=torch.float32, device=head.device)
    w4 = (C.c_float * 4)(*[float(w) for w in weights])
    check(lib().smot_box_decode(_ptr(head), head.stride(0), _ptr(rois), _ptr(count), n, ncls, C.byref(w4), img_w, img_h,
                                int(amodal), _ptr(track_labels), _ptr(out_boxes), _ptr(out_scores), stream_ptr()),
          "smot_box_decode")
    return out_boxes, out_scores


def xcorr(x, k, out=None):
    """x (n,S,S,C), k (n,T,T,C) NHWC -> (n,O,O,C)."""
    _require_cuda(x, k)
    n, S, _, Cc = x.shape
    T = k.shape[1]
    assert x.is_contiguous() and k.is_contiguous() and x.dtype == k.dtype
    O = S - T + 1
    if out is None:
        out = torch.empty((n, O, O, Cc), dtype=x.dtype, device=x.device)
    check(lib().smot_xcorr(_ptr(x), _ptr(k), _ptr(out), n, Cc, S, T, dtype_code(x.dtype), stream_ptr()), "smot_xcorr")
    return out


def roi_align_planar(feats, rois, scales, res, sampling, level_boxes=None, pads=None, count=None, out=None, pyramid=None,
                     row_pitch=_lib.XCORR_ROW_PITCH, plane_pitch=_lib.XCORR_PLANE):
    """smot_roi_align with a channel-planar result: returns (n, C, plane_pitch) in the feature dtype; window element
    (i, j) of channel c sits at [roi, c, i * row_pitch + j].  Elements outside the res x res windows are left as they are
    (zeros when the buffer is allocated here)."""
    _require_cuda(rois, level_boxes, count, *feats)
    n = rois.shape[0]
    Cc = feats[0].shape[3]
    if out is None:
        out = torch.zeros((n, Cc, plane_pitch), dtype=feats[0].dtype, device=feats[0].device)
    if n == 0:
        return out
    p = pyramid or make_pyramid(feats, scales, pads)
    assert rois.dtype == torch.float32 and rois.is_contiguous() and out.is_contiguous()
    assert level_boxes is None or (level_boxes.dtype == torch.float32 and level_boxes.is_contiguous())
    check(lib().smot_roi_align_planar(C.byref(p), _ptr(rois), _ptr(level_boxes), _ptr(count), n, Cc, res, sampling, _ptr(out),
                                      row_pitch, plane_pitch, dtype_code(feats[0].dtype), stream_ptr()), "smot_roi_align_planar")
    return out


def xcorr_planar(x_planar, k, out=None, mma_mode=None, channel_group=None):
    """x_planar (n, C, XCORR_PLANE) fp16 channel-planar 30x30 windows (row pitch XCORR_ROW_PITCH, columns 30/31 zero),
    k (n,15,15,C) NHWC fp16 -> (n,16,16,C) NHWC: the output of xcorr() on the same windows, bit for bit."""
    _require_cuda(x_planar, k)
    n, Cc, plane = x_planar.shape
    if x_planar.dtype != torch.float16 or k.dtype != torch.float16:
        raise TypeError("smot_xcorr_planar is the fp16 tensor-core correlation (got %s / %s)" % (x_planar.dtype, k.dtype))
    assert plane == _lib.XCORR_PLANE
    assert x_planar.is_contiguous() and k.is_contiguous() and tuple(k.shape) == (n, 15, 15, Cc)
    if out is None:
        out = torch.empty((n, 16, 16, Cc), dtype=torch.float16, device=k.device)
    if channel_group is not None:   # planes per CTA (2 / 4 / 8 / 16; 0 = flat form, one CTA per SM): same results, another grid
        check(lib().smot_xcorr_planar_cfg(_ptr(x_planar), _ptr(k), _ptr(out), n, Cc, 1 if mma_mode is None else int(mma_mode),
                                          int(channel_group), stream_ptr()), "smot_xcorr_planar")
    elif mma_mode is None:   # the library's default: trimmed MMA phase (SMOT_XCORR_PLANAR=1 selects the untrimmed one)
        check(lib().smot_xcorr_planar(_ptr(x_planar), _ptr(k), _ptr(out), n, Cc, stream_ptr()), "smot_xcorr_planar")
    else:
        check(lib().smot_xcorr_planar_mode(_ptr(x_planar), _ptr(k), _ptr(out), n, Cc, int(mma_mode), stream_ptr()), "smot_xcorr_planar")
    return out


def emm_decode(maps, sr, tboxes, hann, up, T, pad, use_centerness, sigma, img_w, img_h, amodal):
    """maps: fp32 (n,O,O,ld>=7).  Returns boxes (n,4), conf (n,), valid (n,) int32."""
    _require_cuda(maps, sr, tboxes, hann)
    n, O, _, ld = maps.shape[0], maps.shape[1], maps.shape[2], maps.stride(2)
    dev = maps.device
    boxes = torch.empty((n, 4), dtype=torch.float32, device=dev)
    conf = torch.empty((n,), dtype=torch.float32, device=dev)
    valid = torch.empty((n,), dtype=torch.int32, device=dev)
    scratch = torch.empty((max(n, 1),), dtype=torch.int64, device=dev)
    check(lib().smot_emm_decode(_ptr(maps), ld, n, O, up, T, _ptr(sr), _ptr(tboxes), _ptr(hann), float(pad),
                                int(use_centerness), float(sigma), img_w, img_h, int(amodal), _ptr(boxes), _ptr(conf),
                                _ptr(valid), _ptr(scratch), stream_ptr()), "smot_emm_decode")
    return boxes, conf, valid


# ---- batched detection stage (B images of one size; Engine.batch_plan) ------------------------------------------------------
def image_strides(maps):
    """Host array of the per-image element strides of NHWC maps (B, H, W, C): what the batched entry points add per image."""
    arr = (C.c_longlong * _lib.MAX_LEVELS)()
    for l, m in enumerate(maps):
        B, H, W, _, ld = _nhwc(m)
        arr[l] = H * W * ld
    return arr


def rpn_select_batched_workspace(num_levels, pre_nms_top_n, batch, device):
    nbytes = lib().smot_rpn_select_batched_workspace(num_levels, pre_nms_top_n, batch)
    return torch.empty((nbytes,), dtype=torch.uint8, device=device)


def sort_nms_segmented_workspace(batch, ncls, n_max, device):
    return torch.empty((max(lib().smot_sort_nms_segmented_workspace(batch, ncls, n_max), 8),), dtype=torch.uint8, device=device)


def rpn_select_batched(heads, levels, pre_nms_top_n, post_nms_top_n, nms_thresh, min_size, fpn_post_nms_top_n, img_w, img_h,
                       amodal, out_boxes, out_scores, out_count, workspace):
    """heads: the (B,H,W,ld) fp32 head maps ``levels`` (rpn_levels) describes; outputs (B,n,4), (B,n), (B,) int32."""
    _require_cuda(out_boxes, out_scores, out_count, *heads)
    strides = image_strides(heads)
    check(lib().smot_rpn_select_batched(levels, strides, heads[0].shape[0], len(levels), pre_nms_top_n, post_nms_top_n, nms_thresh,
                                        float(min_size), fpn_post_nms_top_n, img_w, img_h, int(amodal), _ptr(out_boxes),
                                        _ptr(out_scores), _ptr(out_count), _ptr(workspace),
                                        workspace.numel() * workspace.element_size(), stream_ptr()), "smot_rpn_select_batched")


def roi_align_batched(feats, rois, count, scales, res, sampling, out=None):
    """feats: (B,H,W,C) level maps; rois (B,n,4) fp32, count (B,) int32 -> (B*n, res, res, C)."""
    _require_cuda(rois, count, *feats)
    B, n = rois.shape[0], rois.shape[1]
    Cc = feats[0].shape[3]
    if out is None:
        out = torch.empty((B * n, res, res, Cc), dtype=feats[0].dtype, device=feats[0].device)
    p = make_pyramid(feats, scales)
    assert rois.dtype == torch.float32 and rois.is_contiguous() and count.dtype == torch.int32
    check(lib().smot_roi_align_batched(C.byref(p), image_strides(feats), B, _ptr(rois), _ptr(count), n, Cc, res, sampling, _ptr(out),
                                       dtype_code(feats[0].dtype), stream_ptr()), "smot_roi_align_batched")
    return out


def box_decode_batched(head, rois, count, ncls, weights, img_w, img_h, amodal, out_boxes=None, out_scores=None):
    """head: fp32 (B*n, ld); rois (B,n,4); count (B,) -> boxes (B*n, ncls, 4), scores (B*n, ncls)."""
    _require_cuda(head, rois, count)
    B, n = rois.shape[0], rois.shape[1]
    if out_boxes is None:
        out_boxes = torch.empty((B * n, ncls, 4), dtype=torch.float32, device=head.device)
        out_scores = torch.empty((B * n, ncls), dtype=torch.float32, device=head.device)
    w4 = (C.c_float * 4)(*[float(w) for w in weights])
    check(lib().smot_box_decode_batched(_ptr(head), head.stride(0), _ptr(rois), _ptr(count), B, n, ncls, C.byref(w4), img_w, img_h,
                                        int(amodal), _ptr(out_boxes), _ptr(out_scores), stream_ptr()), "smot_box_decode_batched")
    return out_boxes, out_scores


def sort_nms_segmented(boxes, scores, count, batch, ncls, min_score, thresh, max_keep, out_boxes, out_scores, out_block,
                       workspace=None):
    """boxes (B*n, ncls, 4), scores (B*n, ncls), count (B,) -> per-image blocks out_boxes (B,cap,4), out_scores (B,cap),
    out_block (B,1+cap) = count | labels.  See smot.h."""
    _require_cuda(boxes, scores, count, out_boxes, out_scores, out_block)
    n = boxes.shape[0] // batch
    cap = out_scores.shape[1]
    if workspace is None:
        workspace = sort_nms_segmented_workspace(batch, ncls, n, boxes.device)
    check(lib().smot_sort_nms_segmented(_ptr(boxes), _ptr(scores), _ptr(count), batch, n, ncls, min_score, thresh, max_keep, cap,
                                        _ptr(out_boxes), _ptr(out_scores), _ptr(out_block), _ptr(workspace), workspace.numel(),
                                        stream_ptr()), "smot_sort_nms_segmented")
