"""GPU parity of every C-ABI kernel against the CPU oracle / plain torch fp32, on seeded inputs.

Tolerances: SMOT_F32 kernels use IEEE fp32 multiply-adds, so they agree with the CPU oracle up to
summation order: 2e-5 relative to the output scale.  SMOT_F16 (fp16 storage, fp32 accumulate) is
compared with the oracle evaluated on the fp16-rounded inputs: 2e-3 relative (output rounding).
Integer / index outputs (NMS keep lists, arg-max, levels, counts) must be bit-exact.  Convolutions are checked element by
element against the float64 reference and bound of tests/launch_check.py (conv2d_checked).
"""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import prims
from oracle import siammot_oracle as orc

pytestmark = pytest.mark.gpu

DEV = "cuda"


def ops():
    from siammot_b200 import ops as _ops
    return _ops


def nhwc(x, dtype=torch.float32):
    return x.permute(0, 2, 3, 1).contiguous().to(DEV, dtype)


def nchw(x):
    return x.permute(0, 3, 1, 2).float().cpu()


def ohwi(w, dtype=torch.float32):
    return w.permute(0, 2, 3, 1).contiguous().to(DEV, dtype)


def rel_err(a, b):
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def tol(dtype):
    return 2e-5 if dtype == torch.float32 else 2e-3


def conv2d_checked(x, weight, scale=None, bias=None, residual=None, stride=1, pad=0, relu=False, out=None, out_dtype=None,
                   algo=0, workspace=None):
    """ops.conv2d, its output checked element by element against the float64 reference and bound of
    tests/launch_check.py (check_conv)."""
    import launch_check as lc
    B, H, W, _ = x.shape
    KH, KW = weight.shape[1], weight.shape[2]
    if out is None:
        out = torch.empty((B, (H + 2 * pad - KH) // stride + 1, (W + 2 * pad - KW) // stride + 1, weight.shape[0]),
                          dtype=out_dtype or x.dtype, device=x.device)
    d = ops().conv_desc(x, weight, out, scale, bias, residual, stride, pad, relu, algo, workspace)
    ck = lc.check_conv(lc.Memory(DEV), d, lambda: ops().conv2d(x, weight, scale, bias, residual, stride, pad, relu, out=out,
                                                               algo=algo, workspace=workspace))
    assert ck.max_ratio <= 1.0, "conv %s: |err|/bound %.3f at %s" % (lc.describe_conv(d), ck.max_ratio, ck.where)
    return out


def q(x, dtype):
    """Round through the storage dtype (so the oracle sees the same inputs)."""
    return x.to(dtype).float()


CONV_CASES = [
    # B, Cin, H, W, Cout, k, stride, pad, residual, relu, scale
    (1, 3, 37, 53, 16, 7, 1, 3, False, True, True),     # stem: generic (Cin=3) path, Cout<=16 tile
    (1, 16, 40, 56, 16, 3, 1, 1, False, True, True),    # level0: vector path, 256x16 tile
    (1, 16, 41, 57, 32, 3, 2, 1, False, True, True),    # level1: stride 2, odd size
    (1, 32, 96, 112, 64, 3, 2, 1, True, True, True),    # large-M tile (128x64) + residual
    (1, 64, 24, 40, 64, 3, 1, 1, True, True, True),     # small-M tile (64x64)
    (1, 128, 12, 20, 128, 1, 1, 0, False, False, False),  # FPN lateral: bias only
    (5, 128, 16, 16, 256, 3, 1, 1, False, False, False),  # EMM towers: batch of 16x16 maps, no bias/scale
    (1, 128, 30, 44, 15, 1, 1, 0, False, False, False),   # RPN predictor: Cout=15 (scalar epilogue)
    (1, 48, 9, 11, 20, 3, 1, 1, True, False, True),       # ragged everything
]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("case", CONV_CASES)
def test_conv2d(case, dtype):
    B, Cin, H, W, Cout, k, stride, pad, use_res, relu, use_scale = case
    g = torch.Generator().manual_seed(hash(case) % 1000)
    x = q(torch.randn(B, Cin, H, W, generator=g), dtype)
    w = q(torch.randn(Cout, Cin, k, k, generator=g) / math.sqrt(Cin * k * k), dtype)
    scale = (0.5 + torch.rand(Cout, generator=g)) if use_scale else None
    bias = torch.randn(Cout, generator=g)
    OH, OW = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    res = q(torch.randn(B, Cout, OH, OW, generator=g), dtype) if use_res else None
    out_dtype = torch.float32 if Cout == 15 else dtype
    got = conv2d_checked(nhwc(x, dtype), ohwi(w, dtype), scale.to(DEV) if scale is not None else None, bias.to(DEV),
                         nhwc(res, dtype) if res is not None else None, stride, pad, relu, out_dtype=out_dtype)
    torch.cuda.synchronize()
    assert got.dtype == out_dtype


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_conv2d_concat_free_root_and_fc(dtype):
    """1x1 'root' conv reading three producers through channel-slice views of one buffer, with the
    output written into a slice of another buffer (dla.py:183 torch.cat eliminated); FC as 1x1 conv."""
    g = torch.Generator().manual_seed(7)
    H, W = 14, 18
    parts = [q(torch.randn(1, c, H, W, generator=g), dtype) for c in (64, 64, 32)]
    w = q(torch.randn(48, 160, 1, 1, generator=g) / math.sqrt(160), dtype)
    scale, bias = 0.5 + torch.rand(48, generator=g), torch.randn(48, generator=g)
    buf = torch.zeros(1, H, W, 160, dtype=dtype, device=DEV)
    off = 0
    for p in parts:
        buf[..., off:off + p.shape[1]] = nhwc(p, dtype)
        off += p.shape[1]
    outbuf = torch.zeros(1, H, W, 112, dtype=dtype, device=DEV)
    conv2d_checked(buf, ohwi(w, dtype), scale.to(DEV), bias.to(DEV), relu=True, out=outbuf[..., 64:112])
    torch.cuda.synchronize()
    assert float(outbuf[..., :64].abs().max()) == 0.0
    # a 3x3 conv whose INPUT is a slice (pitch 160) of the buffer
    w3 = q(torch.randn(64, 64, 3, 3, generator=g) / 24.0, dtype)
    conv2d_checked(buf[..., 64:128], ohwi(w3, dtype), pad=1)
    # fully connected: 77 rows x 6272 -> 1024 (box head fc6 shape)
    xfc = q(torch.randn(77, 6272, generator=g), dtype)
    wfc = q(torch.randn(1024, 6272, generator=g) / math.sqrt(6272), dtype)
    bfc = torch.randn(1024, generator=g)
    conv2d_checked(xfc.to(DEV, dtype).view(1, 1, 77, 6272), wfc.to(DEV, dtype).view(1024, 1, 1, 6272), None,
                   bfc.to(DEV), relu=True)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_small_tensor_kernels(dtype):
    g = torch.Generator().manual_seed(3)
    x = q(torch.randn(2, 32, 22, 30, generator=g), dtype)
    assert torch.equal(nchw(ops().maxpool2x2(nhwc(x, dtype))), F.max_pool2d(x, 2, 2))
    top = q(torch.randn(1, 16, 11, 20, generator=g), dtype)
    lat = q(torch.randn(1, 16, 22, 40, generator=g), dtype)
    ref = lat + F.interpolate(top, size=(22, 40), mode="bilinear", align_corners=False)
    got = ops().upsample_add_(nhwc(lat, dtype), nhwc(top, dtype))
    assert rel_err(nchw(got), ref) <= tol(dtype)
    lat2 = q(torch.randn(1, 16, 23, 39, generator=g), dtype)  # non-2x size (the reason for the patch)
    ref2 = lat2 + F.interpolate(top, size=(23, 39), mode="bilinear", align_corners=False)
    assert rel_err(nchw(ops().upsample_add_(nhwc(lat2, dtype), nhwc(top, dtype))), ref2) <= tol(dtype)
    y = q(torch.randn(1, 8, 11, 21, generator=g), dtype)
    assert torch.equal(nchw(ops().subsample2(nhwc(y, dtype))), F.max_pool2d(y, 1, 2, 0))
    z = q(torch.randn(3, 128, 16, 16, generator=g), dtype) * 2 + 0.5
    gamma, beta = 0.5 + torch.rand(128, generator=g), torch.randn(128, generator=g)
    refz = F.relu(F.group_norm(z, 32, gamma, beta, 1e-5))
    gotz = ops().groupnorm_relu_(nhwc(z, dtype), gamma.to(DEV), beta.to(DEV), 32, 1e-5, True)
    assert rel_err(nchw(gotz), refz) <= max(tol(dtype), 1e-4)
    # register-resident kernel with a partial pixel loop (9x7 map), generic kernel (8 channels per group; 20x20 map)
    for shape, groups in (((2, 64, 9, 7), 16), ((2, 64, 16, 16), 8), ((1, 32, 20, 20), 8)):
        z = q(torch.randn(*shape, generator=g), dtype) * 1.5 - 0.3
        gamma, beta = 0.5 + torch.rand(shape[1], generator=g), torch.randn(shape[1], generator=g)
        refz = F.relu(F.group_norm(z, groups, gamma, beta, 1e-5))
        gotz = ops().groupnorm_relu_(nhwc(z, dtype), gamma.to(DEV), beta.to(DEV), groups, 1e-5, True)
        assert rel_err(nchw(gotz), refz) <= max(tol(dtype), 1e-4)
    img = torch.randn(3, 19, 23, generator=g)
    got_img = ops().image_to_nhwc(img.to(DEV), dtype)
    assert torch.equal(got_img.float().cpu()[0].permute(2, 0, 1), q(img, dtype))


def _pyramid(g, C, H, W, dtype):
    feats = [q(torch.randn(1, C, H >> i, W >> i, generator=g), dtype) for i in range(5)]
    return feats, [nhwc(f, dtype) for f in feats]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_roi_align_plain_and_padded(dtype):
    g = torch.Generator().manual_seed(11)
    C, H, W = 32, 48, 80  # stride-4 level of a 192x320 image
    feats, dfeats = _pyramid(g, C, H, W, dtype)
    scales = (0.25, 0.125, 0.0625, 0.03125)
    boxes = torch.tensor([[10., 20., 60., 150.], [100., 30., 180., 190.], [5., 5., 300., 185.], [250., 60., 290., 160.],
                          [-30., -20., 40., 50.], [0., 0., 319., 191.], [200., 100., 201., 101.], [310., 180., 400., 260.]])
    # plain 7x7 (box head) and 15x15 (template)
    for res in (7, 15):
        ref = orc.pool_rois(feats, boxes, boxes, scales, res, 2)
        got = ops().roi_align(dfeats, boxes.to(DEV), scales, res, 2)
        assert rel_err(nchw(got), ref) <= tol(dtype)
    # search-region pooling on the virtually padded pyramid (track_utils.py:87-107 eliminated)
    pad = 64
    sr = orc.search_region(boxes, pad, 1.0, 0)
    padded = orc.pad_features(feats, pad)
    ref = orc.pool_rois(padded, boxes, boxes, scales, 30, 2, rois=sr)
    pads = [int(pad / ((2 ** i) * 4)) for i in range(4)]
    got = ops().roi_align(dfeats, sr.to(DEV), scales, 30, 2, level_boxes=boxes.to(DEV), pads=pads)
    assert rel_err(nchw(got), ref) <= tol(dtype)
    # device-side count: rows >= count are zero
    cnt = torch.tensor([3], dtype=torch.int32, device=DEV)
    got = ops().roi_align(dfeats, boxes.to(DEV), scales, 7, 2, count=cnt)
    assert float(got[3:].abs().max()) == 0.0 and float(got[:3].abs().max()) > 0.0


def test_sort_nms_matches_oracle():
    g = torch.Generator().manual_seed(5)
    for n in (1, 37, 300, 1000, 2500):
        xy = torch.rand(n, 2, generator=g) * 300
        wh = torch.rand(n, 2, generator=g) * 120 + 2
        boxes = torch.cat([xy, xy + wh], 1)
        scores = torch.rand(n, generator=g)
        scores[n // 2:] = scores[:n - n // 2].clone()  # plenty of exact ties -> index order must decide
        for thr, max_keep in ((0.5, n), (0.7, 300)):
            keep = prims.nms_legacy(boxes, scores, thr)[:max_keep]
            cnt = torch.zeros(1, dtype=torch.int32, device=DEV)
            idx = torch.full((n,), -1, dtype=torch.int32, device=DEV)
            ob = torch.zeros((n, 4), device=DEV)
            osc = torch.zeros((n,), device=DEV)
            ops().sort_nms(boxes.to(DEV), scores.to(DEV), cnt, thresh=thr, max_keep=max_keep, out_index=idx,
                           out_boxes=ob, out_scores=osc)
            k = int(cnt.item())
            assert k == keep.numel()
            assert idx[:k].cpu().tolist() == keep.tolist()
            assert torch.equal(ob[:k].cpu(), boxes[keep]) and torch.equal(osc[:k].cpu(), scores[keep])
    # min_score filter, count, append semantics, sort-only mode
    boxes = torch.tensor([[0., 0., 10., 10.], [0., 0., 10., 10.], [20., 20., 30., 30.], [40., 40., 50., 50.]])
    scores = torch.tensor([0.9, 0.8, 0.03, 0.7])
    cnt = torch.tensor([2], dtype=torch.int32, device=DEV)  # two rows already present
    idx = torch.full((8,), -1, dtype=torch.int32, device=DEV)
    ops().sort_nms(boxes.to(DEV), scores.to(DEV), cnt, min_score=0.05, thresh=0.5, out_index=idx,
                   count=torch.tensor([4], dtype=torch.int32, device=DEV))
    assert int(cnt.item()) == 4 and idx.cpu().tolist()[:4] == [-1, -1, 0, 3]
    cnt.zero_()
    ops().sort_nms(boxes.to(DEV), scores.to(DEV), cnt, thresh=0.0, max_keep=3, out_index=idx)
    assert int(cnt.item()) == 3 and idx.cpu().tolist()[:3] == [0, 1, 3]


def _rpn_cfg(amodal=False):
    from siammot_b200.config import get_cfg
    cfg = get_cfg()
    cfg.INPUT.AMODAL = amodal
    return cfg


# 192x320: one or two chunks per level; 704x1280: 16 chunks merged out of shared memory; 1056x1920: 36 chunks, merged
# from global memory
@pytest.mark.parametrize("amodal,size", [(False, (192, 320)), (True, (192, 320)), (False, (704, 1280)), (False, (1056, 1920))])
def test_rpn_select_matches_oracle(amodal, size):
    cfg = _rpn_cfg(amodal)
    g = torch.Generator().manual_seed(21)
    (img_h, img_w), A = size, 3
    logits, deltas, heads = [], [], []
    for lvl in range(5):
        h, w = math.ceil(img_h / (4 << lvl)), math.ceil(img_w / (4 << lvl))
        lg = torch.randn(1, A, h, w, generator=g) * 2
        if lvl == 0:  # many exactly tied logits straddling the top-1000 cut (about 500 above, n/7 tied)
            lg.view(-1)[::7] = lg.view(-1).sort(descending=True).values[600]
        dl = torch.randn(1, 4 * A, h, w, generator=g) * 0.5
        logits.append(lg)
        deltas.append(dl)
        head = torch.zeros(1, h, w, 16)
        head[..., :A] = lg.permute(0, 2, 3, 1)
        head[..., A:5 * A] = dl.permute(0, 2, 3, 1)
        heads.append(head.to(DEV))
    ref_b, ref_s = orc.rpn_select(cfg, logits, deltas, img_w, img_h)
    R = cfg.MODEL.RPN
    cells = [prims.cell_anchors(R.ANCHOR_STRIDE[l], (R.ANCHOR_SIZES[l],), R.ASPECT_RATIOS) for l in range(5)]
    levels = ops().rpn_levels(heads, R.ANCHOR_STRIDE, cells)
    ws = ops().rpn_select_workspace(5, R.PRE_NMS_TOP_N_TEST, DEV)
    ob = torch.zeros((R.FPN_POST_NMS_TOP_N_TEST, 4), device=DEV)
    osc = torch.zeros((R.FPN_POST_NMS_TOP_N_TEST,), device=DEV)
    cnt = torch.zeros(1, dtype=torch.int32, device=DEV)
    ops().rpn_select(levels, R.PRE_NMS_TOP_N_TEST, R.POST_NMS_TOP_N_TEST, R.NMS_THRESH, R.MIN_SIZE,
                     R.FPN_POST_NMS_TOP_N_TEST, img_w, img_h, amodal, ob, osc, cnt, ws)
    k = int(cnt.item())
    assert k == ref_b.shape[0]
    assert (osc[:k].cpu() - ref_s).abs().max() <= 1e-6
    assert (ob[:k].cpu() - ref_b).abs().max() <= 1e-3


@pytest.mark.parametrize("tracks", [False, True])
def test_box_decode_matches_oracle(tracks):
    cfg = _rpn_cfg()
    g = torch.Generator().manual_seed(9)
    n, ncls = 50, 3
    logits = torch.randn(n, ncls, generator=g) * 2
    deltas = torch.randn(n, 4 * ncls, generator=g)
    xy = torch.rand(n, 2, generator=g) * 250
    boxes = torch.cat([xy, xy + torch.rand(n, 2, generator=g) * 100 + 4], 1)
    labels = torch.randint(1, ncls, (n,), generator=g) if tracks else None
    head = torch.cat([logits, deltas], 1).to(DEV)
    gb, gs = ops().box_decode(head, boxes.to(DEV), ncls, cfg.MODEL.ROI_HEADS.BBOX_REG_WEIGHTS, 320, 192, False,
                              track_labels=labels.to(DEV, torch.int32) if tracks else None)
    prob = F.softmax(logits, -1)
    dec = prims.clip_boxes(prims.box_decode(deltas, boxes, cfg.MODEL.ROI_HEADS.BBOX_REG_WEIGHTS).reshape(-1, 4), 320, 192)
    if tracks:
        cp = prob.clone()
        prob[:] = 0
        ar = torch.arange(n)
        prob[ar, labels] = cp[ar, labels] + 1.0
    assert (gs.cpu() - prob).abs().max() <= 1e-6
    assert (gb.cpu().reshape(-1, 4) - dec).abs().max() <= 1e-3


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("geom", [(30, 15, 128), (30, 15, 32), (35, 7, 32), (12, 5, 8)])
def test_xcorr_matches_oracle(geom, dtype):
    S, T, C = geom
    g = torch.Generator().manual_seed(S + T)
    for n in (1, 7):
        x = q(torch.randn(n, C, S, S, generator=g), dtype)
        k = q(torch.randn(n, C, T, T, generator=g), dtype)
        ref = orc.xcorr_depthwise(x, k)
        got = ops().xcorr(nhwc(x, dtype), nhwc(k, dtype))
        assert rel_err(nchw(got), ref) <= tol(dtype)


@pytest.mark.parametrize("amodal", [False, True])
def test_emm_decode_matches_oracle(amodal):
    g = torch.Generator().manual_seed(13)
    n, O, up, T, pad = 9, 16, 16, 15, 512
    cls = torch.randn(n, 2, O, O, generator=g)
    ctr = torch.randn(n, 1, O, O, generator=g)
    reg = F.relu(torch.randn(n, 4, O, O, generator=g) * 20 + 40)
    cxy = torch.rand(n, 2, generator=g) * torch.tensor([1280., 704.])
    wh = torch.rand(n, 2, generator=g) * 150 + 20
    tboxes = torch.cat([cxy - wh / 2, cxy + wh / 2], 1)
    tboxes[0] = torch.tensor([1270., 690., 1400., 800.])  # mostly outside: clipped, maybe empty
    sr = orc.search_region(tboxes, pad, 1.0, 0)
    ref_bb, ref_conf = orc.emm_decode(cls, ctr, reg, sr, tboxes, pad, T, True, 0.4)
    maps = torch.zeros(n, O, O, 8)
    maps[..., 0:2] = cls.permute(0, 2, 3, 1)
    maps[..., 2:3] = ctr.permute(0, 2, 3, 1)
    maps[..., 3:7] = reg.permute(0, 2, 3, 1)
    hann = torch.hann_window(O * up, dtype=torch.float)
    bb, conf, valid = ops().emm_decode(maps.to(DEV), sr.to(DEV), tboxes.to(DEV), hann.to(DEV), up, T, pad, True, 0.4,
                                       1280, 704, amodal)
    if not amodal:
        ref_bb = prims.clip_boxes(ref_bb, 1280, 704)
        ref_valid = prims.nonempty_mask(ref_bb)
    else:
        ref_valid = torch.ones(n, dtype=torch.bool)
    assert valid.cpu().bool().tolist() == ref_valid.tolist()
    assert (conf.cpu() - ref_conf).abs().max() <= 1e-5
    assert (bb.cpu() - ref_bb).abs().max() <= 1e-3


TC_CASES = [
    # B, Cin, H, W, Cout, k, residual, relu, scale
    (1, 64, 176, 320, 64, 3, True, True, True),     # level2 block conv: 440 tiles x BN 64
    (1, 128, 88, 160, 128, 3, True, True, True),    # level3: BN 128 path? (110 tiles x 1 -> BN 64)
    (1, 256, 44, 80, 256, 3, False, True, True),    # level4, ragged tile rows (44 = 5.5 x 8)
    (1, 512, 22, 40, 512, 3, True, True, True),     # level5, ragged both ways, K = 4608
    (1, 448, 88, 160, 128, 1, False, True, True),   # root over a 448-channel concat buffer
    (1, 128, 11, 20, 128, 3, False, False, False),  # P6-sized map, bias only
    (30, 128, 16, 16, 256, 3, False, False, False),  # EMM towers at 30 tracks
    (1, 128, 176, 320, 128, 3, False, True, False),  # RPN conv on P2: BN 128
]


@pytest.mark.parametrize("case", TC_CASES)
def test_conv2d_tcgen05_matches_oracle_and_simt(case):
    """The wgmma/TMA member of the conv family and the SIMT member on the same fp16 operands, each within the float64
    bound of tests/launch_check.py."""
    from siammot_b200 import _lib
    B, Cin, H, W, Cout, k, use_res, relu, use_scale = case
    g = torch.Generator().manual_seed(Cin + H)
    dt = torch.float16
    x = q(torch.randn(B, Cin, H, W, generator=g), dt)
    w = q(torch.randn(Cout, Cin, k, k, generator=g) / math.sqrt(Cin * k * k), dt)
    scale = (0.5 + torch.rand(Cout, generator=g)) if use_scale else None
    bias = torch.randn(Cout, generator=g)
    res = q(torch.randn(B, Cout, H, W, generator=g), dt) if use_res else None
    dx, dw = nhwc(x, dt), ohwi(w, dt)
    ds, db = (scale.to(DEV) if scale is not None else None), bias.to(DEV)
    dr = nhwc(res, dt) if res is not None else None
    out = torch.empty((B, H, W, Cout), dtype=dt, device=DEV)
    assert ops().conv2d_algo(dx, dw, out, scale=ds, bias=db, residual=dr, pad=k // 2, relu=relu) == _lib.CONV_TCGEN05
    conv2d_checked(dx, dw, ds, db, dr, 1, k // 2, relu, algo=_lib.CONV_TCGEN05)
    conv2d_checked(dx, dw, ds, db, dr, 1, k // 2, relu, algo=_lib.CONV_SIMT)
    torch.cuda.synchronize()


def test_conv2d_tcgen05_channel_slices_and_fc():
    from siammot_b200 import _lib
    g = torch.Generator().manual_seed(77)
    dt = torch.float16
    H, W = 24, 40
    buf = (torch.randn(1, H, W, 320, generator=g)).to(DEV, dt)
    w3 = q(torch.randn(64, 128, 3, 3, generator=g) / 34.0, dt)
    outbuf = torch.zeros(1, H, W, 192, dtype=dt, device=DEV)
    x_view, o_view = buf[..., 64:192], outbuf[..., 128:192]
    res_view = buf[..., 256:320]
    assert ops().conv2d_algo(x_view, ohwi(w3, dt), o_view, residual=res_view, pad=1, relu=True) == _lib.CONV_TCGEN05
    conv2d_checked(x_view, ohwi(w3, dt), residual=res_view, pad=1, relu=True, out=o_view)
    torch.cuda.synchronize()
    assert float(outbuf[..., :128].abs().max()) == 0.0
    for rows in (300, 30, 128):
        xfc = q(torch.randn(rows, 6272, generator=g), dt)
        wfc = q(torch.randn(1024, 6272, generator=g) / math.sqrt(6272), dt)
        bfc = torch.randn(1024, generator=g)
        conv2d_checked(xfc.to(DEV, dt).view(1, 1, rows, 6272), wfc.to(DEV, dt).view(1024, 1, 1, 6272), None,
                       bfc.to(DEV), relu=True, algo=_lib.CONV_TCGEN05)


@pytest.mark.parametrize("case", [(1, 64, 88, 160, 128), (1, 128, 44, 80, 256), (1, 256, 22, 40, 512), (2, 64, 32, 48, 64)])
def test_conv2d_tcgen05_stride2(case):
    """3x3 stride-2 convs of the DLA trees through the strided TMA box (elementStrides = 2)."""
    from siammot_b200 import _lib
    B, Cin, H, W, Cout = case
    g = torch.Generator().manual_seed(Cin + W)
    dt = torch.float16
    x = q(torch.randn(B, Cin, H, W, generator=g), dt)
    w = q(torch.randn(Cout, Cin, 3, 3, generator=g) / math.sqrt(Cin * 9), dt)
    scale, bias = 0.5 + torch.rand(Cout, generator=g), torch.randn(Cout, generator=g)
    out = torch.empty((B, H // 2, W // 2, Cout), dtype=dt, device=DEV)
    args = (nhwc(x, dt), ohwi(w, dt), scale.to(DEV), bias.to(DEV), None, 2, 1, True)
    assert ops().conv2d_algo(args[0], args[1], out, scale=args[2], bias=args[3], stride=2, pad=1, relu=True) == _lib.CONV_TCGEN05
    conv2d_checked(*args, algo=_lib.CONV_TCGEN05)
    conv2d_checked(*args, algo=_lib.CONV_SIMT)
    torch.cuda.synchronize()


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_conv2d_small_cout_kernel(dtype):
    """Cout <= 16 layers (warp-per-pixel kernel): EMM heads 3x3 (3 / 4 outputs, input = channel slice of the
    tower buffer), box predictor FC 1024 -> 10, RPN predictor 1x1 -> 15, all with fp32 outputs."""
    g = torch.Generator().manual_seed(31)
    tower = q(torch.randn(7, 256, 16, 16, generator=g), dtype)
    dtower = nhwc(tower, dtype)
    maps = torch.zeros(7, 16, 16, 8, dtype=torch.float32, device=DEV)
    for (lo, hi, cout, off, relu) in ((0, 128, 3, 0, False), (128, 256, 4, 3, True)):
        w = q(torch.randn(cout, 128, 3, 3, generator=g) / 34.0, dtype)
        b = torch.randn(cout, generator=g)
        conv2d_checked(dtower[..., lo:hi], ohwi(w, dtype), None, b.to(DEV), pad=1, relu=relu, out=maps[..., off:off + cout])
    assert float(maps[..., 7].abs().max()) == 0.0
    for rows in (300, 30, 1):
        x = q(torch.randn(rows, 1024, generator=g), dtype)
        w = q(torch.randn(10, 1024, generator=g) / 32.0, dtype)
        b = torch.randn(10, generator=g)
        out = torch.zeros(1, 1, rows, 12, dtype=torch.float32, device=DEV)
        conv2d_checked(x.to(DEV, dtype).view(1, 1, rows, 1024), w.to(DEV, dtype).view(10, 1, 1, 1024), None, b.to(DEV),
                       out=out[..., :10])
        assert float(out[..., 10:].abs().max()) == 0.0
    # RPN predictor: 1x1, 128 -> 15 (objectness + deltas), fp32 head with pitch 16; ragged pixel counts, batch 2
    for (B, H, W) in ((1, 22, 40), (1, 11, 20), (2, 5, 7), (1, 44, 80)):
        x = q(torch.randn(B, 128, H, W, generator=g), dtype)
        w = q(torch.randn(15, 128, 1, 1, generator=g) / 11.0, dtype)
        b = torch.randn(15, generator=g)
        head = torch.zeros(B, H, W, 16, dtype=torch.float32, device=DEV)
        conv2d_checked(nhwc(x, dtype), ohwi(w, dtype), None, b.to(DEV), out=head[..., :15])
        assert float(head[..., 15].abs().max()) == 0.0
    # fp16 output with scale + bias + ReLU (the generic epilogue)
    x = q(torch.randn(2, 64, 9, 13, generator=g), dtype)
    w = q(torch.randn(8, 64, 3, 3, generator=g) / 24.0, dtype)
    sc, b = torch.rand(8, generator=g) + 0.5, torch.randn(8, generator=g)
    conv2d_checked(nhwc(x, dtype), ohwi(w, dtype), sc.to(DEV), b.to(DEV), pad=1, relu=True)


HIRES_CASES = [
    # name, Cin, Cout, k, stride, H, W
    ("stem", 3, 16, 7, 1, 72, 104),
    ("level0", 16, 16, 3, 1, 72, 104),
    ("level1", 16, 32, 3, 2, 72, 104),
    ("level2.tree1.conv1", 32, 64, 3, 2, 36, 52),
    ("level0_ragged", 16, 16, 3, 1, 13, 37),
]


@pytest.mark.parametrize("case", HIRES_CASES)
def test_conv2d_hires_kernels(case):
    """mma.sync halo-tile kernels of the DLA stem / levels 0-1 (fp16) and the SIMT kernel, each within the float64 bound."""
    from siammot_b200 import _lib
    name, Cin, Cout, k, stride, H, W = case
    g = torch.Generator().manual_seed(len(name) + H)
    dt = torch.float16
    x = q(torch.randn(2, Cin, H, W, generator=g), dt)
    w = q(torch.randn(Cout, Cin, k, k, generator=g) / math.sqrt(Cin * k * k), dt)
    scale, bias = 0.5 + torch.rand(Cout, generator=g), torch.randn(Cout, generator=g)
    if Cin == 3:
        buf = torch.zeros(2, H, W, 4, dtype=dt, device=DEV)
        buf[..., :3] = nhwc(x, dt)
        dx = buf[..., :3]
    else:
        dx = nhwc(x, dt)
    args = (dx, ohwi(w, dt), scale.to(DEV), bias.to(DEV), None, stride, k // 2, True)
    conv2d_checked(*args)                       # AUTO -> hires kernel
    conv2d_checked(*args, algo=_lib.CONV_SIMT)
    torch.cuda.synchronize()


@pytest.mark.parametrize("case", [("stem", 3, 16, 7, 1, 2, 704, 1280), ("level0", 16, 16, 3, 1, 1, 352, 640), ("stem", 3, 16, 7, 1, 1, 100, 70),
                                  ("level0", 16, 16, 3, 1, 2, 75, 130), ("level1", 16, 32, 3, 2, 2, 704, 1280), ("level1", 16, 32, 3, 2, 1, 70, 132),
                                  ("level2.tree1.conv1", 32, 64, 3, 2, 2, 352, 640), ("level2.tree1.conv1", 32, 64, 3, 2, 1, 38, 76)])
def test_conv2d_hires_persistent_kernels(case, monkeypatch):
    """Persistent forms of the stem / level0 / level1 / level2.tree1.conv1 kernels (one CTA per SM walks output tiles, weights as
    register-resident B fragments, double-buffered halo; stride 1: four output rows per warp): taken when there is a tile per SM,
    forced here for the ragged small shapes.  Bit-identical to the per-tile kernels (SMOT_HIRES_PERSIST=0); torch fp32 within the
    fp16 bar."""
    name, Cin, Cout, k, stride, batch, H, W = case
    g = torch.Generator().manual_seed(len(name) + H)
    dt = torch.float16
    x = q(torch.randn(batch, Cin, H, W, generator=g), dt)
    w = q(torch.randn(Cout, Cin, k, k, generator=g) / math.sqrt(Cin * k * k), dt)
    scale, bias = 0.5 + torch.rand(Cout, generator=g), torch.randn(Cout, generator=g)
    if Cin == 3:
        buf = torch.zeros(batch, H, W, 4, dtype=dt, device=DEV)
        buf[..., :3] = nhwc(x, dt)
        dx = buf[..., :3]
    else:
        dx = nhwc(x, dt)
    args = (dx, ohwi(w, dt), scale.to(DEV), bias.to(DEV), None, stride, k // 2, True)
    monkeypatch.setenv("SMOT_HIRES_PERSIST", "0")
    per_tile = conv2d_checked(*args)
    monkeypatch.setenv("SMOT_HIRES_PERSIST", "2")
    for _ in range(2):                               # back-to-back launches chain through PDL
        got = ops().conv2d(*args)
    torch.cuda.synchronize()
    assert torch.equal(got, per_tile)
    monkeypatch.delenv("SMOT_HIRES_PERSIST")
    assert torch.equal(conv2d_checked(*args), per_tile)   # the default rule, whichever kernel it picks


@pytest.mark.parametrize("mode", ["16", "10"])
def test_conv2d_tcgen05_halo_variant(mode, monkeypatch):
    """Developer variant of the 3x3 wgmma kernel (SMOT_TC_HALO): the input halo of an 8x16 tile stays in shared
    memory and the nine taps are shifted wgmma descriptors over it (patch rows of 16 or 10 pixels).  Same results."""
    from siammot_b200 import _lib
    monkeypatch.setenv("SMOT_TC_HALO", mode)
    g = torch.Generator().manual_seed(int(mode))
    dt = torch.float16
    ws = ops().conv_workspace(DEV)
    for (B, Cin, H, W, Cout, use_ws) in ((1, 128, 88, 160, 128, False), (1, 64, 37, 53, 64, False), (3, 128, 16, 16, 256, False),
                                         (1, 512, 22, 40, 512, True)):
        x = q(torch.randn(B, Cin, H, W, generator=g), dt)
        w = q(torch.randn(Cout, Cin, 3, 3, generator=g) / math.sqrt(Cin * 9), dt)
        res = q(torch.randn(B, Cout, H, W, generator=g), dt)
        scale, bias = 0.5 + torch.rand(Cout, generator=g), torch.randn(Cout, generator=g)
        conv2d_checked(nhwc(x, dt), ohwi(w, dt), scale.to(DEV), bias.to(DEV), nhwc(res, dt), 1, 1, True,
                       algo=_lib.CONV_TCGEN05, workspace=ws if use_ws else None)


def test_conv2d_tcgen05_split_k():
    """Few-tile / long-K layers (level5 convs, fc6) with the split-K workspace: fp32 partial tiles are reduced in
    split order by the last CTA of each output tile; counters must be left zero (call twice, then inspect)."""
    from siammot_b200 import _lib
    g = torch.Generator().manual_seed(123)
    dt = torch.float16
    ws = ops().conv_workspace(DEV)
    # level5 3x3: 9 tiles x 8 n-tiles x K = 4608
    x = q(torch.randn(1, 512, 22, 40, generator=g), dt)
    w = q(torch.randn(512, 512, 3, 3, generator=g) / math.sqrt(512 * 9), dt)
    res = q(torch.randn(1, 512, 22, 40, generator=g), dt)
    scale, bias = 0.5 + torch.rand(512, generator=g), torch.randn(512, generator=g)
    args = (nhwc(x, dt), ohwi(w, dt), scale.to(DEV), bias.to(DEV), nhwc(res, dt), 1, 1, True)
    for _ in range(2):
        conv2d_checked(*args, algo=_lib.CONV_TCGEN05, workspace=ws)
        torch.cuda.synchronize()
    conv2d_checked(*args, algo=_lib.CONV_TCGEN05)
    # fc6 for 300 and 30 rows
    for rows in (300, 30):
        xfc = q(torch.randn(rows, 6272, generator=g), dt)
        wfc = q(torch.randn(1024, 6272, generator=g) / math.sqrt(6272), dt)
        bfc = torch.randn(1024, generator=g)
        conv2d_checked(xfc.to(DEV, dt).view(1, 1, rows, 6272), wfc.to(DEV, dt).view(1024, 1, 1, 6272), None,
                       bfc.to(DEV), relu=True, algo=_lib.CONV_TCGEN05, workspace=ws)
    torch.cuda.synchronize()
    assert int(ws[:_lib.CONV_WS_COUNTER_BYTES].view(torch.int32).abs().sum()) == 0


@pytest.mark.parametrize("case", [(1, 512, 22, 40, 512, 3), (1, 256, 44, 80, 256, 3), (2, 256, 44, 80, 256, 3), (1, 1280, 22, 40, 512, 1),
                                  (1, 6272, 1, 300, 1024, 1), (1, 256, 22, 40, 512, 3), (1, 128, 16, 16, 256, 3)])
def test_conv2d_tcgen05_k_slices_equal_split_k(case, monkeypatch):
    """Few-tile layers: one CTA that adds each K range's register accumulator to a running sum (SMOT_TC_SLICED=1) against the split CTAs + reduce kernel
    (the default): the same K ranges summed in the same order -- the same bits -- for levels 4 / 5, a root 1x1, fc6 and a batch
    of two (frame-pair plans)."""
    from siammot_b200 import _lib
    B, Cin, H, W, Cout, k = case
    g = torch.Generator().manual_seed(Cin + W)
    dt = torch.float16
    ws = ops().conv_workspace(DEV)
    x = q(torch.randn(B, Cin, H, W, generator=g), dt)
    w = q(torch.randn(Cout, Cin, k, k, generator=g) / math.sqrt(Cin * k * k), dt)
    res = q(torch.randn(B, Cout, H, W, generator=g), dt)
    scale, bias = 0.5 + torch.rand(Cout, generator=g), torch.randn(Cout, generator=g)
    args = (nhwc(x, dt), ohwi(w, dt), scale.to(DEV), bias.to(DEV), nhwc(res, dt), 1, k // 2, True)
    monkeypatch.setenv("SMOT_TC_SLICED", "0")
    split = conv2d_checked(*args, algo=_lib.CONV_TCGEN05, workspace=ws)
    torch.cuda.synchronize()
    monkeypatch.setenv("SMOT_TC_SLICED", "1")
    for _ in range(2):
        sliced = conv2d_checked(*args, algo=_lib.CONV_TCGEN05, workspace=ws)
    torch.cuda.synchronize()
    assert torch.equal(sliced, split)
