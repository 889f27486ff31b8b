"""A CPU stand-in for libsmot.so's entry points -- TEST INFRASTRUCTURE, never imported by the product.

Purpose: run the engine's whole HOST side (static launch plan, per-N track plans, buffer arenas, result-block packing, host
solver, next-frame memory, clip pipelining) in a container without a GPU.  Every C-ABI entry point of include/smot.h that the
per-frame path calls is emulated here with the oracle's primitives on the very pointers the engine passes (host memory, fp32);
the CUDA runtime objects the engine uses for ordering (streams, events) become no-ops.  An end-to-end run through this
emulation reproduces the reference goldens iff the host logic wires the calls correctly (tests/test_engine_emulated_cpu.py).
What it does NOT test is the CUDA kernels: those are compared with the same oracle primitives, per op and end to end, by the
`-m gpu` tests on an H100.
"""
import contextlib
import ctypes as C

import torch
import torch.nn.functional as F

from oracle import prims
from oracle import siammot_oracle as orc
from plan_emulator import _view


def _a(p):
    """Address carried by a C-ABI pointer argument (c_void_p / int / None)."""
    if p is None:
        return 0
    if isinstance(p, C.c_void_p):
        return p.value or 0
    return int(p)


def _f32(p, n):
    return torch.frombuffer((C.c_float * max(n, 1)).from_address(_a(p)), dtype=torch.float32)[:n]


def _i32(p, n):
    return torch.frombuffer((C.c_int32 * max(n, 1)).from_address(_a(p)), dtype=torch.int32)[:n]


def _rows(p, n, width, stride):
    """(n, width) fp32 view with `stride` floats between rows."""
    if n == 0:
        return torch.zeros((0, width))
    return _f32(p, (n - 1) * stride + width).as_strided((n, width), (stride, 1))


def deform_columns(inp, off, cols, H, W, Cc, ild, oild, OH, OW, old, stride):
    """Specification of smot_deform_im2col3x3 (DCN v1 sampling) on host pointers, vectorised."""
    x = _view(inp, 1, H, W, Cc, ild)[0]                       # (H, W, C)
    o = _view(off, 1, OH, OW, 18, oild)[0]                    # (OH, OW, 18)
    out = _view(cols, 1, OH, OW, 9 * Cc, old)[0]
    oy = torch.arange(OH, dtype=torch.float32).view(OH, 1) * stride - 1
    ox = torch.arange(OW, dtype=torch.float32).view(1, OW) * stride - 1
    for k in range(9):
        i, j = divmod(k, 3)
        yy, xx = oy + i + o[..., 2 * k], ox + j + o[..., 2 * k + 1]
        inside = (yy > -1) & (yy < H) & (xx > -1) & (xx < W)
        y0, x0 = torch.floor(yy), torch.floor(xx)
        ly, lx = yy - y0, xx - x0
        acc = torch.zeros((OH, OW, Cc))
        for dy_, dx_, wgt in ((0, 0, (1 - ly) * (1 - lx)), (0, 1, (1 - ly) * lx), (1, 0, ly * (1 - lx)), (1, 1, ly * lx)):
            yi, xi = (y0 + dy_).long(), (x0 + dx_).long()
            ok = inside & (yi >= 0) & (yi < H) & (xi >= 0) & (xi < W)
            acc = acc + x[yi.clamp(0, H - 1), xi.clamp(0, W - 1)] * (wgt * ok)[..., None]
        out[..., k * Cc:(k + 1) * Cc] = acc


class FakeLib(object):
    """Entry points of include/smot.h, fp32 only, on host pointers.  Every method returns SMOT_OK (0)."""

    def __init__(self):
        self.calls = {}

    def _count(self, name):
        self.calls[name] = self.calls.get(name, 0) + 1

    # ---- misc
    def smot_abi_version(self):
        from siammot_b200 import _lib
        return _lib.ABI_VERSION

    def smot_last_error(self):
        return b""

    def smot_rpn_select_workspace(self, num_levels, pre_nms_top_n):
        return 64

    def smot_sort_nms_workspace(self, n_max):
        return 64

    def smot_conv2d_algo(self, d):
        return 1

    # ---- dense / small tensor kernels
    def smot_image_to_nhwc(self, chw, out, Cc, H, W, ld, dt, st):
        self._count("smot_image_to_nhwc")
        assert dt == 0
        _view(_a(out), 1, H, W, Cc, ld).copy_(_f32(chw, Cc * H * W).view(Cc, H, W).permute(1, 2, 0)[None])
        return 0

    def smot_conv2d(self, dref, st):
        self._count("smot_conv2d")
        d = dref._obj
        assert d.in_dtype == 0 and d.out_dtype == 0, "the emulation runs the fp32 mode"
        x = _view(d.inp, d.batch, d.H, d.W, d.Cin, d.in_ld).permute(0, 3, 1, 2)
        w = _f32(d.weight, d.Cout * d.KH * d.KW * d.Cin).view(d.Cout, d.KH, d.KW, d.Cin)
        y = F.conv2d(x, w.permute(0, 3, 1, 2), None, d.stride, d.pad)
        assert tuple(y.shape) == (d.batch, d.Cout, d.OH, d.OW)
        if d.scale:
            y = y * _f32(d.scale, d.Cout).view(1, -1, 1, 1)
        if d.bias:
            y = y + _f32(d.bias, d.Cout).view(1, -1, 1, 1)
        if d.residual:
            y = y + _view(d.residual, d.batch, d.OH, d.OW, d.Cout, d.res_ld).permute(0, 3, 1, 2)
        if d.relu:
            y = F.relu(y)
        _view(d.out, d.batch, d.OH, d.OW, d.Cout, d.out_ld).copy_(y.permute(0, 2, 3, 1))
        return 0

    def _pool(self, name, inp, out, B, H, W, Cc, ild, old, dt, st):
        self._count(name)
        x = _view(_a(inp), B, H, W, Cc, ild).permute(0, 3, 1, 2)
        y = F.max_pool2d(x, 2, 2) if name == "smot_maxpool2x2" else F.max_pool2d(x, 3, 2, 1)
        _view(_a(out), B, y.shape[2], y.shape[3], Cc, old).copy_(y.permute(0, 2, 3, 1))
        return 0

    def smot_maxpool2x2(self, *a):
        return self._pool("smot_maxpool2x2", *a)

    def smot_maxpool3x3s2(self, *a):
        return self._pool("smot_maxpool3x3s2", *a)

    def smot_deform_im2col3x3(self, inp, off, cols, H, W, Cc, ild, oild, OH, OW, old, stride, dt, st):
        self._count("smot_deform_im2col3x3")
        deform_columns(_a(inp), _a(off), _a(cols), H, W, Cc, ild, oild, OH, OW, old, stride)
        return 0

    def smot_subsample2(self, inp, out, H, W, Cc, ild, old, dt, st):
        self._count("smot_subsample2")
        y = _view(_a(inp), 1, H, W, Cc, ild)[:, ::2, ::2]
        _view(_a(out), 1, y.shape[1], y.shape[2], Cc, old).copy_(y)
        return 0

    def smot_upsample_add(self, top, Ht, Wt, tld, lat, H, W, lld, Cc, dt, st):
        self._count("smot_upsample_add")
        t = _view(_a(top), 1, Ht, Wt, Cc, tld).permute(0, 3, 1, 2)
        up = F.interpolate(t, size=(H, W), mode="bilinear", align_corners=False)
        lv = _view(_a(lat), 1, H, W, Cc, lld)
        lv.copy_(lv + up.permute(0, 2, 3, 1))
        return 0

    def smot_groupnorm_relu(self, x, gamma, beta, batch, HW, Cc, ld, groups, eps, relu, dt, st):
        self._count("smot_groupnorm_relu")
        v = _view(_a(x), batch, 1, HW, Cc, ld)
        y = F.group_norm(v[:, 0].permute(0, 2, 1), groups, _f32(gamma, Cc), _f32(beta, Cc), eps)
        v[:, 0].copy_((F.relu(y) if relu else y).permute(0, 2, 1))
        return 0

    # ---- ROIAlign
    def _roi_align(self, pref, rois, level_boxes, count, max_rois, Cc, res, sampling):
        p = pref._obj
        n = max_rois if not _a(count) else min(int(_i32(count, 1)[0]), max_rois)
        out = torch.zeros((max_rois, Cc, res, res))
        if n:
            feats = []
            for l in range(p.num_levels):
                f = _view(p.feat[l], 1, p.H[l], p.W[l], Cc, p.ld[l]).permute(0, 3, 1, 2)
                feats.append(F.pad(f, [p.pad[l]] * 4) if p.pad[l] else f)
            r = _rows(rois, max_rois, 4, 4)[:n].clone()
            lb = _rows(level_boxes, max_rois, 4, 4)[:n].clone() if _a(level_boxes) else r
            scales = [float(p.scale[l]) for l in range(p.num_levels)]
            assert p.k_min == 2
            out[:n] = orc.pool_rois(feats, lb, lb, scales, res, sampling, rois=r)
        return out

    def smot_roi_align(self, pref, rois, level_boxes, count, max_rois, Cc, res, sampling, out, dt, st):
        self._count("smot_roi_align")
        if max_rois:
            y = self._roi_align(pref, rois, level_boxes, count, max_rois, Cc, res, sampling)
            _view(_a(out), max_rois, res, res, Cc, Cc).copy_(y.permute(0, 2, 3, 1))
        return 0

    def smot_roi_align_planar(self, pref, rois, level_boxes, count, max_rois, Cc, res, sampling, out, row_pitch, plane_pitch,
                              dt, st):
        self._count("smot_roi_align_planar")
        if max_rois:
            y = self._roi_align(pref, rois, level_boxes, count, max_rois, Cc, res, sampling)
            planes = _f32(out, max_rois * Cc * plane_pitch).view(max_rois, Cc, plane_pitch)
            planes[:, :, :res * row_pitch].view(max_rois, Cc, res, row_pitch)[..., :res] = y
        return 0

    # ---- RPN selection
    def smot_rpn_select(self, levels, num_levels, pre_n, post_n, nms_thresh, min_size, fpn_post_n, img_w, img_h, amodal,
                        out_boxes, out_scores, out_count, ws, ws_bytes, st):
        self._count("smot_rpn_select")
        boxes_all, scores_all = [], []
        for l in range(num_levels):
            L = levels[l]
            head = _rows(L.head, L.H * L.W, 5 * L.A, L.head_ld)
            logit = head[:, :L.A].reshape(-1)
            reg = head[:, L.A:5 * L.A].reshape(-1, 4)
            k = min(pre_n, logit.numel())
            idx = torch.sort(logit, descending=True, stable=True)[1][:k]
            obj = logit[idx].sigmoid()
            cell = torch.tensor([L.cell_anchors[i] for i in range(4 * L.A)], dtype=torch.float32).view(L.A, 4)
            anchors = prims.grid_anchors(cell, L.stride, L.H, L.W)[idx]
            prop = prims.box_decode(reg[idx], anchors, (1.0, 1.0, 1.0, 1.0))
            if not amodal:
                prop = prims.clip_boxes(prop, img_w, img_h)
            keep = prims.remove_small_mask(prop, min_size).nonzero().squeeze(1)
            prop, obj = prop[keep], obj[keep]
            keep = prims.nms_legacy(prop, obj, nms_thresh)[:post_n]
            boxes_all.append(prop[keep])
            scores_all.append(obj[keep])
        boxes, scores = torch.cat(boxes_all), torch.cat(scores_all)
        k = min(fpn_post_n, scores.numel())
        inds = torch.sort(scores, descending=True, stable=True)[1][:k]
        _rows(out_boxes, fpn_post_n, 4, 4)[:k] = boxes[inds]
        _f32(out_scores, fpn_post_n)[:k] = scores[inds]
        _i32(out_count, 1)[0] = k
        return 0

    # ---- sort + NMS
    def smot_sort_nms(self, boxes, box_stride, scores, score_stride, count, n_max, min_score, thresh, max_keep, tag, out_index,
                      out_boxes, out_scores, out_tag, out_count, ws, ws_bytes, st):
        self._count("smot_sort_nms")
        if n_max == 0:
            return 0
        n = n_max if not _a(count) else min(int(_i32(count, 1)[0]), n_max)
        b = _rows(boxes, n, 4, box_stride).clone()
        s = _rows(scores, n, 1, score_stride)[:, 0].clone() if n else torch.zeros((0,))
        cand = (s > min_score).nonzero().squeeze(1)
        if thresh > 0:
            keep = prims.nms_legacy(b[cand], s[cand], thresh)
        else:
            keep = torch.sort(s[cand], descending=True, stable=True)[1]
        keep = cand[keep][:max_keep]
        base = int(_i32(out_count, 1)[0])
        m = keep.numel()
        if m:
            if _a(out_index):
                _i32(out_index, base + m)[base:] = keep.to(torch.int32)
            if _a(out_boxes):
                _rows(out_boxes, base + m, 4, 4)[base:] = b[keep]
            if _a(out_scores):
                _f32(out_scores, base + m)[base:] = s[keep]
            if _a(out_tag):
                _i32(out_tag, base + m)[base:] = tag
        _i32(out_count, 1)[0] = base + m
        return 0

    # ---- box head post-processing
    def smot_box_decode(self, head, head_ld, rois, count, n_max, ncls, w4ref, img_w, img_h, amodal, track_labels, out_boxes,
                        out_scores, st):
        self._count("smot_box_decode")
        n = n_max if not _a(count) else min(int(_i32(count, 1)[0]), n_max)
        ob = _rows(out_boxes, n_max, 4 * ncls, 4 * ncls)
        os_ = _rows(out_scores, n_max, ncls, ncls)
        ob[n:] = 0.0
        os_[n:] = -1.0
        if n:
            h = _rows(head, n, 5 * ncls, head_ld)
            prob = F.softmax(h[:, :ncls], -1)
            r = _rows(rois, n, 4, 4)
            w = [float(v) for v in w4ref._obj]
            dec = prims.box_decode(h[:, ncls:5 * ncls], r, w).reshape(-1, 4)
            if not amodal:
                dec = prims.clip_boxes(dec, img_w, img_h)
            if _a(track_labels):
                lab = _i32(track_labels, n).to(torch.int64)
                cp = prob.clone()
                prob = torch.zeros_like(prob)
                ar = torch.arange(n)
                prob[ar, lab] = cp[ar, lab] + 1.0
            ob[:n] = dec.reshape(n, 4 * ncls)
            os_[:n] = prob
        return 0

    def smot_track_combine(self, det_boxes, det_scores, ncap, dec_boxes, dec_scores, ncls, labels, conf, valid, active, n,
                           tracktor, cat_boxes, cat_scores, zero_count, st):
        self._count("smot_track_combine")
        if _a(zero_count):
            _i32(zero_count, 1)[0] = 0
        cb, cs = _rows(cat_boxes, ncap + n, 4, 4), _f32(cat_scores, ncap + n)
        if ncap:
            cb[:ncap] = _rows(det_boxes, ncap, 4, 4)
            cs[:ncap] = _f32(det_scores, ncap)
        if n:
            lab = _i32(labels, n).to(torch.int64)
            ar = torch.arange(n)
            det_part = _rows(dec_scores, n, ncls, ncls)[ar, lab]
            s = det_part if tracktor else (det_part + (_f32(conf, n) + 1.0)) / 2.0
            s = s + _f32(active, n)
            cb[ncap:] = _rows(dec_boxes, n, 4 * ncls, 4 * ncls).view(n, ncls, 4)[ar, lab]
            cs[ncap:] = torch.where(_i32(valid, n) != 0, s, torch.full_like(s, -1.0))
        return 0

    def smot_track_combine_grouped(self, det_boxes, det_scores, ncap, dec_boxes, dec_scores, ncls, labels, conf, valid, active,
                                   n, tracktor, cat_boxes, cat_scores, zero_count, perm, st):
        """The reference's order for several foreground classes (roi_heads.py:60-84 over inference.py:145-191), restated."""
        self._count("smot_track_combine_grouped")
        if _a(zero_count):
            _i32(zero_count, 1)[0] = 0
        cb, cs = _rows(cat_boxes, ncap + n, 4, 4), _f32(cat_scores, ncap + n)
        if ncap:
            cb[:ncap] = _rows(det_boxes, ncap, 4, 4)
            cs[:ncap] = _f32(det_scores, ncap)
        if n:
            lab = _i32(labels, n).to(torch.int64)
            V = (_i32(valid, n) != 0).nonzero().squeeze(1)                         # tracks the EMM kept, memory order
            G = V[torch.sort(lab[V], stable=True)[1]]                              # ... as the box head returns them
            m = V.numel()
            trk_scores = _f32(conf, n)[V] + 1.0                                    # roi_heads.py:67 (before the box head)
            det_part = _rows(dec_scores, n, ncls, ncls)[G, lab[G]]
            s = det_part if tracktor else (det_part + trk_scores) / 2.0            # roi_heads.py:76: position by position
            s = s + _f32(active, n)[G]
            cb[ncap:] = 0.0
            cs[ncap:] = -1.0
            cb[ncap:ncap + m] = _rows(dec_boxes, n, 4 * ncls, 4 * ncls).view(n, ncls, 4)[G, lab[G]]
            cs[ncap:ncap + m] = s
            pm = _i32(perm, n)
            pm[:] = -1
            pm[:m] = G.to(torch.int32)
        return 0

    # ---- EMM
    def smot_xcorr(self, x, k, out, n, Cc, S, T, dt, st):
        self._count("smot_xcorr")
        if n:
            O = S - T + 1
            y = orc.xcorr_depthwise(_view(_a(x), n, S, S, Cc, Cc).permute(0, 3, 1, 2), _view(_a(k), n, T, T, Cc, Cc).permute(0, 3, 1, 2))
            _view(_a(out), n, O, O, Cc, Cc).copy_(y.permute(0, 2, 3, 1))
        return 0

    def smot_xcorr_planar(self, xp, k, out, n, Cc, st):
        self._count("smot_xcorr_planar")
        from siammot_b200 import _lib
        if n:
            S, T, O, RP, PL = 30, 15, 16, _lib.XCORR_ROW_PITCH, _lib.XCORR_PLANE
            planes = _f32(xp, n * Cc * PL).view(n, Cc, PL)
            rows = planes[:, :, :S * RP].view(n, Cc, S, RP)
            assert float(rows[..., S:S + 2].abs().max()) == 0.0, "columns 30/31 of the planar windows must be zero"
            y = orc.xcorr_depthwise(rows[..., :S], _view(_a(k), n, T, T, Cc, Cc).permute(0, 3, 1, 2))
            _view(_a(out), n, O, O, Cc, Cc).copy_(y.permute(0, 2, 3, 1))
        return 0

    def smot_xcorr_planar_mode(self, xp, k, out, n, Cc, mma_mode, st):
        return self.smot_xcorr_planar(xp, k, out, n, Cc, st)

    def smot_xcorr_planar_cfg(self, xp, k, out, n, Cc, mma_mode, cg, st):
        assert cg in (0, 2, 4, 8, 16) and Cc % (cg or 4) == 0
        return self.smot_xcorr_planar(xp, k, out, n, Cc, st)

    def smot_emm_decode(self, maps, map_ld, n, O, up, T, sr, tboxes, hann, pad, use_centerness, sigma, img_w, img_h, amodal,
                        out_boxes, out_conf, out_valid, scratch, st):
        self._count("smot_emm_decode")
        if n == 0:
            return 0
        m = _view(_a(maps), n, O, O, 7, map_ld).permute(0, 3, 1, 2)
        assert torch.equal(_f32(hann, O * up), torch.hann_window(O * up, dtype=torch.float))
        s, tb = _rows(sr, n, 4, 4).clone(), _rows(tboxes, n, 4, 4).clone()
        bb, conf = orc.emm_decode(m[:, 0:2], m[:, 2:3], m[:, 3:7], s, tb, pad, T, bool(use_centerness), float(sigma), up)
        valid = torch.ones(n, dtype=torch.int32)
        if not amodal:
            bb = prims.clip_boxes(bb, img_w, img_h)
            valid = prims.nonempty_mask(bb).to(torch.int32)
        _rows(out_boxes, n, 4, 4).copy_(bb)
        _f32(out_conf, n).copy_(conf)
        _i32(out_valid, n).copy_(valid)
        return 0


class _Event(object):
    def __init__(self, *a, **k):
        pass

    def record(self, *a):
        pass

    def synchronize(self):
        pass

    def wait(self, *a):
        pass

    def elapsed_time(self, other):
        return 1.0   # ms: any positive number -- timings taken under the emulation are meaningless


class _Stream(object):
    cuda_stream = 0

    def __init__(self, *a, **k):
        pass

    def wait_stream(self, *a):
        pass

    def wait_event(self, *a):
        pass


class _Graph(object):
    """torch.cuda.CUDAGraph stand-in: "capture" runs the launches once, replay does nothing (timings are meaningless here)."""

    def replay(self):
        pass


def install(monkeypatch):
    """Route the product's libsmot calls to FakeLib and neutralise the CUDA runtime objects.  Returns the FakeLib."""
    from siammot_b200 import _lib, engine, ops, preprocess
    from siammot_b200.modelling import rcnn
    fake = FakeLib()
    for mod in (_lib, engine, ops, preprocess):
        monkeypatch.setattr(mod, "lib", lambda: fake)
    for mod in (_lib, ops):
        monkeypatch.setattr(mod, "stream_ptr", lambda: C.c_void_p(0))
    monkeypatch.setattr(ops, "_require_cuda", lambda *a: None)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: _Stream())
    monkeypatch.setattr(torch.cuda, "Event", _Event)
    monkeypatch.setattr(torch.cuda, "Stream", _Stream)
    monkeypatch.setattr(torch.cuda, "stream", lambda s: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    monkeypatch.setattr(torch.cuda, "CUDAGraph", _Graph)
    monkeypatch.setattr(torch.cuda, "graph", lambda g, *a, **k: contextlib.nullcontext())
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self, *a, **k: self)

    def host_engine(self):
        if self._engine is None:
            self._engine = engine.Engine(self.cfg, device="cpu", use_graph=False)
            self._engine_stale = True
        if self._engine_stale:
            self._engine.load_state_dict(self.state_dict())
            self._engine_stale = False
        self.roi_heads.engine = self._engine
        if self.cfg.MODEL.TRACK_ON:
            self.roi_heads.track.tracker.engine = self._engine
        return self._engine

    monkeypatch.setattr(rcnn.SiamMOT, "engine", host_engine)
    return fake


def install_for_bench(monkeypatch):
    """install() + what bench.py touches beyond the model: device placement and the device-side test transform (emulated by
    the oracle's restatement of the reference transform)."""
    from oracle import preprocess as opp
    from siammot_b200 import preprocess
    fake = install(monkeypatch)
    orig_init = preprocess.FramePreprocessor.__init__

    def init(self, cfg, device="cuda"):
        orig_init(self, cfg, device)
        self._cfg = cfg

    def into(self, frame, out, lane=0):
        out.copy_(opp.preprocess(frame.numpy() if torch.is_tensor(frame) else frame, self._cfg))
        return out

    monkeypatch.setattr(preprocess.FramePreprocessor, "__init__", init)
    monkeypatch.setattr(preprocess.FramePreprocessor, "into", into)
    monkeypatch.setattr(torch.cuda, "set_device", lambda *a: None)
    monkeypatch.setattr(torch.nn.Module, "to", lambda self, *a, **k: self)
    return fake
