"""Per-frame execution engine: weight preparation, static launch plan, dynamic tracker stage.

This is the H100 (sm_90a) replacement for everything beneath ``SiamMOT.forward``
(/root/reference/siammot/modelling/rcnn.py:41-68).  Design:

* activations live in NHWC device buffers allocated once per input resolution; DLA roots read their
  children through channel-slice views (no torch.cat, dla.py:183), FrozenBN / bias / residual / ReLU
  ride in the conv epilogues;
* the frame-independent stage (backbone -> FPN -> RPN head -> proposal selection -> box head ->
  per-class NMS) is a fixed list of C-ABI launches with device-side counts, captured once into a
  CUDA graph (independent layers as parallel branches) and replayed per frame;
* the track-dependent stage (search-region ROIAlign with virtual padding -> xcorr -> EMM towers ->
  fused decode -> box-head refinement -> solver NMS) is a launch list per N = tracks in memory, replayed as a
  CUDA graph from its second use;
* decoded uint8 frames are resized / normalised on the device (preprocess.py), bit-identically to the CPU transform;
* exactly one device->host copy per frame (the solver needs ids on the host, track_solver.py:62-106),
  against >= 10 hidden syncs in the reference (SURVEY.md section 3.3).

All compute is libsmot.so (hand-written sm_90a CUDA for the H100); torch is used for memory, streams, graphs and
a few single-element glue ops on tiny tensors.  No CPU fallback exists.
"""
import ctypes as C
import math
import os

import torch

from . import _lib, ops
from ._lib import check, lib


def _ohwi(w, dtype, device):
    return w.detach().to(torch.float32).permute(0, 2, 3, 1).contiguous().to(device=device, dtype=dtype)


def _f32(t, device):
    return t.detach().to(device=device, dtype=torch.float32).contiguous()


def cell_anchors(stride, sizes, aspect_ratios):
    """Detectron-style cell anchors (upstream rpn/anchor_generator.py generate_anchors): float64
    maths, legacy rounding, cast to fp32.  Returned as an (A,4) CPU tensor; also the value of the
    reference's ``rpn.anchor_generator.cell_anchors.*`` buffers."""
    import numpy as np
    scales = np.array(sizes, dtype=np.float64) / stride
    ratios = np.array(aspect_ratios, dtype=np.float64)

    def whctr(a):
        w, h = a[2] - a[0] + 1, a[3] - a[1] + 1
        return w, h, a[0] + 0.5 * (w - 1), a[1] + 0.5 * (h - 1)

    def mk(ws, hs, xc, yc):
        ws, hs = ws[:, None], hs[:, None]
        return np.hstack((xc - 0.5 * (ws - 1), yc - 0.5 * (hs - 1), xc + 0.5 * (ws - 1), yc + 0.5 * (hs - 1)))

    w, h, xc, yc = whctr(np.array([0, 0, stride - 1, stride - 1], dtype=np.float64))
    ws = np.round(np.sqrt(w * h / ratios))
    hs = np.round(ws * ratios)
    rows = []
    for ra in mk(ws, hs, xc, yc):
        w, h, xc, yc = whctr(ra)
        rows.append(mk(w * scales, h * scales, xc, yc))
    return torch.from_numpy(np.vstack(rows)).float()


class _NoTimer(object):
    def __enter__(self):
        return None

    def __exit__(self, *exc):
        return False


_NO_TIMER = _NoTimer()


class _Timed(object):
    """Engine.timed(): CUDA-event bracket (+ optional NVTX range) around the enclosed launches."""

    def __init__(self, eng, name):
        self.eng, self.name = eng, name

    def __enter__(self):
        eng = self.eng
        if eng.nvtx:
            torch.cuda.nvtx.range_push("smot/" + self.name)
        if eng.timers is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e1 = torch.cuda.Event(enable_timing=True)
            self.e0.record()

    def __exit__(self, *exc):
        eng = self.eng
        if eng.timers is not None:
            self.e1.record()
            eng.timers.setdefault(self.name, []).append((self.e0, self.e1))
        if eng.nvtx:
            torch.cuda.nvtx.range_pop()
        return False


class _Plan(object):
    """Launch list for one input resolution.  Each step is (callable, args-before-stream)."""

    def __init__(self, engine, H, W):
        self.e = engine
        self.H, self.W = H, W
        self.steps = []
        self.keep = []  # ctypes objects / tensors that must outlive the plan
        self.graph = None
        self.dev = engine.device
        self.dtype = engine.dtype
        self.ws = engine.conv_ws      # split-K scratch of the stream this plan runs on
        self.static_done = None       # event recorded after the plan when it runs on the side stream (forward_clip)
        self.backbone_done = None     # three-stage clip mode: event after part 0
        self.part_graphs = [None, None]
        self.branch = None            # while building: steps appended go to this parallel branch (None = main line)
        self.batch = 1                # images per backbone pass (2 = a frame PAIR of a clip, see Engine.pair_plan)
        self.batched = False          # Engine.batch_plan: the detection tail runs over all `batch` images too
        self.branch_wss = None        # split-K scratch per parallel branch when the plan owns them (batch plans)
        self.bufs = []                # activation buffers in allocation order
        self.view_of, self.view_index, self._cursor = None, 0, 0

    def new(self, H, W, Cc, dtype=None):
        """An activation buffer (batch, H, W, Cc).  A frame plan that belongs to a pair plan (view_of) does not allocate: it
        takes image ``view_index`` of the pair plan's buffer with the same allocation number -- both plans are built by the
        same code, so the k-th allocation of one is the k-th of the other."""
        dtype = dtype or self.dtype
        if self.view_of is not None:
            src = self.view_of.bufs[self._cursor]
            self._cursor += 1
            t = src[self.view_index:self.view_index + 1]
            if tuple(t.shape) != (1, H, W, Cc) or t.dtype != dtype:
                raise RuntimeError("pair plan / frame plan allocation order diverged: %s %s vs (1, %d, %d, %d) %s"
                                   % (tuple(t.shape), t.dtype, H, W, Cc, dtype))
        else:
            t = torch.zeros((self.batch, H, W, Cc), dtype=dtype, device=self.dev)
        self.bufs.append(t)
        self.keep.append(t)
        return t

    def per_image(self, fn, make_args, tag):
        """Kernels without a batch argument run once per image of the batch (make_args(i) builds the call for image i)."""
        for i in range(self.batch):
            self.call(fn, make_args(i), tag)

    def conv(self, x, name, out, residual=None, stride=1, pad=0, relu=False):
        w, scale, bias = self.e.weights[name]
        if self.branch is None:
            ws = self.ws
        elif self.branch_wss is not None:
            ws = self.branch_wss[self.branch]
        else:
            ws = self.e.branch_ws(self.branch)
        d = ops.conv_desc(x, w, out, scale, bias, residual, stride, pad, relu, workspace=ws)
        self.keep.append(d)
        self.steps.append((lib().smot_conv2d, (C.byref(d),), "conv:" + name, self.branch))
        return out

    def call(self, fn, args, tag):
        self.steps.append((fn, args, tag, self.branch))

    # Independent layers (the FPN laterals, the per-level FPN-output -> RPN chains) are enqueued on parallel branches:
    # fork(n) .. join() become parallel paths of the CUDA graph (streams in eager mode), so the small-level kernels
    # (<= 30 CTAs, mostly fixed launch / prologue / epilogue cost) run under the big P2 ones instead of after them.
    def fork(self, n):
        self.steps.append(("fork", n, None, None))

    def join(self):
        self.branch = None
        self.steps.append(("join", None, None, None))

    def split_index(self):
        """First step of the detection tail (RPN selection .. per-class NMS): everything before it is the backbone / FPN /
        RPN-head part, whose kernels fill the GPU; the tail is a serial chain of small kernels."""
        for i, (_fn, _args, tag, _branch) in enumerate(self.steps):
            if tag == "rpn_select":
                return i
        return len(self.steps)        # a backbone-only (pair) plan: everything is part 0

    def run_eager(self, lo=0, hi=None):
        main = torch.cuda.current_stream(self.dev)
        st = C.c_void_p(main.cuda_stream)
        active = []
        for fn, args, tag, branch in self.steps[lo:hi]:
            if fn == "fork":
                active = self.e.branch_streams(args)
                for b in active:
                    b.wait_stream(main)
            elif fn == "join":
                for b in active:
                    main.wait_stream(b)
                active = []
            elif branch is None:
                check(fn(*args, st), tag)
            else:
                check(fn(*args, C.c_void_p(active[branch].cuda_stream)), tag)

    def run(self):
        if self.e.use_graph:
            if self.graph is None:
                self.run_eager()  # warm-up: sets function attributes, surfaces argument errors
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self.run_eager()
                self.graph = g
            self.graph.replay()
        else:
            self.run_eager()

    def run_part(self, part):
        """Run one half of the plan on the current stream (part 0: image .. RPN heads, part 1: proposal selection ..
        detections), each half its own CUDA graph -- SiamMOT.forward_clip's three-stage mode runs the halves of
        consecutive frames on different streams."""
        k = self.split_index()
        lo, hi = (0, k) if part == 0 else (k, len(self.steps))
        if not self.e.use_graph:
            return self.run_eager(lo, hi)
        if self.part_graphs[part] is None:
            self.run_eager(lo, hi)  # warm-up on live data (the other half has run): sets function attributes
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self.run_eager(lo, hi)
            self.part_graphs[part] = g
        self.part_graphs[part].replay()


class _TrackArena(object):
    """Buffers shared by every per-n launch plan of one static plan (only one plan runs at a time):
    device work buffers for up to ``cap`` tracks and two pinned host blocks.  Plans are views."""

    def __init__(self, eng, P, ncap, cap):
        dev, dt, f32 = eng.device, eng.dtype, torch.float32
        Cc, S, O = eng.C, eng.s_res, eng.o_res
        self.cap, self.ncap = cap, ncap
        tmax = ncap + cap
        self.inputs = torch.zeros((10 * cap,), dtype=f32, device=dev)
        self.inputs_host = torch.zeros((10 * cap,), dtype=f32).pin_memory()
        self.res = torch.zeros((1 + 7 * tmax + cap,), dtype=f32, device=dev)
        self.cat_boxes = torch.zeros((tmax, 4), dtype=f32, device=dev)
        self.host = torch.zeros((1 + 7 * tmax + cap + 1 + ncap,), dtype=f32).pin_memory()
        self.srf = torch.zeros((cap * S * S * Cc,), dtype=dt, device=dev)
        # channel-planar search windows (developer switch SMOT_XCORR_PLANAR): zero-filled once, the pad columns stay zero
        self.srp = torch.zeros((cap * Cc * _lib.XCORR_PLANE,), dtype=dt, device=dev) if eng.xcorr_planar_ok() else None
        self.tmpl = torch.zeros((cap * eng.t_res * eng.t_res * Cc,), dtype=dt, device=dev)   # the frame's templates (fixed address)
        self.resp = torch.zeros((cap * O * O * Cc,), dtype=dt, device=dev)
        self.tower = torch.zeros((cap * O * O * 2 * Cc,), dtype=dt, device=dev)
        self.maps = torch.zeros((cap * O * O * 8,), dtype=f32, device=dev)
        self.tb = torch.zeros((cap, 4), dtype=f32, device=dev)
        self.conf = torch.zeros((cap,), dtype=f32, device=dev)
        self.valid = torch.zeros((cap,), dtype=torch.int32, device=dev)
        self.scratch = torch.zeros((cap,), dtype=torch.int64, device=dev)
        self.box = eng._box_buffers(cap)
        self.staged_mem = None   # the Memory whose inputs currently sit in self.inputs (device)
        self.done = torch.cuda.Event()


class _TrackPlan(object):
    """Launch list of the track-dependent stage for exactly n tracks in memory (cached per n):
    SR ROIAlign -> xcorr -> towers+GN -> heads -> fused decode -> box-head refinement -> candidate
    assembly -> solver NMS, then ONE device->host copy of the result block.  All operands except the
    template features are views of the shared _TrackArena; the small per-track inputs (search regions,
    template boxes, labels, active flags) arrive in one host->device copy."""

    def __init__(self, eng, P, n, arena, det=None, persistent=True):
        dev, dt, cfg = eng.device, eng.dtype, eng.cfg
        L = lib()
        self.e, self.P, self.n, self.arena = eng, P, n, arena
        A = arena
        det_boxes, det_scores, det_block = det if det is not None else (P.det_boxes, P.det_scores, P.det_block)
        self.det_block = det_block
        self.keep_det = (det_boxes, det_scores)
        ncap = det_boxes.shape[0]
        assert ncap == A.ncap and n <= A.cap
        total = ncap + n
        self.ncap, self.total = ncap, total
        self.keep, self.steps = [], []
        self.graph, self.warm = None, False
        self.part_graphs, self.part_warm = [None, None], [False, False]
        self.det_is_static = det is None or persistent   # one-off plans over foreign detection arrays are not worth capturing
        f32 = torch.float32
        # ---- inputs block: sr (4n) | boxes (4n) | labels (n, int32 bits) | active (n)
        self.inputs = A.inputs[:max(10 * n, 1)]
        self.inputs_host = A.inputs_host[:max(10 * n, 1)]
        self.sr = A.inputs[0:4 * n].view(n, 4)
        self.boxes = A.inputs[4 * n:8 * n].view(n, 4)
        self.labels = A.inputs[8 * n:9 * n].view(torch.int32)
        self.active = A.inputs[9 * n:10 * n]
        # ---- result block: kept_boxes (4t, 16B aligned for float4 stores) | keep_cnt | keep_idx (t) | kept_scores (t) | cat_scores (t)
        #      [| perm (n): candidate position -> memory row, only with more than one foreground class]
        t = max(total, 1)
        self.grouped = bool(n) and eng.ncls > 2
        rlen = 1 + 7 * t + (n if self.grouped else 0)
        self.res = A.res[:rlen]
        self.kept_boxes = self.res[0:4 * t].view(t, 4)
        self.keep_cnt = self.res[4 * t:4 * t + 1].view(torch.int32)
        self.keep_idx = self.res[4 * t + 1:5 * t + 1].view(torch.int32)
        self.kept_scores = self.res[5 * t + 1:6 * t + 1]
        self.cat_scores = self.res[6 * t + 1:7 * t + 1]
        self.perm = self.res[7 * t + 1:7 * t + 1 + n].view(torch.int32) if self.grouped else None
        self.cat_boxes = A.cat_boxes[:t]
        self.host_res = A.host[:rlen]
        self.host_det = A.host[rlen:rlen + 1 + ncap].view(torch.int32)
        self.done = A.done
        T = cfg.MODEL.TRACK_HEAD
        Cc, S, O, Tr = eng.C, eng.s_res, eng.o_res, eng.t_res
        dc = _lib.dtype_code(dt)
        self.xcorr_slot = None
        if n:
            self.srf = A.srf[:n * S * S * Cc].view(n, S, S, Cc)
            self.tmpl = A.tmpl[:n * Tr * Tr * Cc].view(n, Tr, Tr, Cc)
            self.resp = A.resp[:n * O * O * Cc].view(n, O, O, Cc)
            self.tower = A.tower[:n * O * O * 2 * Cc].view(n, O, O, 2 * Cc)
            self.maps = A.maps[:n * O * O * 8].view(n, O, O, 8)
            self.tb, self.conf, self.valid, self.scratch = A.tb[:n], A.conf[:n], A.valid[:n], A.scratch[:n]
            pyr_pad = ops.make_pyramid(P.feats, T.POOLER_SCALES, eng.pads)
            self.keep.append(pyr_pad)
            self.xcorr_kernel = "xcorr_mma_kernel (smot_xcorr)" if dt == torch.float16 else "xcorr_kernel (smot_xcorr)"
            if A.srp is not None:
                # search windows exchanged channel-planar: the correlation stages them with bulk copies (DESIGN.md 5.2)
                self.srp = A.srp[:n * Cc * _lib.XCORR_PLANE].view(n, Cc, _lib.XCORR_PLANE)
                self.steps.append((L.smot_roi_align_planar, (C.byref(pyr_pad), ops._ptr(self.sr), ops._ptr(self.boxes), None, n, Cc,
                                                             S, T.POOLER_SAMPLING_RATIO, ops._ptr(self.srp), _lib.XCORR_ROW_PITCH,
                                                             _lib.XCORR_PLANE, dc), "sr_roi_align"))
                self.xcorr_slot = len(self.steps)
                self.steps.append((L.smot_xcorr_planar_mode, (ops._ptr(self.srp), ops._ptr(self.tmpl), ops._ptr(self.resp), n, Cc,
                                                              eng.xcorr_planar_mode), "xcorr"))
                # the library's rule (csrc/emm.cu smot_xcorr_planar_mode): the flat form only under its developer switch
                flat = os.environ.get("SMOT_XCORR_FLAT", "0") == "1" and n * Cc <= 28 * eng.sm_count()
                self.xcorr_kernel = ("xcorr_flat_kernel<%d> (smot_xcorr_planar_mode)" if flat
                                     else "xcorr_planar_kernel<%d,CG> (smot_xcorr_planar_mode)") % eng.xcorr_planar_mode
                self.xcorr_note = ("fp16 banded-Toeplitz mma.sync form on channel-planar windows staged with cp.async.bulk (one mbarrier "
                                   "per plane pair); mode 1 = structurally-zero MMA halves dropped (45 instead of 60 k16-MMAs per plane); "
                                   "CG = 16 planes per CTA while all CTAs are co-resident, else 8; bound by shared-memory wavefronts "
                                   "(~137 per plane) and the launch -> dependency wait -> L2 round trip -> drain chain (DESIGN.md 5.2)")
            else:
                self.steps.append((L.smot_roi_align, (C.byref(pyr_pad), ops._ptr(self.sr), ops._ptr(self.boxes), None, n, Cc, S,
                                                      T.POOLER_SAMPLING_RATIO, ops._ptr(self.srf), dc), "sr_roi_align"))
                self.xcorr_slot = len(self.steps)
                self.steps.append((L.smot_xcorr, (ops._ptr(self.srf), ops._ptr(self.tmpl), ops._ptr(self.resp), n, Cc, S, Tr, dc),
                                   "xcorr"))
            self._conv(self.resp, "emm.towers", self.tower, pad=1)
            self.steps.append((L.smot_groupnorm_relu, (ops._ptr(self.tower), ops._ptr(eng.gn_gamma), ops._ptr(eng.gn_beta), n,
                                                       O * O, 2 * Cc, 2 * Cc, 2 * cfg.MODEL.GROUP_NORM.NUM_GROUPS,
                                                       cfg.MODEL.GROUP_NORM.EPSILON, 1, dc), "emm_gn"))
            self._conv(self.tower[..., :Cc], "emm.clsctr", self.maps[..., 0:3], pad=1)
            self._conv(self.tower[..., Cc:], "emm.reg", self.maps[..., 3:7], pad=1, relu=True)
            self.steps.append((L.smot_emm_decode, (ops._ptr(self.maps), 8, n, O, eng.up, Tr, ops._ptr(self.sr), ops._ptr(self.boxes),
                                                   ops._ptr(eng.hann), float(T.PAD_PIXELS), int(T.EMM.USE_CENTERNESS),
                                                   float(T.EMM.COSINE_WINDOW_WEIGHT), P.W, P.H, int(cfg.INPUT.AMODAL),
                                                   ops._ptr(self.tb), ops._ptr(self.conf), ops._ptr(self.valid),
                                                   ops._ptr(self.scratch)), "emm_decode"))
            # refinement by the box head (roi_heads.py:60-84)
            self.box = {k: (v[:n] if k in ("pooled", "dec_boxes", "dec_scores") else (v[:, :, :n] if torch.is_tensor(v) else v))
                        for k, v in A.box.items()}
            Q = _Plan(eng, P.H, P.W)
            Q.ws = eng.conv_ws_track   # this stage may run while the other stream executes the next frame's static stage
            Q.feats = P.feats
            eng._box_steps(Q, self.box, self.tb, None, n, self.labels)
            self.keep.append(Q)
            self.steps += [st[:3] for st in Q.steps]
            dec_b, dec_s = self.box["dec_boxes"], self.box["dec_scores"]
        else:
            dec_b = dec_s = None
        if self.grouped:
            # several foreground classes: the reference's class-grouped order / position-paired scores (roi_heads.py:60-84)
            self.steps.append((L.smot_track_combine_grouped, (ops._ptr(det_boxes), ops._ptr(det_scores), ncap, ops._ptr(dec_b),
                                                              ops._ptr(dec_s), eng.ncls, ops._ptr(self.labels), ops._ptr(self.conf),
                                                              ops._ptr(self.valid), ops._ptr(self.active), n, int(T.TRACKTOR),
                                                              ops._ptr(self.cat_boxes), ops._ptr(self.cat_scores),
                                                              ops._ptr(self.keep_cnt), ops._ptr(self.perm)), "track_combine"))
        else:
            self.steps.append((L.smot_track_combine, (ops._ptr(det_boxes), ops._ptr(det_scores), ncap, ops._ptr(dec_b),
                                                      ops._ptr(dec_s), eng.ncls, ops._ptr(self.labels) if n else None,
                                                      ops._ptr(self.conf) if n else None, ops._ptr(self.valid) if n else None,
                                                      ops._ptr(self.active) if n else None, n, int(T.TRACKTOR),
                                                      ops._ptr(self.cat_boxes), ops._ptr(self.cat_scores), ops._ptr(self.keep_cnt)),
                               "track_combine"))
        if total:
            ws = eng.nms_workspace(total)
            self.steps.append((L.smot_sort_nms, (ops._ptr(self.cat_boxes), 4, ops._ptr(self.cat_scores), 1, None, total, -0.5, 0.5,
                                                 total, 0, ops._ptr(self.keep_idx), ops._ptr(self.kept_boxes),
                                                 ops._ptr(self.kept_scores), None, ops._ptr(self.keep_cnt), ops._ptr(ws),
                                                 ws.numel()), "solver_nms"))

    @property
    def staged_mem(self):
        return self.arena.staged_mem

    @staged_mem.setter
    def staged_mem(self, m):
        self.arena.staged_mem = m

    def _conv(self, x, name, out, **kw):
        w, scale, bias = self.e.weights[name]
        d = ops.conv_desc(x, w, out, scale, bias, workspace=self.e.conv_ws_track, **kw)
        self.keep.append(d)
        self.steps.append((lib().smot_conv2d, (C.byref(d),), "conv:" + name))

    def _enqueue(self):
        """The whole stage on the current stream: inputs H2D, kernels, result block D2H (all addresses fixed)."""
        eng = self.e
        st = _lib.stream_ptr()
        if self.n:
            self.inputs.copy_(self.inputs_host, non_blocking=True)
        for i, (fn, args, tag) in enumerate(self.steps):
            if i == self.xcorr_slot and eng.time_kernels:
                with eng.timed("xcorr"):
                    check(fn(*args, st), tag)
            else:
                check(fn(*args, st), tag)
        self.host_res.copy_(self.res, non_blocking=True)
        self.host_det.copy_(self.det_block, non_blocking=True)

    def _enqueue_part(self, part):
        """part 0: inputs H2D .. box-head refinement (needs the frame's feature maps and the memory, not its detections);
        part 1: candidate assembly, solver NMS, result block D2H (needs the detections)."""
        st = _lib.stream_ptr()
        k = next(i for i, stp in enumerate(self.steps) if stp[2] == "track_combine")
        if part == 0:
            if self.n:
                self.inputs.copy_(self.inputs_host, non_blocking=True)
            for fn, args, tag in self.steps[:k]:
                check(fn(*args, st), tag)
        else:
            for fn, args, tag in self.steps[k:]:
                check(fn(*args, st), tag)
            self.host_res.copy_(self.res, non_blocking=True)
            self.host_det.copy_(self.det_block, non_blocking=True)

    def run_split(self, feat, between):
        """The stage in two halves with ``between()`` called after the first is enqueued (SiamMOT.forward's overlap mode waits
        there for the detection tail, which runs meanwhile on another stream).  One CUDA graph per half from the second use."""
        eng = self.e
        if self.n and feat.data_ptr() != self.tmpl.data_ptr():
            self.tmpl.copy_(feat.view(self.tmpl.shape), non_blocking=True)
        use_graph = eng.use_graph and self.det_is_static
        for part in (0, 1):
            if use_graph and self.part_graphs[part] is None and self.part_warm[part]:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self._enqueue_part(part)
                self.part_graphs[part] = g
            if use_graph and self.part_graphs[part] is not None:
                self.part_graphs[part].replay()
            else:
                self._enqueue_part(part)
                self.part_warm[part] = True
            if part == 0:
                between()
        self.done.record()

    def run(self, feat, wait=True):
        """Launch the stage and (wait=True) block on its result block: the frame's only device->host sync.
        The launch list is replayed as a CUDA graph from its second use on (the first use runs it eagerly, which also
        sets kernel attributes); the template features are copied to the plan's fixed buffer first."""
        eng = self.e
        if eng.nvtx:
            torch.cuda.nvtx.range_push("smot/track_stage")
        if self.n and feat.data_ptr() != self.tmpl.data_ptr():
            self.tmpl.copy_(feat.view(self.tmpl.shape), non_blocking=True)
        if eng.use_graph and not (eng.timers is not None and eng.time_kernels) and self.det_is_static:
            if self.graph is None and self.warm:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self._enqueue()
                self.graph = g
            if self.graph is not None:
                self.graph.replay()
            else:
                self._enqueue()
                self.warm = True
        else:
            self._enqueue()
        self.done.record()
        if eng.nvtx:
            torch.cuda.nvtx.range_pop()
        if wait:
            self.done.synchronize()

    def wait(self):
        self.done.synchronize()


class Engine(object):
    def sm_count(self):
        try:
            return torch.cuda.get_device_properties(self.device).multi_processor_count
        except Exception:      # no CUDA runtime (the host-side emulation tests)
            return 132

    def __init__(self, cfg, device="cuda", dtype=None, use_graph=True):
        if not torch.cuda.is_available():
            raise RuntimeError("siammot_b200 needs an sm_90a CUDA device (H100); there is no CPU path")
        lib()  # fail loudly if the CUDA library is missing
        self.cfg = cfg
        self.device = torch.device(device)
        if dtype is None:
            dtype = {"float32": torch.float32, "float16": torch.float16}[cfg.DTYPE]
        self.dtype = dtype
        self.use_graph = use_graph
        self.weights = {}
        self.plans = {}
        from .synthetic import backbone_channels, is_resnet
        from .synthetic import DLA_ARCHS, RESNET_BLOCKS
        if cfg.MODEL.BACKBONE.CONV_BODY not in DLA_ARCHS and cfg.MODEL.BACKBONE.CONV_BODY not in RESNET_BLOCKS:
            raise NotImplementedError("body %s: implemented are %s (dla.py:307-372; DLA-34-FPN is the SURVEY.md section 8 path) and "
                                      "%s (upstream resnet.py; R-50-FPN is BASELINE.json configs[4])"
                                      % (cfg.MODEL.BACKBONE.CONV_BODY, ", ".join(sorted(DLA_ARCHS)), ", ".join(sorted(RESNET_BLOCKS))))
        # configuration switches whose alternatives are not built fail here, loudly, instead of silently computing the default
        unsupported = [("MODEL.ROI_BOX_HEAD.FEATURE_EXTRACTOR", cfg.MODEL.ROI_BOX_HEAD.FEATURE_EXTRACTOR, "FPN2MLPFeatureExtractor"),
                       ("MODEL.ROI_BOX_HEAD.PREDICTOR", cfg.MODEL.ROI_BOX_HEAD.PREDICTOR, "FPNPredictor"),
                       ("MODEL.ROI_BOX_HEAD.USE_GN", cfg.MODEL.ROI_BOX_HEAD.USE_GN, False),
                       ("MODEL.RPN.RPN_HEAD", cfg.MODEL.RPN.RPN_HEAD, "SingleConvRPNHead"),
                       ("MODEL.RPN.USE_FPN", cfg.MODEL.RPN.USE_FPN, True), ("MODEL.ROI_HEADS.USE_FPN", cfg.MODEL.ROI_HEADS.USE_FPN, True),
                       ("MODEL.FPN.USE_GN", cfg.MODEL.FPN.USE_GN, False), ("MODEL.FPN.USE_RELU", cfg.MODEL.FPN.USE_RELU, False),
                       ("MODEL.RPN_ONLY", cfg.MODEL.RPN_ONLY, False), ("MODEL.MASK_ON", cfg.MODEL.MASK_ON, False),
                       ("MODEL.KEYPOINT_ON", cfg.MODEL.KEYPOINT_ON, False), ("MODEL.RETINANET_ON", cfg.MODEL.RETINANET_ON, False)]
        for key, value, supported in unsupported:
            if value != supported:
                raise NotImplementedError("%s = %r: the engine implements %r (the value of every shipped SiamMOT configuration)"
                                          % (key, value, supported))
        if len(cfg.MODEL.RPN.ANCHOR_STRIDE) != 5 or len(cfg.MODEL.RPN.ANCHOR_SIZES) != 5:
            raise NotImplementedError("the FPN RPN runs on five levels (P2..P6): ANCHOR_STRIDE / ANCHOR_SIZES need five entries each")
        self.resnet = is_resnet(cfg)
        if self.resnet:
            R = cfg.MODEL.RESNETS
            if (R.NUM_GROUPS != 1 or R.RES5_DILATION != 1 or any(R.STAGE_WITH_DCN) or R.STEM_FUNC != "StemWithFixedBatchNorm"
                    or R.TRANS_FUNC != "BottleneckWithFixedBatchNorm"):
                raise NotImplementedError("ResNet bodies: only the plain FrozenBN bottleneck form (no groups / dilation / DCN)")
        self.C = backbone_channels(cfg)[1]
        self.ncls = cfg.MODEL.ROI_BOX_HEAD.NUM_CLASSES
        R = cfg.MODEL.RPN
        self.cells = [cell_anchors(st, (sz,), R.ASPECT_RATIOS) for st, sz in zip(R.ANCHOR_STRIDE, R.ANCHOR_SIZES)]
        self.n_anchor = self.cells[0].shape[0]
        T = cfg.MODEL.TRACK_HEAD
        self.t_res = T.POOLER_RESOLUTION
        self.s_res = int(T.POOLER_RESOLUTION * T.SEARCH_REGION)
        self.o_res = self.s_res - self.t_res + 1
        self.up = 16
        self.hann = torch.hann_window(self.o_res * self.up, dtype=torch.float).to(self.device)
        self.pads = [int(T.PAD_PIXELS / ((2 ** i) * 4)) for i in range(len(T.POOLER_SCALES))]
        self._nms_ws = {}
        # split-K scratch: one for the frame-independent stage, one for the track stage -- forward_clip runs the two
        # stages of consecutive frames on different streams, launches within a stage are stream-ordered
        self.conv_ws = ops.conv_workspace(self.device)
        self.conv_ws_track = ops.conv_workspace(self.device)
        # the detection tail (box-head FCs) has its own: in forward_clip's three-stage mode it runs on a third stream while
        # the next frame's backbone uses conv_ws
        self.conv_ws_det = ops.conv_workspace(self.device)
        self._side = None
        self._tail = None
        # SiamMOT.forward: detection tail of the frame on a second stream under the EMM half of its track stage
        # (default; identical tracks; =0 restores the serial order)
        self.frame_overlap = os.environ.get("SMOT_FRAME_OVERLAP", "1") == "1"
        # forward_clip (DESIGN.md section 4): SMOT_CLIP_SPLIT=1 (default) is the three-stage pipeline, which runs the detection
        # tail of frame t on a third stream under the backbone of frame t+1 (round 2: measured 989 / 1071 FPS value / e2e faster
        # than the two-stream pipeline on earlier hardware, identical tracks); SMOT_CLIP_SPLIT=0 = two-stream.
        # SMOT_CLIP_SLOTS = number of static-plan copies of the three-stage pipeline (2 to 4, default 3)
        self.clip_split = os.environ.get("SMOT_CLIP_SPLIT", "1") == "1"
        self.clip_slots = max(2, min(4, int(os.environ.get("SMOT_CLIP_SLOTS", "3"))))
        # forward_clip (three-stage): backbone half over frame pairs (Engine.pair_plan); SMOT_CLIP_PAIRS=0 = one frame per pass
        self.clip_pairs = os.environ.get("SMOT_CLIP_PAIRS", "1") == "1"
        self._pre = None
        self._branch_ws = {}
        self._branch_streams = []
        self._track_plans = {}
        self._arenas = {}
        # SMOT_NVTX=1: NVTX ranges around the stages (see timed())
        self.nvtx = os.environ.get("SMOT_NVTX", "0") == "1"
        # channel-planar search-window exchange (default since round 2: bit-equal windows, 1.5-2x faster correlation on the
        # earlier hardware); 0 = NHWC windows + xcorr_mma_kernel, 1 = planar with the untrimmed MMA phase, 2 = trimmed (libsmot reads it)
        self.xcorr_planar = os.environ.get("SMOT_XCORR_PLANAR", "2") in ("1", "2")
        self.xcorr_planar_mode = 0 if os.environ.get("SMOT_XCORR_PLANAR", "2") == "1" else 1   # the engine passes it per call
        self.timers = None  # optional dict name -> list of (start_event, end_event), see timed()
        self.host_timers = None   # optional dict: host-side seconds per phase of CombinedROIHeads.finish_frame (bench.py)
        self.time_kernels = False  # also bracket single kernels of the track stage (forces its eager path)

    def clip_mode_name(self):
        return ("three-stage clip pipeline (backbone half / detection tail / track stage on three streams, %d static-plan copies)"
                % self.clip_slots) if self.clip_split else "two-stream clip pipeline (static stage / track stage, 2 static-plan copies)"

    def xcorr_planar_ok(self):
        """The planar exchange applies to the fp16 correlation at the TAO geometry (S = 30, T = 15) with C % 16 == 0."""
        return (self.xcorr_planar and self.dtype == torch.float16 and self.s_res == 30 and self.t_res == 15
                and self.C % 16 == 0)

    def timed(self, name):
        """Context manager: when self.timers is a dict, brackets the enclosed launches with CUDA events on
        the launching stream (bench.py's live per-kernel timing); with SMOT_NVTX=1 also an NVTX range "smot/<name>"
        (stages: preprocess, static, static_tail, track_stage, next_memory) for `ncu --nvtx --nvtx-include`."""
        if self.timers is None and not self.nvtx:
            return _NO_TIMER          # the common case costs one attribute test, not a class creation per call
        return _Timed(self, name)

    # ------------------------------------------------------------------------------------------
    # weights
    # ------------------------------------------------------------------------------------------
    def load_state_dict(self, sd):
        """sd: flat dict with the reference key layout (SURVEY.md Appendix B)."""
        dev, dt, Wt = self.device, self.dtype, self.weights
        Wt.clear()

        def bn(prefix):
            scale = sd[prefix + ".weight"].float() * sd[prefix + ".running_var"].float().rsqrt()
            bias = sd[prefix + ".bias"].float() - sd[prefix + ".running_mean"].float() * scale
            return _f32(scale, dev), _f32(bias, dev)

        body = "backbone.body."
        pairs = []
        for k in sd:
            if k.startswith(body) and k.endswith(".weight") and sd[k].dim() == 4:
                conv = k[:-len(".weight")]
                leaf = conv.rsplit(".", 1)[1]
                parent = conv.rsplit(".", 1)[0]
                if conv.endswith(".conv2.offset"):
                    # DFConv2d's offset predictor (MODEL.DLA.STAGE_WITH_DCN): a regular 3x3 conv with bias, no FrozenBN
                    Wt[conv[len("backbone."):]] = (_ohwi(sd[k], dt, dev), None, _f32(sd[conv + ".bias"], dev))
                    continue
                if conv.endswith(".conv2.conv"):
                    # ... and its deformable conv: the 3x3 weight read as [Cout][9*Cin] over the sampled columns, then bn2
                    blk = conv[:-len(".conv2.conv")]
                    s_, b_ = bn(blk + ".bn2")
                    w = _ohwi(sd[k], dt, dev)
                    Wt[conv[len("backbone."):]] = (w.reshape(w.shape[0], 1, 1, -1).contiguous(), s_, b_)
                    continue
                if leaf in ("conv1", "conv2", "conv3"):
                    bnn = parent + ".bn" + leaf[-1]
                elif leaf == "conv":
                    bnn = parent + ".bn"
                else:  # Sequential: conv at index i, bn at i+1
                    bnn = parent + "." + str(int(leaf) + 1)
                pairs.append((conv, bnn))
        for conv, bnn in pairs:
            s, b = bn(bnn)
            Wt[conv[len("backbone."):]] = (_ohwi(sd[conv + ".weight"], dt, dev), s, b)
        for i in range(1, 5):
            for kind in ("fpn_inner", "fpn_layer"):
                k = "backbone.fpn.%s%d" % (kind, i)
                Wt["fpn.%s%d" % (kind, i)] = (_ohwi(sd[k + ".weight"], dt, dev), None, _f32(sd[k + ".bias"], dev))
        Wt["rpn.conv"] = (_ohwi(sd["rpn.head.conv.weight"], dt, dev), None, _f32(sd["rpn.head.conv.bias"], dev))
        wp = torch.cat([sd["rpn.head.cls_logits.weight"], sd["rpn.head.bbox_pred.weight"]], 0)
        bp = torch.cat([sd["rpn.head.cls_logits.bias"], sd["rpn.head.bbox_pred.bias"]], 0)
        Wt["rpn.pred"] = (_ohwi(wp, dt, dev), None, _f32(bp, dev))
        pre = "roi_heads.box."
        res = self.cfg.MODEL.ROI_BOX_HEAD.POOLER_RESOLUTION
        w6 = sd[pre + "feature_extractor.fc6.weight"].float()
        rep = w6.shape[0]
        # reference flattens (C, res, res); ROIAlign here emits (res, res, C): permute fc6's input axis once
        w6 = w6.view(rep, self.C, res, res).permute(0, 2, 3, 1).reshape(rep, 1, 1, res * res * self.C)
        Wt["box.fc6"] = (w6.contiguous().to(dev, dt), None, _f32(sd[pre + "feature_extractor.fc6.bias"], dev))
        w7 = sd[pre + "feature_extractor.fc7.weight"].float()
        Wt["box.fc7"] = (w7.reshape(w7.shape[0], 1, 1, w7.shape[1]).contiguous().to(dev, dt), None,
                         _f32(sd[pre + "feature_extractor.fc7.bias"], dev))
        wb, bb = sd[pre + "predictor.bbox_pred.weight"], sd[pre + "predictor.bbox_pred.bias"]
        if self.cfg.MODEL.CLS_AGNOSTIC_BBOX_REG:
            # the predictor has two regressors and every class uses the last one (inference.py:66-72: box_regression[:, -4:],
            # decoded once and repeated per class): replicate that row block per class in the fused GEMM -- same numbers
            wb, bb = wb[-4:].repeat(self.ncls, 1), bb[-4:].repeat(self.ncls)
        wc = torch.cat([sd[pre + "predictor.cls_score.weight"], wb], 0).float()
        bc = torch.cat([sd[pre + "predictor.cls_score.bias"], bb], 0)
        Wt["box.pred"] = (wc.reshape(wc.shape[0], 1, 1, wc.shape[1]).contiguous().to(dev, dt), None, _f32(bc, dev))
        pre = "roi_heads.track.tracker.predictor."
        if self.cfg.MODEL.TRACK_ON:                  # a detector-only model (MODEL.TRACK_ON False, roi_heads.py:92) has no track head
            wt = torch.cat([sd[pre + "cls_tower.0.weight"], sd[pre + "reg_tower.0.weight"]], 0)
            Wt["emm.towers"] = (_ohwi(wt, dt, dev), None, None)
            self.gn_gamma = _f32(torch.cat([sd[pre + "cls_tower.1.weight"], sd[pre + "reg_tower.1.weight"]]), dev)
            self.gn_beta = _f32(torch.cat([sd[pre + "cls_tower.1.bias"], sd[pre + "reg_tower.1.bias"]]), dev)
            wcc = torch.cat([sd[pre + "cls.weight"], sd[pre + "center.weight"]], 0)
            bcc = torch.cat([sd[pre + "cls.bias"], sd[pre + "center.bias"]], 0)
            Wt["emm.clsctr"] = (_ohwi(wcc, dt, dev), None, _f32(bcc, dev))
            Wt["emm.reg"] = (_ohwi(sd[pre + "reg.weight"], dt, dev), None, _f32(sd[pre + "reg.bias"], dev))
        self.plans.clear()
        self._track_plans.clear()
        self._arenas.clear()

    # ------------------------------------------------------------------------------------------
    # static plan
    # ------------------------------------------------------------------------------------------
    def _tree_general(self, P, name, x, levels, cin, cout, stride, level_root, bottleneck, root_residual, out=None, rootbuf=None,
                      off=None, with_dcn=False):
        """DlaTree (dla.py:192-238) of any depth with either block type (every DLA body, dla.py:307-372) as launches,
        concat-free.  x / out are NHWC views; returns the output view.
        The innermost tree2 of a nest owns the root (dla.py:209-210); its input [x2 | x1 | bottom? | x1 of every enclosing
        tree, outermost first] (dla.py:229-237) is ONE buffer allocated where the nest starts: every producer writes its
        channel slice in place.  ``rootbuf`` / ``off``: that buffer and its next free channel when this call is the tree2 chain
        of an enclosing tree.  The ``project`` of a tree whose tree1 is itself a tree is dead code (dla.py:228 overwrites its
        result): skipped, results identical."""
        _, H, W, _ = x.shape
        Ho, Wo = H // stride, W // stride
        if rootbuf is None:
            total = 2 * cout + (cin if level_root else 0) + (levels - 1) * cout
            rootbuf = P.new(Ho, Wo, total)
            off = 2 * cout
        else:
            assert not level_root and stride == 1
        bottom = x
        if level_root:
            assert stride > 1, "level_root trees of the DLA family down-sample"
            bottom = rootbuf[..., off:off + cin]
            P.call(lib().smot_maxpool2x2, self._pool_args(x, bottom), "maxpool:" + name)
            off += cin
        elif stride > 1 and levels == 1:
            bottom = P.new(Ho, Wo, cin)
            P.call(lib().smot_maxpool2x2, self._pool_args(x, bottom), "maxpool:" + name)
        if levels > 1:
            t1 = rootbuf[..., off:off + cout]
            self._tree_general(P, name + ".tree1", x, levels - 1, cin, cout, stride, False, bottleneck, root_residual, out=t1,
                               with_dcn=with_dcn)
            return self._tree_general(P, name + ".tree2", t1, levels - 1, cout, cout, 1, False, bottleneck, root_residual,
                                      out=out, rootbuf=rootbuf, off=off + cout, with_dcn=with_dcn)
        assert off == rootbuf.shape[3], (name, off, rootbuf.shape)
        if cin != cout:
            residual = P.new(Ho, Wo, cout)
            P.conv(bottom, "body." + name + ".project.0", residual)
        else:
            residual = bottom
        x2v, x1v = rootbuf[..., 0:cout], rootbuf[..., cout:2 * cout]

        def block(pre, inp, outv, s, res):
            if bottleneck:                                     # DlaBottleneck (dla.py:63-101): mid = out / 2
                mid = cout // 2
                a = P.conv(inp, pre + ".conv1", P.new(inp.shape[1], inp.shape[2], mid), relu=True)
                if with_dcn and bottleneck:
                    # DFConv2d (dla.py:74-78): offsets from a regular 3x3 conv (fp32), bilinear gather of the 9 taps, then the
                    # deformable conv proper as a GEMM over the 9*mid gathered columns (+ bn2 + ReLU in its epilogue)
                    offs = P.new(Ho, Wo, 20, dtype=torch.float32)
                    P.conv(a, pre + ".conv2.offset", offs[..., :18], stride=s, pad=1)
                    cols = P.new(Ho, Wo, 9 * mid)
                    P.call(lib().smot_deform_im2col3x3, (ops._ptr(a), ops._ptr(offs), ops._ptr(cols), a.shape[1], a.shape[2], mid,
                                                          ops._nhwc(a)[4], 20, Ho, Wo, 9 * mid, s, _lib.dtype_code(self.dtype)),
                           "deform_im2col:" + pre)
                    b = P.conv(cols, pre + ".conv2.conv", P.new(Ho, Wo, mid), relu=True)
                else:
                    b = P.conv(a, pre + ".conv2", P.new(Ho, Wo, mid), stride=s, pad=1, relu=True)
                P.conv(b, pre + ".conv3", outv, residual=res, relu=True)
            else:                                              # DlaBasic (dla.py:30-57)
                a = P.conv(inp, pre + ".conv1", P.new(Ho, Wo, cout), stride=s, pad=1, relu=True)
                P.conv(a, pre + ".conv2", outv, residual=res, pad=1, relu=True)
        block("body." + name + ".tree1", x, x1v, stride, residual)
        block("body." + name + ".tree2", x1v, x2v, 1, x1v)
        if out is None:
            out = P.new(Ho, Wo, cout)
        P.conv(rootbuf, "body." + name + ".root.conv", out, residual=x2v if root_residual else None, relu=True)
        return out

    def _dla_body_general(self, P, img):
        """DLA.forward (dla.py:289-304) for every member of the DLA family (synthetic.DLA_ARCHS), DLA-34 included."""
        from .synthetic import DLA_ARCHS
        A = DLA_ARCHS[self.cfg.MODEL.BACKBONE.CONV_BODY]
        ch, lv = A["channels"], A["levels"]
        H, W = img.shape[1], img.shape[2]
        x = P.conv(img[..., :3], "body.base_layer.0", P.new(H, W, ch[0]), pad=3, relu=True)
        for name, n, stride, c in (("level0", lv[0], 1, ch[0]), ("level1", lv[1], 2, ch[1])):
            for i in range(n):
                s_ = stride if i == 0 else 1
                x = P.conv(x, "body.%s.%d" % (name, 3 * i), P.new(x.shape[1] // s_, x.shape[2] // s_, c), stride=s_, pad=1, relu=True)
        outs = []
        for lvl in range(2, 6):
            x = self._tree_general(P, "level%d" % lvl, x, lv[lvl], ch[lvl - 1], ch[lvl], 2, lvl > 2, A["block"] == "bottleneck",
                                   A["residual_root"], with_dcn=bool(self.cfg.MODEL.DLA.STAGE_WITH_DCN[lvl]))
            outs.append(x)
        return outs

    def _resnet_body(self, P, img):
        """Upstream maskrcnn_benchmark ResNet-50 (modeling/backbone/resnet.py, "R-50-FPN") as launches: stem 7x7/2 + FrozenBN +
        ReLU, 3x3/2 max-pool, four stages of bottleneck blocks (1x1 -> 3x3 -> 1x1, FrozenBN / ReLU / residual in the conv
        epilogues).  With STRIDE_IN_1X1 the strided 1x1 convs of a stage's first block (conv1 and the identity projection) read
        only the even pixels: the input is subsampled once (smot_subsample2) and both run as plain GEMMs on the tensor cores.
        Returns [C2, C3, C4, C5]."""
        L = lib()
        cfg = self.cfg
        R = cfg.MODEL.RESNETS
        dc = _lib.dtype_code(self.dtype)
        H, W = img.shape[1], img.shape[2]
        stem = R.STEM_OUT_CHANNELS
        H2, W2 = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        x = P.conv(img[..., :3], "body.stem.conv1", P.new(H2, W2, stem), stride=2, pad=3, relu=True)
        H4, W4 = (H2 - 1) // 2 + 1, (W2 - 1) // 2 + 1
        pooled = P.new(H4, W4, stem)
        P.call(L.smot_maxpool3x3s2, self._pool_args(x, pooled), "stem_pool")
        x, cin = pooled, stem
        outs = []
        from .synthetic import RESNET_BLOCKS
        for li, nb in enumerate(RESNET_BLOCKS[cfg.MODEL.BACKBONE.CONV_BODY]):
            mid, cout = R.NUM_GROUPS * R.WIDTH_PER_GROUP * 2 ** li, R.RES2_OUT_CHANNELS * 2 ** li
            for b in range(nb):
                name = "body.layer%d.%d" % (li + 1, b)
                stride = 2 if (b == 0 and li > 0) else 1
                s1, s3 = (stride, 1) if R.STRIDE_IN_1X1 else (1, stride)
                h, w = x.shape[1], x.shape[2]
                ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
                xs = x
                if stride == 2:   # the even pixels, once, for every strided 1x1 of the block
                    xs = P.new(ho, wo, cin)
                    P.per_image(L.smot_subsample2, lambda b, x=x, xs=xs, h=h, w=w, cin=cin: (ops._ptr(x[b:b + 1]), ops._ptr(xs[b:b + 1]), h, w,
                                                                                              cin, ops._nhwc(x)[4], cin, dc), "sub2:" + name)
                identity = x
                if cin != cout:
                    identity = P.conv(xs, name + ".downsample.0", P.new(ho, wo, cout))
                a = P.conv(xs if s1 == 2 else x, name + ".conv1", P.new(ho if s1 == 2 else h, wo if s1 == 2 else w, mid), relu=True)
                bmap = P.conv(a, name + ".conv2", P.new(ho, wo, mid), stride=s3, pad=1, relu=True)
                x = P.conv(bmap, name + ".conv3", P.new(ho, wo, cout), residual=identity, relu=True)
                cin = cout
            outs.append(x)
        return outs

    def _pool_args(self, x, out):
        B, H, W, Cc, ld = ops._nhwc(x)
        return (ops._ptr(x), ops._ptr(out), B, H, W, Cc, ld, ops._nhwc(out)[4], _lib.dtype_code(x.dtype))

    def plan(self, H, W, slot=0):
        """Static launch plan (+ its buffers and CUDA graph) for one input size.  ``slot`` selects one of
        several independent copies so that frame t+1 can be in flight while frame t's features are still
        needed (SiamMOT.forward_clip double-buffers with slots 0/1)."""
        key = (H, W, slot)
        if key in self.plans:
            return self.plans[key]
        self._check_plan_size(H, W)
        P = _Plan(self, H, W)
        P.slot = slot
        self._build_static(P)
        self.plans[key] = P
        return P

    def pair_plan(self, H, W, pslot=0):
        """Backbone plan over a PAIR of clip frames (batch 2) + the two per-frame plans that read its halves.

        Below level 2 every DLA / FPN / RPN layer has at most 110..120 CTAs for the 132 SMs of an H100 and costs ~10 us whatever its size
        (launch, barrier setup, TMA round trips, epilogue): run over two frames at once those layers cost
        the same and do twice the work, only the layers that already fill the GPU (stem, level 0-2, P2) double.
        forward_clip's three-stage mode therefore runs the backbone half of frames (2k, 2k+1) as ONE batch-2 pass; the
        detection tail and the track stage stay per frame and read image i of the batched buffers through the frame plans
        ``pair.frames[i]`` (same launch lists as a standalone plan, activation buffers = views).  Results are identical: every
        kernel treats the batch images independently."""
        key = (H, W, "pair", pslot)
        if key in self.plans:
            return self.plans[key]
        self._check_plan_size(H, W)
        PP = _Plan(self, H, W)
        PP.batch = 2
        PP.slot = ("pair", pslot)
        PP.ws = self.conv_ws
        self._build_static(PP, backbone_only=True)
        PP.frames = []
        for i in range(PP.batch):
            P = _Plan(self, H, W)
            P.view_of, P.view_index = PP, i
            P.slot = ("pair", pslot, i)
            P.ws = self.conv_ws
            self._build_static(P)
            if P._cursor != len(PP.bufs):
                raise RuntimeError("frame plan used %d of the pair plan's %d buffers" % (P._cursor, len(PP.bufs)))
            P.pair = PP
            PP.frames.append(P)
        self.plans[key] = PP
        return PP

    def batch_plan(self, H, W, B):
        """Static plan of the whole frame-independent stage (backbone, FPN, RPN heads, proposal selection, box head, per-class
        NMS) over B images of one size as ONE launch list, captured as a CUDA graph like the per-frame plans; cached per
        (H, W, B).  The detection tail uses the batched entry points (smot_rpn_select_batched, smot_roi_align_batched,
        smot_box_decode_batched, smot_sort_nms_segmented) and the box-head GEMMs run as B images of 1 x nprop rows, so every
        image's detections equal those of plan(H, W) on that image bit for bit.  Outputs: det_boxes (B, cap, 4), det_scores
        (B, cap), det_block (B, 1 + cap) = count | labels.  B = 1 is plan(H, W)."""
        if B < 2:
            raise ValueError("batch_plan is for B >= 2 images (B = 1 runs on Engine.plan)")
        key = (H, W, "batch", B)
        if key in self.plans:
            return self.plans[key]
        self._check_plan_size(H, W)
        P = _Plan(self, H, W)
        P.batch = B
        P.batched = True
        P.slot = ("batch", B)
        # Split-K scratch scaled to B images.  A layer's split factor depends on one image's tiles, but it is taken only when
        # the partial tiles of the whole batch fit the scratch: B times the single-image room keeps every split decision, and
        # with it the fp32 summation order, equal to the B = 1 plan's.
        nbytes = _lib.CONV_WS_COUNTER_BYTES + B * (self.conv_ws.numel() - _lib.CONV_WS_COUNTER_BYTES)
        P.ws = ops.conv_workspace(self.device, nbytes)
        P.branch_wss = [ops.conv_workspace(self.device, nbytes) for _ in range(4)]
        P.det_ws = ops.conv_workspace(self.device, _lib.CONV_WS_COUNTER_BYTES + B * (self.conv_ws_det.numel()
                                                                                      - _lib.CONV_WS_COUNTER_BYTES))
        P.keep += [P.ws, P.det_ws] + P.branch_wss
        self._build_static(P)
        self.plans[key] = P
        return P

    def run_batch(self, images):
        """images: (B, 3, H, W) float tensor (any device), B >= 2.  Enqueues batch_plan(H, W, B) on the current stream."""
        B, _, H, W = images.shape
        P = self.batch_plan(H, W, B)
        P.img_batch.copy_(images, non_blocking=True)
        with self.timed("static"):
            P.run()
        return P

    def _check_plan_size(self, H, W):
        if not self.weights:
            raise RuntimeError("Engine.load_state_dict() must be called before the first frame")
        if H % 32 or W % 32:
            raise ValueError("DLA-34 needs an input divisible by 32 (got %dx%d); the reference resizes to such a size "
                             "(DATALOADER.SIZE_DIVISIBILITY 32) and fails in dla.py:54 otherwise" % (H, W))

    def _build_static(self, P, backbone_only=False):
        """Fill plan P with the launches of the frame-independent stage (P.batch images per pass); backbone_only: stop after
        the RPN heads (part 0 of the plan)."""
        H, W = P.H, P.W
        cfg, dev, dt = self.cfg, self.device, self.dtype
        L = lib()
        dc = _lib.dtype_code(dt)
        # ---- input: (batch, 3, H, W) fp32; a frame plan of a pair reads / is fed through its image of the pair's buffer
        if P.view_of is not None:
            P.img_batch = P.view_of.img_batch[P.view_index:P.view_index + 1]
        else:
            P.img_batch = torch.zeros((P.batch, 3, H, W), dtype=torch.float32, device=dev)
        P.img_in = P.img_batch[0]
        img = P.new(H, W, 4)
        P.per_image(L.smot_image_to_nhwc, lambda i: (ops._ptr(P.img_batch[i]), ops._ptr(img[i:i + 1]), 3, H, W, 4, dc), "image_to_nhwc")
        body = self._resnet_body(P, img) if self.resnet else self._dla_body_general(P, img)
        # ---- FPN (fpn_patch.py:29-61)
        Cc = self.C
        R = cfg.MODEL.RPN
        A = self.n_anchor
        hld = ((5 * A + 3) // 4) * 4
        feats, heads, inner = [None] * 5, [None] * 5, [None] * 4
        P.fork(4)                                   # the four lateral 1x1 convs are independent
        for i in range(4, 0, -1):
            f = body[i - 1]
            P.branch = 4 - i
            inner[i - 1] = P.conv(f, "fpn.fpn_inner%d" % i, P.new(f.shape[1], f.shape[2], Cc))
        P.join()
        for i in range(3, 0, -1):                   # top-down pathway: sequential
            last, cur = inner[i], inner[i - 1]
            P.per_image(L.smot_upsample_add, lambda b, last=last, cur=cur: (ops._ptr(last[b:b + 1]), last.shape[1], last.shape[2], Cc,
                                                                              ops._ptr(cur[b:b + 1]), cur.shape[1], cur.shape[2], Cc, Cc, dc),
                        "upsample_add%d" % (i + 1))

        def rpn_head(l):
            f = feats[l]
            t = P.conv(f, "rpn.conv", P.new(f.shape[1], f.shape[2], Cc), pad=1, relu=True)
            heads[l] = P.new(f.shape[1], f.shape[2], hld, dtype=torch.float32)
            P.conv(t, "rpn.pred", heads[l][..., :5 * A])

        P.fork(4)                                   # per level: FPN output conv -> RPN conv -> RPN predictor
        for l in range(4):
            P.branch = l
            feats[l] = P.conv(inner[l], "fpn.fpn_layer%d" % (l + 1), P.new(inner[l].shape[1], inner[l].shape[2], Cc), pad=1)
            rpn_head(l)
            if l == 3:                              # P6 = stride-2 subsample of P5 (fpn_patch.py:57-59), same branch
                p5 = feats[3]
                feats[4] = P.new((p5.shape[1] - 1) // 2 + 1, (p5.shape[2] - 1) // 2 + 1, Cc)
                P.per_image(L.smot_subsample2, lambda b, p5=p5: (ops._ptr(p5[b:b + 1]), ops._ptr(feats[4][b:b + 1]), p5.shape[1],
                                                                  p5.shape[2], Cc, Cc, Cc, dc), "p6")
                rpn_head(4)
        P.join()
        P.feats = feats
        if backbone_only:
            return
        if P.batched:
            return self._batched_tail(P, heads, feats)
        if P.batch != 1:
            raise RuntimeError("the detection tail runs per frame: build it on a frame plan (Engine.pair_plan(...).frames[i])")
        # ---- RPN selection
        P.rpn_levels = ops.rpn_levels(heads, R.ANCHOR_STRIDE, self.cells)
        P.keep.append(P.rpn_levels)
        nprop = R.FPN_POST_NMS_TOP_N_TEST
        P.props = torch.zeros((nprop, 4), dtype=torch.float32, device=dev)
        P.prop_scores = torch.zeros((nprop,), dtype=torch.float32, device=dev)
        P.prop_count = torch.zeros((1,), dtype=torch.int32, device=dev)
        ws = ops.rpn_select_workspace(len(feats), R.PRE_NMS_TOP_N_TEST, dev)
        P.keep.append(ws)
        P.call(L.smot_rpn_select, (P.rpn_levels, len(feats), R.PRE_NMS_TOP_N_TEST, R.POST_NMS_TOP_N_TEST,
                                   R.NMS_THRESH, float(R.MIN_SIZE), nprop, W, H, int(cfg.INPUT.AMODAL),
                                   ops._ptr(P.props), ops._ptr(P.prop_scores), ops._ptr(P.prop_count), ops._ptr(ws),
                                   ws.numel()), "rpn_select")
        # ---- box head on the proposals (box_head.py:46-51, inference.py:46-191)
        P.ws = self.conv_ws_det   # split-K scratch of the detection tail (see Engine.__init__)
        P.box = self._box_buffers(nprop)
        self._box_steps(P, P.box, P.props, P.prop_count, nprop, None)
        ncls = self.ncls
        cap = nprop * (ncls - 1)
        P.det_boxes = torch.zeros((cap, 4), dtype=torch.float32, device=dev)
        P.det_scores = torch.zeros((cap,), dtype=torch.float32, device=dev)
        P.det_block = torch.zeros((1 + cap,), dtype=torch.int32, device=dev)   # [count | labels]: one D2H
        P.det_count = P.det_block[0:1]
        P.det_labels = P.det_block[1:]
        nws = ops.sort_nms_workspace(nprop, dev)
        P.keep.append(nws)
        P.call(lambda st: self._fill_dets(P), (), "det_init")
        H_ = cfg.MODEL.ROI_HEADS
        for j in range(1, ncls):
            P.call(L.smot_sort_nms, (C.c_void_p(P.box["dec_boxes"].data_ptr() + 16 * j), 4 * ncls,
                                     C.c_void_p(P.box["dec_scores"].data_ptr() + 4 * j), ncls, ops._ptr(P.prop_count),
                                     nprop, H_.SCORE_THRESH, H_.NMS, nprop, j, None, ops._ptr(P.det_boxes),
                                     ops._ptr(P.det_scores), ops._ptr(P.det_labels), ops._ptr(P.det_count), ops._ptr(nws),
                                     nws.numel()), "det_nms%d" % j)

    def _batched_tail(self, P, heads, feats):
        """The detection tail of a batch plan: the per-frame tail's steps over P.batch images, each step one launch set."""
        cfg, dev, L = self.cfg, self.device, lib()
        B, H, W = P.batch, P.H, P.W
        R, Hh, H_ = cfg.MODEL.RPN, cfg.MODEL.ROI_BOX_HEAD, cfg.MODEL.ROI_HEADS
        ncls, res = self.ncls, Hh.POOLER_RESOLUTION
        # ---- RPN selection, all images
        P.rpn_levels = ops.rpn_levels(heads, R.ANCHOR_STRIDE, self.cells)
        head_strides = ops.image_strides(heads)
        nprop = R.FPN_POST_NMS_TOP_N_TEST
        P.props = torch.zeros((B, nprop, 4), dtype=torch.float32, device=dev)
        P.prop_scores = torch.zeros((B, nprop), dtype=torch.float32, device=dev)
        P.prop_count = torch.zeros((B,), dtype=torch.int32, device=dev)
        ws = ops.rpn_select_batched_workspace(len(feats), R.PRE_NMS_TOP_N_TEST, B, dev)
        P.keep += [P.rpn_levels, head_strides, ws]
        P.call(L.smot_rpn_select_batched, (P.rpn_levels, head_strides, B, len(feats), R.PRE_NMS_TOP_N_TEST, R.POST_NMS_TOP_N_TEST,
                                           R.NMS_THRESH, float(R.MIN_SIZE), nprop, W, H, int(cfg.INPUT.AMODAL), ops._ptr(P.props),
                                           ops._ptr(P.prop_scores), ops._ptr(P.prop_count), ops._ptr(ws), ws.numel()), "rpn_select")
        # ---- box head: ROIAlign over B segments of nprop rows, then fc6 / fc7 / predictor as B images of 1 x nprop rows (the
        # split-K factor is chosen per image, so each image's sums run in the B = 1 order)
        P.ws = P.det_ws
        rep = Hh.MLP_HEAD_DIM
        hld = ((5 * ncls + 3) // 4) * 4
        dt = self.dtype
        box = P.box = dict(pooled=torch.zeros((B * nprop, res, res, self.C), dtype=dt, device=dev),
                           fc6=torch.zeros((B, 1, nprop, rep), dtype=dt, device=dev),
                           fc7=torch.zeros((B, 1, nprop, rep), dtype=dt, device=dev),
                           head=torch.zeros((B, 1, nprop, hld), dtype=torch.float32, device=dev),
                           dec_boxes=torch.zeros((B * nprop, ncls, 4), dtype=torch.float32, device=dev),
                           dec_scores=torch.zeros((B * nprop, ncls), dtype=torch.float32, device=dev), n=nprop)
        pyr = ops.make_pyramid(feats, Hh.POOLER_SCALES)
        feat_strides = ops.image_strides(feats[:len(Hh.POOLER_SCALES)])
        P.keep += [pyr, feat_strides]
        P.call(L.smot_roi_align_batched, (C.byref(pyr), feat_strides, B, ops._ptr(P.props), ops._ptr(P.prop_count), nprop, self.C,
                                          res, Hh.POOLER_SAMPLING_RATIO, ops._ptr(box["pooled"]), _lib.dtype_code(dt)), "box_roi_align")
        P.conv(box["pooled"].view(B, 1, nprop, res * res * self.C), "box.fc6", box["fc6"], relu=True)
        P.conv(box["fc6"], "box.fc7", box["fc7"], relu=True)
        P.conv(box["fc7"], "box.pred", box["head"][..., :5 * ncls])
        w4 = (C.c_float * 4)(*[float(w) for w in H_.BBOX_REG_WEIGHTS])
        P.keep.append(w4)
        P.call(L.smot_box_decode_batched, (ops._ptr(box["head"]), hld, ops._ptr(P.props), ops._ptr(P.prop_count), B, nprop, ncls,
                                           C.byref(w4), W, H, int(cfg.INPUT.AMODAL), ops._ptr(box["dec_boxes"]),
                                           ops._ptr(box["dec_scores"])), "box_decode")
        # ---- per-class NMS of every (image, class) segment into per-image blocks
        cap = nprop * (ncls - 1)
        # boxes | scores | [count | labels] of all images in ONE buffer: the batch's results leave in one copy
        P.det_packed = torch.zeros((B * (6 * cap + 1),), dtype=torch.float32, device=dev)
        P.det_boxes = P.det_packed[:B * cap * 4].view(B, cap, 4)
        P.det_scores = P.det_packed[B * cap * 4:B * cap * 5].view(B, cap)
        P.det_block = P.det_packed[B * cap * 5:].view(torch.int32).view(B, 1 + cap)
        nws = ops.sort_nms_segmented_workspace(B, ncls, nprop, dev)
        P.keep.append(nws)
        P.call(L.smot_sort_nms_segmented, (ops._ptr(box["dec_boxes"]), ops._ptr(box["dec_scores"]), ops._ptr(P.prop_count), B, nprop,
                                           ncls, H_.SCORE_THRESH, H_.NMS, nprop, cap, ops._ptr(P.det_boxes), ops._ptr(P.det_scores),
                                           ops._ptr(P.det_block), ops._ptr(nws), nws.numel()), "det_nms")

    def _fill_dets(self, P):
        P.det_scores.fill_(-1.0)
        P.det_count.zero_()
        return 0

    def _box_buffers(self, n):
        dev, dt, ncls = self.device, self.dtype, self.ncls
        res = self.cfg.MODEL.ROI_BOX_HEAD.POOLER_RESOLUTION
        rep = self.cfg.MODEL.ROI_BOX_HEAD.MLP_HEAD_DIM
        hld = ((5 * ncls + 3) // 4) * 4
        return dict(pooled=torch.zeros((n, res, res, self.C), dtype=dt, device=dev),
                    fc6=torch.zeros((1, 1, n, rep), dtype=dt, device=dev),
                    fc7=torch.zeros((1, 1, n, rep), dtype=dt, device=dev),
                    head=torch.zeros((1, 1, n, hld), dtype=torch.float32, device=dev),
                    dec_boxes=torch.zeros((n, ncls, 4), dtype=torch.float32, device=dev),
                    dec_scores=torch.zeros((n, ncls), dtype=torch.float32, device=dev), n=n)

    def _box_steps(self, P, B, rois, count, n, track_labels):
        """ROIAlign 7x7 -> fc6 -> fc7 -> [cls | bbox] -> softmax/decode.  Appends launches to plan P."""
        cfg, L = self.cfg, lib()
        Hh = cfg.MODEL.ROI_BOX_HEAD
        res = Hh.POOLER_RESOLUTION
        pyr = ops.make_pyramid(P.feats, Hh.POOLER_SCALES)
        P.keep.append(pyr)
        P.call(L.smot_roi_align, (C.byref(pyr), ops._ptr(rois), None, ops._ptr(count), n, self.C, res,
                                  Hh.POOLER_SAMPLING_RATIO, ops._ptr(B["pooled"]), _lib.dtype_code(self.dtype)), "box_roi_align")
        P.conv(B["pooled"].view(1, 1, n, res * res * self.C), "box.fc6", B["fc6"], relu=True)
        P.conv(B["fc6"], "box.fc7", B["fc7"], relu=True)
        P.conv(B["fc7"], "box.pred", B["head"][..., :5 * self.ncls])
        w4 = (C.c_float * 4)(*[float(w) for w in cfg.MODEL.ROI_HEADS.BBOX_REG_WEIGHTS])
        P.keep.append(w4)
        P.call(L.smot_box_decode, (ops._ptr(B["head"]), B["head"].shape[3], ops._ptr(rois), ops._ptr(count), n, self.ncls,
                                   C.byref(w4), P.W, P.H, int(cfg.INPUT.AMODAL), ops._ptr(track_labels),
                                   ops._ptr(B["dec_boxes"]), ops._ptr(B["dec_scores"])), "box_decode")

    # ------------------------------------------------------------------------------------------
    # per-frame entry points
    # ------------------------------------------------------------------------------------------
    def branch_ws(self, b):
        """Split-K scratch of parallel branch b (concurrent convolutions must not share one).  Every plan shares it: the
        backbone halves, which hold the branches, run one after another on one stream."""
        if b not in self._branch_ws:
            self._branch_ws[b] = ops.conv_workspace(self.device)
        return self._branch_ws[b]

    def branch_streams(self, n):
        while len(self._branch_streams) < n:
            self._branch_streams.append(torch.cuda.Stream(device=self.device))
        return self._branch_streams[:n]

    def side_stream(self):
        """The stream forward_clip runs the frame-independent stage on (created on first use)."""
        if self._side is None:
            self._side = torch.cuda.Stream(device=self.device)
        return self._side

    def tail_stream(self):
        """The stream of the detection tail (three-stage clip mode, per-frame overlap mode)."""
        if self._tail is None:
            self._tail = torch.cuda.Stream(device=self.device)
        return self._tail

    def run_static(self, image, slot=0, part=None):
        """image: (3,H,W) or (1,3,H,W) float tensor (any device).  Enqueues backbone..detections on the current stream.
        part=0: only the input copy and the backbone / FPN / RPN-head half (the detection tail follows with run_tail)."""
        if image.dim() == 4:
            if image.shape[0] != 1:
                raise ValueError("one image per forward (track_core.py:75 asserts the same)")
            image = image[0]
        P = self.plan(image.shape[1], image.shape[2], slot)
        P.img_in.copy_(image, non_blocking=True)
        with self.timed("static"):
            P.run() if part is None else P.run_part(part)
        return P

    def pair_ok(self, frames):
        """Frame pairs need kernels that take a batch (everything but the DCN gather) and frames of one size and kind."""
        if any(self.cfg.MODEL.DLA.STAGE_WITH_DCN) and not self.resnet and self.cfg.MODEL.BACKBONE.CONV_BODY != "DLA-34-FPN":
            return False
        f0 = frames[0]
        raw = not torch.is_tensor(f0) or f0.dtype == torch.uint8
        shape = tuple(f0.shape)
        for f in frames:
            if tuple(f.shape) != shape or (not torch.is_tensor(f) or f.dtype == torch.uint8) != raw:
                return False
        return raw or len(shape) == 3 or shape[0] == 1

    def run_backbone_pair(self, f0, f1, pslot):
        """Stage two clip frames (normalised (3,H,W) tensors or decoded uint8 frames) and enqueue ONE batch-2 backbone / FPN /
        RPN-head pass on the current stream.  Returns the pair plan; its .frames[i] are the per-frame plans."""
        raw = not torch.is_tensor(f0) or f0.dtype == torch.uint8
        if raw:
            pre = self.preprocessor()
            H, W = pre.output_size(f0.shape[0], f0.shape[1])
        else:
            H, W = f0.shape[-2], f0.shape[-1]
        PP = self.pair_plan(H, W, pslot)
        for i, f in enumerate((f0, f1)):
            if raw:
                with self.timed("preprocess"):
                    pre.into(f, PP.img_batch[i], 2 * pslot + i)
            else:
                PP.img_batch[i].copy_(f[0] if f.dim() == 4 else f, non_blocking=True)
        with self.timed("static"):
            PP.run_part(0)
        return PP

    def run_tail(self, P):
        """The detection tail (proposal selection, box head, per-class NMS) of a plan whose part 0 has been enqueued."""
        with self.timed("static_tail"):
            P.run_part(1)
        return P

    def preprocessor(self):
        if self._pre is None:
            from .preprocess import FramePreprocessor
            self._pre = FramePreprocessor(self.cfg, self.device)
        return self._pre

    def run_static_raw(self, frame, slot=0, part=None):
        """frame: decoded RGB uint8 (H0, W0, 3) frame (host or device).  The reference's test transform (resize to
        the cfg's test size, ToTensor, Normalize) runs on the device straight into the plan's input buffer, then the
        frame-independent stage is enqueued as in run_static."""
        pre = self.preprocessor()
        oh, ow = pre.output_size(frame.shape[0], frame.shape[1])
        P = self.plan(oh, ow, slot)
        with self.timed("preprocess"):
            pre.into(frame, P.img_in)
        with self.timed("static"):
            P.run() if part is None else P.run_part(part)
        return P

    def box_head_eager(self, P, rois, track_labels=None):
        """Box head on an arbitrary host-sized set of boxes (track refinement roi_heads.py:69, given
        detections roi_heads.py:29).  Returns (dec_boxes (n,ncls,4), dec_scores (n,ncls))."""
        n = rois.shape[0]
        B = self._box_buffers(n)
        Q = _Plan(self, P.H, P.W)
        Q.ws = self.conv_ws_track
        Q.feats = P.feats
        self._box_steps(Q, B, rois, None, n, track_labels)
        Q.keep.append(B)
        Q.run_eager()
        return B["dec_boxes"], B["dec_scores"]

    def emm_track(self, P, mem_feat, mem_sr, mem_boxes):
        """EMM.forward inference branch (track_core.py:28-79) for N tracks; device tensors in, device out:
        boxes (N,4), conf (N,), valid (N,) int32."""
        cfg = self.cfg
        T = cfg.MODEL.TRACK_HEAD
        n = mem_boxes.shape[0]
        if self.xcorr_planar_ok():
            with self.timed("sr_roi_align"):
                srp = ops.roi_align_planar(P.feats, mem_sr, T.POOLER_SCALES, self.s_res, T.POOLER_SAMPLING_RATIO,
                                           level_boxes=mem_boxes, pads=self.pads)
            with self.timed("xcorr"):
                resp = ops.xcorr_planar(srp, mem_feat.contiguous(), mma_mode=self.xcorr_planar_mode)
        else:
            with self.timed("sr_roi_align"):
                srf = ops.roi_align(P.feats, mem_sr, T.POOLER_SCALES, self.s_res, T.POOLER_SAMPLING_RATIO,
                                    level_boxes=mem_boxes, pads=self.pads)
            with self.timed("xcorr"):
                resp = ops.xcorr(srf, mem_feat)
        O, Cc = self.o_res, self.C
        w, _, _ = self.weights["emm.towers"]
        tower = ops.conv2d(resp, w, pad=1)
        ops.groupnorm_relu_(tower, self.gn_gamma, self.gn_beta, 2 * self.cfg.MODEL.GROUP_NORM.NUM_GROUPS,
                            self.cfg.MODEL.GROUP_NORM.EPSILON, True)
        maps = torch.zeros((n, O, O, 8), dtype=torch.float32, device=self.device)
        w, _, b = self.weights["emm.clsctr"]
        ops.conv2d(tower[..., :Cc], w, None, b, pad=1, out=maps[..., 0:3])
        w, _, b = self.weights["emm.reg"]
        ops.conv2d(tower[..., Cc:], w, None, b, pad=1, relu=True, out=maps[..., 3:7])
        self.last_maps = maps
        return ops.emm_decode(maps, mem_sr, mem_boxes, self.hann, self.up, self.t_res, T.PAD_PIXELS,
                              T.EMM.USE_CENTERNESS, T.EMM.COSINE_WINDOW_WEIGHT, P.W, P.H, cfg.INPUT.AMODAL)

    def templates_into(self, P, tp, n_act, feat):
        """templates() for the clip / per-frame hot path: the first n_act boxes of track plan tp (already on the device at a
        fixed address) -> feat[:n_act], one ctypes call without the generic wrapper's checks and views."""
        T = self.cfg.MODEL.TRACK_HEAD
        if getattr(P, "pyr_plain", None) is None:
            P.pyr_plain = ops.make_pyramid(P.feats, T.POOLER_SCALES)
            P.pyr_plain_ref = C.byref(P.pyr_plain)
        bp = getattr(tp, "boxes_ptr", None)
        if bp is None:
            bp = tp.boxes_ptr = C.c_void_p(tp.boxes.data_ptr())
        check(lib().smot_roi_align(P.pyr_plain_ref, bp, None, None, n_act, self.C, self.t_res, T.POOLER_SAMPLING_RATIO,
                                   C.c_void_p(feat.data_ptr()), _lib.dtype_code(self.dtype), _lib.stream_ptr()), "smot_roi_align")

    def templates(self, P, boxes_dev, out=None):
        """EMM.extract_cache feature part (track_core.py:92): ROIAlign T x T on the unpadded pyramid."""
        T = self.cfg.MODEL.TRACK_HEAD
        if getattr(P, "pyr_plain", None) is None:
            P.pyr_plain = ops.make_pyramid(P.feats, T.POOLER_SCALES)
            P.pyr_plain_ref = C.byref(P.pyr_plain)
        return ops.roi_align(P.feats, boxes_dev, T.POOLER_SCALES, self.t_res, T.POOLER_SAMPLING_RATIO, out=out,
                             pyramid=P.pyr_plain)

    def gather_templates(self, feat, first, sources):
        """feat[first + j] = sources[j][0][sources[j][1]]: the cached templates of dormant tracks (rows of earlier frames'
        template tensors, track_head.py:77-97) appended behind the active tracks' templates.  Device-side, current stream.
        Consecutive rows of one source tensor move as one slice copy (in steady state the dormant tracks of a video sit in
        the previous memory in the same order: a single copy instead of one indexing op per track)."""
        j, m = 0, len(sources)
        while j < m:
            t, r = sources[j]
            k = j + 1
            while k < m and sources[k][0] is t and sources[k][1] == r + (k - j):
                k += 1
            feat[first + j:first + k].copy_(t[r:r + (k - j)], non_blocking=True)
            j = k

    def track_arena(self, P, n, ncap=None):
        """The shared buffer arena of static plan P, grown (x2) when n exceeds its capacity."""
        ncap = P.det_boxes.shape[0] if ncap is None else ncap
        key = (P.H, P.W, getattr(P, "slot", 0), ncap)
        A = self._arenas.get(key)
        if A is None or A.cap < n:
            cap = 64 if A is None else A.cap
            while cap < n:
                cap *= 2
            old = A
            A = self._arenas[key] = _TrackArena(self, P, ncap, cap)
            for k in [k for k, tp in self._track_plans.items() if tp.arena is old]:   # only the plans that were views of the old arena
                self._track_plans.pop(k)
        return A

    @staticmethod
    def given_capacity(rows):
        """Capacity class of an external-detection set: next power of two >= max(rows, 64).  Arenas, buffers and plans of the
        public-detection path are keyed on the class, not on the frame's detection count (a MOT17 video has dozens of
        distinct counts; one arena per count leaked ~30 MB each)."""
        return max(64, 1 << (max(int(rows), 1) - 1).bit_length())

    def given_buffers(self, P, rows):
        """Persistent (det_boxes, det_scores, det_block) of static plan P for external detections, per capacity class."""
        cap = self.given_capacity(rows)
        bufs = getattr(P, "given_bufs", None)
        if bufs is None:
            bufs = P.given_bufs = {}
        if cap not in bufs:
            dev = self.device
            bufs[cap] = (torch.zeros((cap, 4), dtype=torch.float32, device=dev),
                         torch.full((cap,), -1.0, dtype=torch.float32, device=dev),
                         torch.zeros((1 + cap,), dtype=torch.int32, device=dev))
        return bufs[cap]

    def track_plan(self, P, n, det=None):
        if det is not None:
            # external detections: their arrays are the plan's persistent per-capacity buffers (given_buffers), so the plan is
            # cached per (slot, n, capacity) and replayed as a graph like the default one; foreign arrays get a one-off plan
            ncap = det[0].shape[0]
            if getattr(P, "given_bufs", {}).get(ncap, (None,))[0] is not det[0]:
                return _TrackPlan(self, P, n, self.track_arena(P, n, ncap), det=det, persistent=False)
            A = self.track_arena(P, n, ncap)
            key = (P.H, P.W, getattr(P, "slot", 0), n, "given", ncap)
            tp = self._track_plans.get(key)
            if tp is None:
                tp = self._track_plans[key] = _TrackPlan(self, P, n, A, det=det, persistent=True)
            return tp
        A = self.track_arena(P, n)
        key = (P.H, P.W, getattr(P, "slot", 0), n)
        tp = self._track_plans.get(key)
        if tp is None:
            tp = self._track_plans[key] = _TrackPlan(self, P, n, A)
        return tp

    def nms_workspace(self, n):
        n = max(64, 1 << (max(n, 1) - 1).bit_length())
        if n not in self._nms_ws:
            self._nms_ws[n] = ops.sort_nms_workspace(n, self.device)
        return self._nms_ws[n]
