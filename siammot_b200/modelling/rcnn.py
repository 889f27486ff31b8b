"""``build_siammot(cfg)`` -> drop-in replacement of the reference's SiamMOT module
(/root/reference/siammot/modelling/rcnn.py:15-73) for inference.

Same surface: ``forward(images, targets=None, given_detection=None) -> [BoxList]``,
``reset_siammot_status()``, ``flush_memory(cache)``, ``track_memory``, sub-modules ``backbone``
(``body`` / ``fpn``), ``rpn``, ``roi_heads`` (``box`` / ``track`` / ``solver``), the reference's
state-dict keys, and the ``SIAMESE_TRACKER`` plugin registry.  All arithmetic runs in libsmot.so
through :class:`siammot_b200.engine.Engine`; this file is host control flow only
(CombinedROIHeads.forward roi_heads.py:21-51, TrackSolver.forward track_solver.py:36-108,
TrackHead.get_track_memory track_head.py:54-110), restructured so that a frame costs one
device->host copy.
"""
import time

import numpy as np
import torch
from torch import nn

from .. import ops
from ..engine import Engine, cell_anchors
from ..structures import BoxList
from ..synthetic import backbone_channels, body_layout, make_state_dict
from . import registry
from .track_utils import build_track_utils


# ----------------------------------------------------------------------------------------------
# parameter containers (reference module tree / state-dict keys, SURVEY.md Appendix B)
# ----------------------------------------------------------------------------------------------
class _Holder(nn.Module):
    """Plain container: parameters and buffers only, no forward."""


def _attach(root, key, tensor, as_buffer):
    parts = key.split(".")
    mod = root
    for p in parts[:-1]:
        if p not in mod._modules:
            mod.add_module(p, _Holder())
        mod = mod._modules[p]
    if as_buffer:
        mod.register_buffer(parts[-1], tensor)
    else:
        mod.register_parameter(parts[-1], nn.Parameter(tensor, requires_grad=False))


def _is_frozen_bn_key(key, bn_names):
    return key.rsplit(".", 1)[0] in bn_names


class Memory(object):
    """Track memory for the next frame: N = active tracks (first) + dormant tracks.
    Host-side arrays are numpy fp32 / int64 (same IEEE arithmetic as the reference's torch ops)."""

    def __init__(self, feat, sr, boxes, ids, labels, n_active, device, frame_size=None, pad_pixels=0):
        self.frame_size = frame_size      # (W, H) of the network input the boxes live in: makes the object read as the reference's tuple
        self.pad_pixels = pad_pixels
        self.feat = feat                  # device (N,T,T,C) activation dtype
        self.sr = sr                      # np (N,4) fp32, padded frame
        self.boxes = boxes                # np (N,4) fp32
        self.ids = ids                    # np int64 (N,)
        self.labels = labels              # np int64 (N,)
        self.n_active = n_active
        self.n = int(boxes.shape[0])
        self.device = device

    def stage(self, tp):
        """Write sr | boxes | labels | active into the plan's pinned input block."""
        n = self.n
        h = tp.inputs_host.numpy()
        h[0:4 * n] = self.sr.reshape(-1)
        h[4 * n:8 * n] = self.boxes.reshape(-1)
        h[8 * n:9 * n].view(np.int32)[:] = self.labels
        h[9 * n:9 * n + self.n_active] = 1.0
        h[9 * n + self.n_active:10 * n] = 0.0

    # ``model.track_memory`` read the reference way -- ``feats, sr, boxes = model.track_memory`` / ``model.track_memory[0]`` --
    # yields TrackHead.get_track_memory's tuple (track_head.py:54-110), built on demand
    def __len__(self):
        return 3

    def __getitem__(self, i):
        if self.frame_size is None:
            raise TypeError("this Memory does not know its frame size: use as_reference_tuple(image_size, pad_pixels)")
        return self.as_reference_tuple(self.frame_size, self.pad_pixels)[i]

    def __iter__(self):
        if self.frame_size is None:
            raise TypeError("this Memory does not know its frame size: use as_reference_tuple(image_size, pad_pixels)")
        return iter(self.as_reference_tuple(self.frame_size, self.pad_pixels))

    def as_reference_tuple(self, image_size, pad_pixels):
        """The same memory in the reference's form -- (template_features (N,C,T,T), [sr BoxList], [boxes BoxList with ids /
        labels]) as TrackHead.get_track_memory returns it (track_head.py:54-110) -- for callers that inspect or store
        ``model.track_memory`` the reference way; ``flush_memory`` accepts it back."""
        W, H = image_size
        feats = self.feat.permute(0, 3, 1, 2) if self.feat is not None else torch.zeros((0,))
        sr = BoxList(torch.from_numpy(self.sr.copy()), (int(W + 2 * pad_pixels), int(H + 2 * pad_pixels)), "xyxy")
        boxes = BoxList(torch.from_numpy(self.boxes.copy()), (W, H), "xyxy")
        boxes.add_field("ids", torch.from_numpy(self.ids.copy()))
        boxes.add_field("labels", torch.from_numpy(self.labels.copy()))
        return feats, [sr], [boxes]

    # views used by the generic (plugin / given-detection) path
    def torch_views(self):
        dev = self.device
        return (torch.from_numpy(self.sr).to(dev), torch.from_numpy(self.boxes).to(dev),
                torch.from_numpy(self.labels.astype(np.int32)).to(dev))


class FeaturesView(object):
    """The ``features`` argument of the tracker plugin contract (track_core.py:28,81-98: a tuple of NCHW feature maps, P2..P6)
    over the engine's per-frame plan: ``features[i]`` is a zero-copy NCHW view (``permute`` of the plan's NHWC buffer, in the
    engine's storage dtype) created on first access, ``len(features)`` the number of FPN levels; ``features.plan`` is the plan
    itself, which the built-in EMM uses to run its fused kernels.  A tracker written against the reference -- pooling
    ``features`` with its own ops -- therefore runs unchanged; only the maps' dtype (fp16 when DTYPE is float16) differs."""

    def __init__(self, plan):
        self.plan = plan
        self._views = {}

    def __len__(self):
        return len(self.plan.feats)

    def __getitem__(self, i):
        if isinstance(i, slice):
            return tuple(self[j] for j in range(*i.indices(len(self))))
        if i < 0:
            i += len(self)
        v = self._views.get(i)
        if v is None:
            v = self._views[i] = self.plan.feats[i].permute(0, 3, 1, 2)
        return v

    def __iter__(self):
        return (self[i] for i in range(len(self)))


def _plan_of(features):
    return features.plan if isinstance(features, FeaturesView) else features


@registry.SIAMESE_TRACKER.register("EMM")
class EMM(nn.Module):
    """The Explicit Motion Model tracker (track_core.py:14-98) on the engine.  ``SiamMOT.forward`` runs it
    through the engine's fused per-N launch plan; ``forward`` / ``extract_cache`` keep the reference's
    plugin contract for callers that drive the tracker themselves."""

    def __init__(self, cfg, track_utils):
        super().__init__()
        self.cfg = cfg
        self.track_utils = track_utils
        self.predictor = _Holder()
        self.engine = None  # set by SiamMOT

    def forward(self, features, boxes, sr, targets=None, template_features=None):
        """Reference contract: ({}, [BoxList], {}) with clipped, non-empty track boxes.
        ``features``: a FeaturesView (NCHW maps + the engine plan) or the plan itself."""
        dev = self.engine.device
        b, s = boxes[0], sr[0]
        if template_features.dim() == 4 and template_features.shape[1] == self.engine.C and template_features.shape[3] != self.engine.C:
            template_features = template_features.permute(0, 2, 3, 1).contiguous()     # the reference's NCHW templates
        tb, conf, valid = self.engine.emm_track(_plan_of(features), template_features, s.bbox.to(dev).contiguous(),
                                                b.bbox.to(dev).contiguous())
        keep = valid.bool()
        out = BoxList(tb[keep], b.size, mode="xyxy")
        out.add_field("ids", b.get_field("ids").to(dev)[keep])
        out.add_field("labels", b.get_field("labels").to(dev)[keep])
        out.add_field("scores", conf[keep])
        return {}, [out], {}

    def extract_cache(self, features, detection):
        dev = self.engine.device
        x = self.engine.templates(_plan_of(features), detection.bbox.to(dev).contiguous())
        sr = self.track_utils.extend_bbox(self.track_utils.update_boxes_in_pad_images([detection.to("cpu")]))
        return x, sr, [detection]


class TrackHead(nn.Module):
    def __init__(self, tracker, sampler, track_utils, track_pool):
        super().__init__()
        self.tracker = tracker
        self.sampler = sampler
        self.track_utils = track_utils
        self.track_pool = track_pool

    def reset_track_pool(self):
        self.track_pool.reset()


class TrackSolver(nn.Module):
    def __init__(self, track_pool, track_thresh=0.3, start_track_thresh=0.5, resume_track_thresh=0.4):
        super().__init__()
        self.track_pool = track_pool
        self.track_thresh = track_thresh
        self.start_thresh = start_track_thresh
        self.resume_track_thresh = resume_track_thresh

    def resolve(self, scores_adj, ids, all_track_ids):
        """Host half of TrackSolver.forward (track_solver.py:71-106) on the NMS survivors (numpy, NMS order).
        scores_adj still carries the +1 (dormant / refined) and +2 (active) offsets.  Returns the folded
        scores and the final ids; updates the pool exactly like the reference."""
        pool = self.track_pool
        _scores = scores_adj.astype(np.float32, copy=True)
        m = _scores >= np.float32(2.)
        _scores[m] = _scores[m] - np.float32(2.)
        m = _scores >= np.float32(1.)
        _scores[m] = _scores[m] - np.float32(1.)
        _ids = ids.astype(np.int64, copy=True)
        start_idxs = np.nonzero((_ids < 0) & (_scores >= np.float32(self.start_thresh)))[0]
        inactive_idxs = (_ids >= 0) & (_scores < np.float32(self.track_thresh))
        nms_track_ids = set(_ids[_ids >= 0].tolist())
        nms_removed_ids = all_track_ids - nms_track_ids
        inactive_ids = set(_ids[inactive_idxs].tolist()) | nms_removed_ids
        dormant_ids = pool.get_dormant_ids()
        if dormant_ids:
            dormant_mask = np.fromiter((x in dormant_ids for x in _ids.tolist()), dtype=bool, count=_ids.shape[0])
            for _id in _ids[dormant_mask & (_scores >= np.float32(self.resume_track_thresh))].tolist():
                pool.resume_track(_id)
        for _idx in start_idxs.tolist():
            _ids[_idx] = pool.start_track()
        active_ids = pool.get_active_ids()
        for _id in inactive_ids:
            if _id in active_ids:
                pool.suspend_track(_id)
        _ids[inactive_idxs] = -1
        pool.expire_tracks()
        pool.increment_frame()
        return _scores, _ids


class CombinedROIHeads(nn.ModuleDict):
    def __init__(self, cfg, heads):
        super().__init__(heads)
        self.cfg = cfg
        self.engine = None
        self._out_host = None
        self.results_on_host = False   # True: forward returns CPU BoxLists (what demo / inferencer convert to anyway)

    def reset_roi_status(self):
        if self.cfg.MODEL.TRACK_ON:
            self.track.reset_track_pool()

    # -- detections from externally provided boxes (roi_heads.py:26-34): box head + per-class NMS, eager
    def _given_detections(self, P, given):
        eng, dev, cfg = self.engine, self.engine.device, self.cfg
        ncls = eng.ncls
        rois = given.convert("xyxy").bbox.to(dev, torch.float32).contiguous()
        n = rois.shape[0]
        # persistent buffers per capacity class (power of two): one arena / plan per class, not per detection count
        det_boxes, det_scores, det_block = eng.given_buffers(P, n * (ncls - 1))
        det_scores.fill_(-1.0)
        det_block.zero_()
        if n:
            dec_b, dec_s = eng.box_head_eager(P, rois)
            H = cfg.MODEL.ROI_HEADS
            for j in range(1, ncls):
                ops.sort_nms(dec_b[:, j], dec_s[:, j], det_block[0:1], n_max=n, min_score=H.SCORE_THRESH, thresh=H.NMS,
                             max_keep=n, tag=j, out_boxes=det_boxes, out_scores=det_scores, out_tag=det_block[1:],
                             workspace=eng.nms_workspace(n), box_stride=4 * ncls, score_stride=ncls)
        return det_boxes, det_scores, det_block

    def run_frame(self, P, mem, given_detection=None):
        """One frame after the static stage (CombinedROIHeads.forward roi_heads.py:21-51).
        Returns (BoxList on the model device, Memory for the next frame)."""
        return self.finish_frame(self.launch_frame(P, mem, given_detection))

    def launch_frame(self, P, mem, given_detection=None):
        """Enqueue the track-dependent stage of a frame (no host wait).  Returns a pending-frame token."""
        eng, cfg = self.engine, self.cfg
        if not cfg.MODEL.TRACK_ON:
            return self._launch_detections_only(P, given_detection)
        pool = self.track.track_pool
        if mem is None:
            pool.reset()                                                  # track_head.py:39-40
        n = mem.n if (mem is not None and mem.feat is not None and mem.feat.numel() > 0) else 0
        if given_detection is None:
            tp = eng.track_plan(P, n)
        else:
            # external detections replace the RPN/box-head ones: a one-off plan bound to their arrays
            tp = eng.track_plan(P, n, det=self._given_detections(P, given_detection[0]))
        if n and tp.staged_mem is not mem:      # normally staged by the previous frame's finish; a flushed-in memory is staged here
            mem.stage(tp)
            tp.staged_mem = mem
        tp.run(mem.feat if n else None, wait=False)
        return (P, tp, mem, n)

    # -- MODEL.TRACK_ON False: the model is the detector alone (roi_heads.py:36 skips track head and solver; rcnn.py:57-61)
    def _launch_detections_only(self, P, given_detection):
        eng = self.engine
        det_boxes, det_scores, det_block = (self._given_detections(P, given_detection[0]) if given_detection is not None
                                            else (P.det_boxes, P.det_scores, P.det_block))
        cap = det_boxes.shape[0]
        host = getattr(P, "det_host", None)
        if host is None or host.numel() < 6 * cap + 1:
            host = P.det_host = torch.zeros((6 * cap + 1,), dtype=torch.float32).pin_memory()
            P.det_done = torch.cuda.Event()
        host[0:4 * cap].view(cap, 4).copy_(det_boxes, non_blocking=True)
        host[4 * cap:5 * cap].copy_(det_scores, non_blocking=True)
        host[5 * cap:6 * cap + 1].view(torch.int32).copy_(det_block, non_blocking=True)
        P.det_done.record()
        return (P, None, cap, (det_boxes, det_scores, det_block))     # the arrays stay alive until the copies have run

    def _finish_detections_only(self, pending):
        P, _, cap, _keep = pending
        P.det_done.synchronize()
        h = P.det_host.numpy()
        blk = h[5 * cap:6 * cap + 1].view(np.int32)
        k = int(blk[0])
        boxes = np.array(h[0:4 * cap].reshape(cap, 4)[:k], dtype=np.float32, copy=True)
        scores = np.array(h[4 * cap:4 * cap + k], dtype=np.float32, copy=True)
        labels = blk[1:1 + k].astype(np.int64)
        ids = np.full((k,), -1, dtype=np.int64)                         # inference.py:90: detections carry id -1
        return self._to_boxlist(boxes, scores, ids, labels, (P.W, P.H)), None

    # -- MODEL.TRACK_ON False over a (B,3,H,W) batch (rcnn.py:46-51 with roi_heads.py:25; inferencer.py:60 with CLIP_LEN > 1)
    def detections_batch(self, P):
        """B BoxLists, in image order, from the result blocks of batch plan P (enqueued on the current stream): one packed
        device-to-host copy and one host wait for the whole batch."""
        B, cap = P.det_scores.shape
        host = getattr(P, "det_host", None)
        if host is None:
            host = P.det_host = torch.zeros((P.det_packed.numel(),), dtype=torch.float32).pin_memory()
            P.det_done = torch.cuda.Event()
        host.copy_(P.det_packed, non_blocking=True)
        P.det_done.record()
        P.det_done.synchronize()
        h = host.numpy()
        boxes = h[:B * cap * 4].reshape(B, cap, 4)
        scores = h[B * cap * 4:B * cap * 5].reshape(B, cap)
        blk = h[B * cap * 5:].view(np.int32).reshape(B, 1 + cap)
        items = []
        for b in range(B):
            k = int(blk[b, 0])
            items.append((np.array(boxes[b, :k], dtype=np.float32, copy=True), np.array(scores[b, :k], dtype=np.float32, copy=True),
                          np.full((k,), -1, dtype=np.int64), blk[b, 1:1 + k].astype(np.int64)))   # inference.py:90: ids -1
        return self._to_boxlists(items, (P.W, P.H), P)

    def _to_boxlists(self, items, size, P):
        """_to_boxlist for a batch: with results on the device, ONE packed pinned block and one host-to-device copy for all
        images (the BoxList fields are views of it); the block is per plan and reused once its previous copy has completed."""
        if self.results_on_host:
            return [self._to_boxlist(bx, sc, ids, lab, size) for bx, sc, ids, lab in items]
        ks = [bx.shape[0] for bx, _, _, _ in items]
        spans = [(36 * k + 7) & ~7 for k in ks]   # each image's fields start 8-byte aligned (int64 views)
        nbytes = sum(spans)
        stage = getattr(P, "out_stage", None)
        if stage is not None:
            stage[1].synchronize()
        if stage is None or stage[0].numel() < nbytes:
            stage = P.out_stage = [torch.zeros((max(nbytes, 36 * 256),), dtype=torch.uint8).pin_memory(), torch.cuda.Event()]
        h = stage[0].numpy()
        offs, o = [], 0
        for (bx, sc, ids, lab), k, span in zip(items, ks, spans):
            h[o:o + 8 * k].view(np.int64)[:] = ids
            h[o + 8 * k:o + 16 * k].view(np.int64)[:] = lab
            h[o + 16 * k:o + 32 * k].view(np.float32)[:] = bx.reshape(-1)
            h[o + 32 * k:o + 36 * k].view(np.float32)[:] = sc
            offs.append(o)
            o += span
        d = torch.empty((max(nbytes, 8),), dtype=torch.uint8, device=self.engine.device)
        d[:nbytes].copy_(stage[0][:nbytes], non_blocking=True)
        stage[1].record()
        out = []
        for o, k in zip(offs, ks):
            r = BoxList(d[o + 16 * k:o + 32 * k].view(torch.float32).view(k, 4), size, mode="xyxy")
            r.add_field("scores", d[o + 32 * k:o + 36 * k].view(torch.float32))
            r.add_field("ids", d[o:o + 8 * k].view(torch.int64))
            r.add_field("labels", d[o + 8 * k:o + 16 * k].view(torch.int64))
            out.append(r)
        return out

    def finish_frame(self, pending, next_P=None, defer=None):
        """Wait for the frame's result block, resolve ids on the host, build the next-frame memory.
        next_P: the static plan the NEXT frame will run on (clip pipelining); defaults to this frame's.
        defer: a list -> the host work nothing downstream waits for (the result BoxList, the per-id cache update) is appended
        to it as a callable returning the BoxList instead of being done here; the clip pipelines run it right after the NEXT
        frame's track stage has been enqueued, i.e. under that stage instead of in front of it."""
        if pending[1] is None:
            return self._finish_detections_only(pending)
        P, tp, mem, n = pending
        ht = self.engine.host_timers
        t0 = time.perf_counter() if ht is not None else 0.0
        tp.wait()
        t1 = time.perf_counter() if ht is not None else 0.0
        # ---- host: unpack the result block
        total, ncap = tp.total, tp.ncap
        t = max(total, 1)
        hf = tp.host_res.numpy()
        hi = hf.view(np.int32)
        k = int(hi[4 * t])
        keep = hi[4 * t + 1:4 * t + 1 + k]
        kboxes = hf[0:4 * t].reshape(t, 4)[:k]
        kscores = hf[5 * t + 1:5 * t + 1 + k]
        det_labels = tp.host_det.numpy()[1:1 + ncap]
        is_trk = keep >= ncap
        ids = np.full((k,), -1, dtype=np.int64)
        labels = np.zeros((k,), dtype=np.int64)
        labels[~is_trk] = det_labels[keep[~is_trk]]
        all_track_ids = set()
        if n:
            if tp.grouped:
                # several foreground classes: candidate position g holds memory row perm[g] (class-grouped order of the
                # reference's box head, inference.py:145-191); -1 marks the unused tail
                perm = hi[7 * t + 1:7 * t + 1 + n]
                valid_rows = perm[perm >= 0]
                any_valid = valid_rows.size > 0
                rows = perm[keep[is_trk] - ncap]
            else:
                trk_valid = hf[6 * t + 1 + ncap:6 * t + 1 + total] > -0.5
                any_valid = trk_valid.any()
                valid_rows = trk_valid
                rows = keep[is_trk] - ncap
            if not any_valid:
                # roi_heads.py:64-65 returns a bare BoxList here and :44 then evaluates list + BoxList
                raise TypeError("can only concatenate list (not \"BoxList\") to list")
            all_track_ids = set(mem.ids[valid_rows].tolist())
            ids[is_trk] = mem.ids[rows]
            labels[is_trk] = mem.labels[rows]
        if k == 0:                                                        # track_solver.py:51-52 (early return)
            scores = np.zeros((0,), dtype=np.float32)
        else:
            scores, ids = self.solver.resolve(kscores, ids, all_track_ids)
        boxes = np.array(kboxes, dtype=np.float32, copy=True)
        t2 = time.perf_counter() if ht is not None else 0.0
        late = [] if defer is not None else None
        with self.engine.timed("next_memory"):
            new_mem = self._build_memory(P, boxes, ids, labels, next_P, late)
        t3 = time.perf_counter() if ht is not None else 0.0
        size = (P.W, P.H)
        if defer is not None:
            def finish_late():
                tl = time.perf_counter() if ht is not None else 0.0
                for fn in late:
                    fn()
                res = self._to_boxlist(boxes, scores, ids, labels, size)
                if ht is not None:
                    ht["deferred"] = ht.get("deferred", 0.0) + time.perf_counter() - tl
                return res
            defer.append(finish_late)
            out = None
        else:
            out = self._to_boxlist(boxes, scores, ids, labels, size)
        if ht is not None:   # where the sequential part of a video goes (bench.py stage_ms): wait = the track stage as the host sees it
            t4 = time.perf_counter()
            for k, v in (("track_wait", t1 - t0), ("solver", t2 - t1), ("next_memory", t3 - t2), ("boxlist", t4 - t3)):
                ht[k] = ht.get(k, 0.0) + v
            ht["frames"] = ht.get("frames", 0) + 1
        return out, new_mem

    def _to_boxlist(self, boxes, scores, ids, labels, size):
        """One packed pinned buffer -> one H2D copy; the BoxList fields are views of the device copy.
        With ``results_on_host`` (SURVEY 8 (f) rank 2: result egress) the BoxList is built from the host arrays the solver
        just produced -- no H2D here and no D2H + sync in the caller's ``.to('cpu')`` (inferencer.py:65-67)."""
        dev = self.engine.device
        k = boxes.shape[0]
        if self.results_on_host:
            # copies: the inputs may be views of the pinned result block, which the next frame overwrites
            out = BoxList(torch.from_numpy(np.array(boxes, dtype=np.float32, copy=True).reshape(k, 4)), size, mode="xyxy")
            out.add_field("scores", torch.from_numpy(np.array(scores, dtype=np.float32, copy=True)))
            out.add_field("ids", torch.from_numpy(np.array(ids, dtype=np.int64, copy=True)))
            out.add_field("labels", torch.from_numpy(np.array(labels, dtype=np.int64, copy=True)))
            return out
        nbytes = 36 * k
        # pinned staging ring: the H2D copy below is asynchronous and (in the clip pipelines) enqueued behind the next frame's
        # track stage, so a staging block is reused only once the copy that read it has completed (event per block)
        if self._out_host is None:
            self._out_host = [[None, None] for _ in range(3)]
            self._out_next = 0
        slot = self._out_host[self._out_next]
        self._out_next = (self._out_next + 1) % len(self._out_host)
        if slot[1] is not None:
            slot[1].synchronize()
        if slot[0] is None or slot[0].numel() < nbytes:
            slot[0] = torch.zeros((max(nbytes, 36 * 256),), dtype=torch.uint8).pin_memory()
        out_host = slot[0]
        h = out_host.numpy()
        h[0:8 * k].view(np.int64)[:] = ids
        h[8 * k:16 * k].view(np.int64)[:] = labels
        h[16 * k:32 * k].view(np.float32)[:] = boxes.reshape(-1)
        h[32 * k:36 * k].view(np.float32)[:] = scores
        d = torch.empty((max(nbytes, 8),), dtype=torch.uint8, device=dev)
        d[:nbytes].copy_(out_host[:nbytes], non_blocking=True)
        if slot[1] is None:
            slot[1] = torch.cuda.Event()
        slot[1].record()
        out = BoxList(d[16 * k:32 * k].view(torch.float32).view(k, 4), size, mode="xyxy")
        out.add_field("scores", d[32 * k:36 * k].view(torch.float32))
        out.add_field("ids", d[0:8 * k].view(torch.int64))
        out.add_field("labels", d[8 * k:16 * k].view(torch.int64))
        return out

    def _build_memory(self, P, boxes, ids, labels, next_P=None, late=None):
        """TrackHead.get_track_memory (track_head.py:54-110) + EMM.extract_cache (track_core.py:81-98).
        boxes/ids/labels: numpy, solver output order.  late: list -> the per-id cache update (needed by the NEXT frame's
        memory construction, not by its track stage) is appended to it instead of being done here."""
        eng, dev = self.engine, self.engine.device
        ht = eng.host_timers
        ta = time.perf_counter() if ht is not None else 0.0
        pool = self.track.track_pool
        tu = self.track.track_utils
        active_ids = pool.get_active_ids()
        ids_l = ids.tolist()
        sel = np.array([i in active_ids for i in ids_l], dtype=bool)
        a_boxes, a_ids, a_labels = boxes[sel], ids[sel], labels[sel]
        n_act = int(a_ids.shape[0])
        cache = pool.get_cache()
        dormant = [cache[i] for i in pool.get_dormant_ids() if i in cache] if cache else []
        n = n_act + len(dormant)
        m_boxes = np.empty((n, 4), dtype=np.float32)
        m_sr = np.empty((n, 4), dtype=np.float32)
        m_ids = np.empty((n,), dtype=np.int64)
        m_labels = np.empty((n,), dtype=np.int64)
        m_boxes[:n_act], m_ids[:n_act], m_labels[:n_act] = a_boxes, a_ids, a_labels
        if n_act:
            m_sr[:n_act] = tu.search_region_np(a_boxes)
        for j, d in enumerate(dormant):
            r = n_act + j
            m_boxes[r], m_sr[r], m_ids[r], m_labels[r] = d[3][d[1]], d[2][d[1]], d[4], d[5]
        if n == 0:
            return Memory(None, m_sr, m_boxes, m_ids, m_labels, 0, dev, (P.W, P.H), tu.pad_pixels)
        # next frame's plan: stage its inputs now (the boxes are needed on the device anyway)
        tb = time.perf_counter() if ht is not None else 0.0
        tp = eng.track_plan(next_P if next_P is not None else P, n)
        tc = time.perf_counter() if ht is not None else 0.0
        mem = Memory(None, m_sr, m_boxes, m_ids, m_labels, n_act, dev, (P.W, P.H), tu.pad_pixels)
        mem.stage(tp)
        tp.staged_mem = mem
        tp.inputs.copy_(tp.inputs_host, non_blocking=True)
        td = time.perf_counter() if ht is not None else 0.0
        feat = torch.empty((n, eng.t_res, eng.t_res, eng.C), dtype=eng.dtype, device=dev)
        te = time.perf_counter() if ht is not None else 0.0
        if n_act:
            eng.templates_into(P, tp, n_act, feat)
        if dormant:
            eng.gather_templates(feat, n_act, [(d[0], d[1]) for d in dormant])
        mem.feat = feat
        if ht is not None:
            tf = time.perf_counter()
            for k, v in (("mem_numpy", tb - ta), ("mem_track_plan", tc - tb), ("mem_stage_h2d", td - tc), ("mem_alloc", te - td),
                         ("mem_templates", tf - te)):
                ht[k] = ht.get(k, 0.0) + v

        def update_cache():
            # per id: (template tensor, row, search regions, boxes, id, label) -- the arrays of this memory are never written
            # again, so the rows are read from them when a dormant track is revived instead of being copied out for every track
            ids_py, labels_py = m_ids.tolist(), m_labels.tolist()
            pool.update_cache({i: (feat, r, m_sr, m_boxes, i, labels_py[r]) for r, i in enumerate(ids_py)})
        if late is None:
            update_cache()
        else:
            late.append(update_cache)
        return mem


class SiamMOT(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        # ---- parameter tree with the reference's names; values: seeded synthetic init (no checkpoints offline)
        bn_names = set("backbone.body." + n for kind, n, _ in body_layout(cfg) if kind == "bn")
        self.backbone = _Holder()
        self.backbone.out_channels = backbone_channels(cfg)[1]
        self.rpn = _Holder()
        heads = [("box", _Holder())]
        if cfg.MODEL.TRACK_ON:                        # build_roi_heads (roi_heads.py:87-100): track head + solver only when tracking
            track_utils, track_pool = build_track_utils(cfg)
            tracker = registry.SIAMESE_TRACKER[cfg.MODEL.TRACK_HEAD.MODEL](cfg, track_utils)
            if not isinstance(tracker, EMM):
                # SiamMOT.forward runs the track head as ONE fused launch list built around the EMM (engine._TrackPlan); a
                # tracker registered by someone else can be constructed and driven through its own forward / extract_cache
                # on FeaturesView(plan) (NCHW maps, the reference's contract), but it is not what forward() would execute:
                # refuse loudly instead of silently tracking with the EMM
                raise NotImplementedError("MODEL.TRACK_HEAD.MODEL = %r: SiamMOT.forward executes the built-in EMM track stage; drive "
                                          "a third-party SIAMESE_TRACKER through tracker.forward(FeaturesView(plan), ...) yourself"
                                          % cfg.MODEL.TRACK_HEAD.MODEL)
            sampler = registry.TRACKER_SAMPLER.get(cfg.MODEL.TRACK_HEAD.MODEL, lambda c, t: None)(cfg, track_utils)
            T = cfg.MODEL.TRACK_HEAD
            heads += [("track", TrackHead(tracker, sampler, track_utils, track_pool)),
                      ("solver", TrackSolver(track_pool, T.TRACK_THRESH, T.START_TRACK_THRESH, T.RESUME_TRACK_THRESH))]
        self.roi_heads = CombinedROIHeads(cfg, heads)
        for key, val in make_state_dict(cfg, seed=0).items():
            if not cfg.MODEL.TRACK_ON and key.startswith("roi_heads.track."):
                continue
            _attach(self, key, val, as_buffer=_is_frozen_bn_key(key, bn_names))
        R = cfg.MODEL.RPN
        for i, (st, sz) in enumerate(zip(R.ANCHOR_STRIDE, R.ANCHOR_SIZES)):
            _attach(self, "rpn.anchor_generator.cell_anchors.%d" % i, cell_anchors(st, (sz,), R.ASPECT_RATIOS), True)
        self.track_memory = None
        self._mem = None
        self._engine = None
        self._engine_stale = True
        self.eval()

    # ---- engine management
    def engine(self):
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("siammot_b200 runs on CUDA only (model is on %s): call .to('cuda'); there is no CPU path" % dev)
        if self._engine is None or self._engine.device != dev:
            self._engine = Engine(self.cfg, device=dev)
            self._engine_stale = True
        if self._engine_stale:
            self._engine.load_state_dict(self.state_dict())
            self._engine_stale = False
        self.roi_heads.engine = self._engine
        if self.cfg.MODEL.TRACK_ON:
            self.roi_heads.track.tracker.engine = self._engine
        return self._engine

    def load_state_dict(self, state_dict, strict=True):
        sd = {(k[7:] if k.startswith("module.") else k): v for k, v in state_dict.items()}
        r = super().load_state_dict(sd, strict=strict)
        self._engine_stale = True
        return r

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        self._engine_stale = True
        return r

    @property
    def results_on_host(self):
        """True: forward / forward_clip return CPU BoxLists built straight from the solver's host arrays (the reference's
        callers move every result to the CPU anyway: demo_inference.py:107, inferencer.py:65).  Default False = the
        reference contract (BoxList on the model's device)."""
        return self.roi_heads.results_on_host

    @results_on_host.setter
    def results_on_host(self, v):
        self.roi_heads.results_on_host = bool(v)

    # ---- reference API
    def flush_memory(self, cache=None):
        self.track_memory = cache
        self._mem = cache if (cache is None or isinstance(cache, Memory)) else self._memory_from_tuple(cache)

    def reset_siammot_status(self):
        self.flush_memory()
        self.roi_heads.reset_roi_status()

    def _memory_from_tuple(self, cache):
        """Accept the reference's (template_features, [sr BoxList], [boxes BoxList]) memory tuple."""
        feats, sr, boxes = cache
        b = boxes[0].to("cpu")
        ids = b.get_field("ids").to(torch.int64).numpy()
        active = self.roi_heads.track.track_pool.get_active_ids()
        n_act = sum(1 for i in ids.tolist() if i in active)
        eng = self.engine()
        dev = eng.device
        if feats.numel():
            T, Cc = eng.t_res, eng.C
            if feats.dim() == 4 and tuple(feats.shape[1:]) == (Cc, T, T) and Cc != T:
                feats = feats.permute(0, 2, 3, 1)            # the reference's NCHW templates (track_core.py:92) -> NHWC
            elif feats.dim() != 4 or tuple(feats.shape[1:]) != (T, T, Cc):
                raise ValueError("template features must be (N, %d, %d, %d) [reference layout] or (N, %d, %d, %d) [engine layout], got %s"
                                 % (Cc, T, T, T, T, Cc, tuple(feats.shape)))
            if feats.shape[0] != b.bbox.shape[0]:
                raise ValueError("%d template features for %d boxes" % (feats.shape[0], b.bbox.shape[0]))
            feats = feats.to(device=dev, dtype=eng.dtype).contiguous()
        else:
            feats = None
        return Memory(feats, sr[0].bbox.to("cpu").float().numpy(), b.bbox.float().numpy(),
                      ids, b.get_field("labels").to(torch.int64).numpy(), n_act, dev, tuple(b.size),
                      self.roi_heads.track.track_utils.pad_pixels)

    @torch.no_grad()
    def forward(self, images, targets=None, given_detection=None):
        if self.training:
            raise NotImplementedError("siammot_b200 is an inference engine: call .eval() (training is out of scope)")
        eng = self.engine()
        sizes = getattr(images, "image_sizes", None)
        if hasattr(images, "tensors"):
            images = images.tensors
        if torch.is_tensor(images) and images.dim() == 4 and images.shape[0] > 1 and images.dtype != torch.uint8:
            return self._forward_batch(eng, images, sizes, given_detection)
        mem_in = self._mem
        overlap = (eng.frame_overlap and given_detection is None and self.cfg.MODEL.TRACK_ON and mem_in is not None
                   and mem_in.feat is not None and mem_in.feat.numel() > 0)
        part = 0 if overlap else None
        if _is_raw_frame(images):
            # decoded RGB uint8 HWC frame: the test transform (demo_inference.py:74-82) runs on the device; boxes come
            # back in resized-frame pixels exactly as if the caller had applied the transform (demo_inference.py:108)
            P = eng.run_static_raw(images, part=part)
        else:
            P = eng.run_static(images, part=part)
        if overlap:
            result, mem = self._forward_overlapped(eng, P, mem_in)
        else:
            result, mem = self.roi_heads.run_frame(P, mem_in, given_detection)
        self._mem = mem
        self.track_memory = mem
        return [result]


def _forward_batch(self, eng, images, sizes, given_detection):
    """A (B,3,H,W) batch, B >= 2, through a detector-only model: Engine.batch_plan runs the frame-independent stage of all B
    images as one launch list; returns B BoxLists in image order, each equal to model(images[i:i+1])[0]."""
    B, _, H, W = images.shape
    if self.cfg.MODEL.TRACK_ON:
        raise ValueError("a tracking model (MODEL.TRACK_ON True) takes one image per forward, as the reference's EMM asserts "
                         "(track_core.py:75); got a batch of %d" % B)
    if given_detection is not None:
        raise ValueError("given_detection is supported for one image per forward only; got a batch of %d images" % B)
    if sizes is not None and any(tuple(int(v) for v in sz) != (H, W) for sz in sizes):
        raise ValueError("padded ImageList: image_sizes %s differ from the batch tensor's %dx%d; a batch must hold images of one "
                         "size" % ([tuple(int(v) for v in sz) for sz in sizes], H, W))
    P = eng.run_batch(images)
    result = self.roi_heads.detections_batch(P)
    self._mem = None
    self.track_memory = None
    return result


SiamMOT._forward_batch = _forward_batch


def _forward_overlapped(self, eng, P, mem):
    """Per-frame latency mode (developer switch SMOT_FRAME_OVERLAP=1).  The track stage needs the frame's detections only for its
    last two steps (candidate assembly, solver NMS); everything before -- search-region pooling, correlation, EMM heads, decode,
    box-head refinement -- needs the feature maps and the memory.  So once the backbone half is enqueued on the caller's stream,
    the detection tail goes to a second stream and runs under that EMM half; the caller's stream waits for it just before the
    candidate assembly.  B + max(D, T_emm) + T_tail instead of B + D + T; results identical."""
    cur = torch.cuda.current_stream(eng.device)
    sD = eng.tail_stream()
    if P.backbone_done is None:
        P.backbone_done = torch.cuda.Event()
    P.backbone_done.record(cur)
    with torch.cuda.stream(sD):
        sD.wait_event(P.backbone_done)
        eng.run_tail(P)
        if P.static_done is None:
            P.static_done = torch.cuda.Event()
        P.static_done.record(sD)
    heads = self.roi_heads
    tp = eng.track_plan(P, mem.n)
    if tp.staged_mem is not mem:
        mem.stage(tp)
        tp.staged_mem = mem
    tp.run_split(mem.feat, between=lambda: cur.wait_event(P.static_done))
    return heads.finish_frame((P, tp, mem, mem.n))


SiamMOT._forward_overlapped = _forward_overlapped


def _is_raw_frame(x):
    return (isinstance(x, np.ndarray) and x.dtype == np.uint8) or (torch.is_tensor(x) and x.dtype == torch.uint8)


def _forward_clip(self, frames, before_frame=None, given_detections=None):
    """Process consecutive frames of ONE video as a two-stage pipeline: the frame-independent stage (backbone ..
    detections, double-buffered static plans) of frame t+1 runs on a side stream while the track stage of frame t
    runs on the current stream and the host resolves ids.  Results are identical to calling the model frame by
    frame; this is the throughput API (the reference has INFERENCE.CLIP_LEN but processes one frame per forward,
    defaults.py:96, track_core.py:75).  frames: sequence / tensor of normalised (3,H,W) frames or of decoded
    uint8 (H,W,3) RGB frames (preprocessed on the device).
    before_frame(t): optional hook called right before frame t's tracker stage is enqueued.
    given_detections: optional per-frame list of public detections, each what ``forward(..., given_detection=)`` takes (a
    one-element list holding a BoxList, roi_heads.py:26-34; inferencer.py:47-54), or None for a frame without any."""
    if self.training:
        raise NotImplementedError("siammot_b200 is an inference engine: call .eval()")
    eng = self.engine()
    n_frames = len(frames)
    results = []
    if not n_frames:
        return results
    if given_detections is not None and len(given_detections) != n_frames:
        raise ValueError("given_detections: %d entries for %d frames" % (len(given_detections), n_frames))
    if eng.clip_split:
        return _forward_clip_three_stage(self, eng, frames, before_frame, given_detections)
    cur = torch.cuda.current_stream(eng.device)
    side = eng.side_stream()
    side.wait_stream(cur)          # the frames (and anything else already enqueued) are visible to the side stream
    slot_free = [None, None]       # event: every reader of the slot's buffers (track stage, template pooling) is enqueued-complete

    def static(t):
        with torch.cuda.stream(side):
            if slot_free[t & 1] is not None:
                side.wait_event(slot_free[t & 1])
            P = eng.run_static_raw(frames[t], t & 1) if _is_raw_frame(frames[t]) else eng.run_static(frames[t], t & 1)
            if P.static_done is None:
                P.static_done = torch.cuda.Event()
            P.static_done.record(side)
        return P

    deferred = []
    with torch.no_grad():
        P_next = static(0)
        for t in range(n_frames):
            P = P_next
            if before_frame is not None:
                before_frame(t)
            cur.wait_event(P.static_done)
            pending = self.roi_heads.launch_frame(P, self._mem, given_detections[t] if given_detections is not None else None)
            _run_deferred(deferred, results)       # frame t-1's result object / cache update, under frame t's track stage
            if t + 1 < n_frames:
                P_next = static(t + 1)
            result, mem = self.roi_heads.finish_frame(pending, next_P=P_next, defer=deferred)
            ev = torch.cuda.Event()
            ev.record(cur)
            slot_free[t & 1] = ev
            self.__dict__["_mem"] = self.__dict__["track_memory"] = mem      # (plain attributes: bypass nn.Module.__setattr__)
            results.append(result)
        _run_deferred(deferred, results)
        cur.wait_stream(side)
    return results


def _run_deferred(deferred, results):
    """Run the host work the previous frame put off (CombinedROIHeads.finish_frame(defer=...)): its callable returns the frame's
    BoxList, which replaces the placeholder at the end of ``results``."""
    for fn in deferred:
        results[-1] = fn()
    del deferred[:]


def _forward_clip_three_stage(self, eng, frames, before_frame=None, given_detections=None):
    """forward_clip with the frame-independent stage cut in two (developer switch SMOT_CLIP_SPLIT=1, DESIGN.md section 4):

      stream A   B(t): input copy / test transform, backbone, FPN, RPN heads   -- the kernels that fill the GPU
      stream D   D(t): proposal selection, box head, per-class NMS             -- a serial chain of small kernels
      caller's   T(t): track stage, then the host solver H(t) and the next-frame memory

    Dependencies: D(t) after B(t); T(t) after D(t) and H(t-1); B(t + K) after T(t) and H(t)'s template pooling (slot reuse,
    K = SMOT_CLIP_SLOTS static-plan copies).  So D(t) and T(t) run under B(t+1) (.. B(t+K-1)), and the per-frame period is
    max(B, T + H) instead of B + D.  The three stages use disjoint split-K scratch (conv_ws / conv_ws_det / conv_ws_track)
    and per-slot buffers; every cross-stream edge is an event recorded BEFORE the wait on it is enqueued.
    Results are identical to frame-by-frame calls."""
    n_frames = len(frames)
    if eng.clip_pairs and n_frames >= 2 and eng.pair_ok(frames):
        return _forward_clip_pairs(self, eng, frames, before_frame, given_detections)
    K = eng.clip_slots
    results = []
    cur = torch.cuda.current_stream(eng.device)
    sA, sD = eng.side_stream(), eng.tail_stream()
    sA.wait_stream(cur)            # the frames (and anything else already enqueued) are visible to the worker streams
    sD.wait_stream(cur)
    slot_free = [None] * K         # event: every reader of the slot's buffers (D, T, template pooling) is enqueued-complete
    plans = {}

    def backbone(t):
        s = t % K
        with torch.cuda.stream(sA):
            if slot_free[s] is not None:
                sA.wait_event(slot_free[s])
            P = (eng.run_static_raw(frames[t], s, part=0) if _is_raw_frame(frames[t]) else eng.run_static(frames[t], s, part=0))
            if P.backbone_done is None:
                P.backbone_done = torch.cuda.Event()
            P.backbone_done.record(sA)
        plans[t] = P

    def detect(t):
        P = plans[t]
        with torch.cuda.stream(sD):
            sD.wait_event(P.backbone_done)
            eng.run_tail(P)
            if P.static_done is None:
                P.static_done = torch.cuda.Event()
            P.static_done.record(sD)

    deferred = []
    with torch.no_grad():
        for t in range(min(K - 1, n_frames)):
            backbone(t)
        detect(0)
        for t in range(n_frames):
            P = plans.pop(t)
            if before_frame is not None:
                before_frame(t)
            cur.wait_event(P.static_done)          # D(t) complete (hence B(t))
            pending = self.roi_heads.launch_frame(P, self._mem, given_detections[t] if given_detections is not None else None)
            _run_deferred(deferred, results)       # frame t-1's result object / cache update, under frame t's track stage
            if t + K - 1 < n_frames:
                backbone(t + K - 1)                # slot of frame t-1: its slot_free event was recorded in iteration t-1
            if t + 1 < n_frames:
                detect(t + 1)
            result, mem = self.roi_heads.finish_frame(pending, next_P=plans.get(t + 1), defer=deferred)
            ev = torch.cuda.Event()
            ev.record(cur)
            slot_free[t % K] = ev
            self.__dict__["_mem"] = self.__dict__["track_memory"] = mem      # (plain attributes: bypass nn.Module.__setattr__)
            results.append(result)
        _run_deferred(deferred, results)
        cur.wait_stream(sA)
        cur.wait_stream(sD)
    return results


def _forward_clip_pairs(self, eng, frames, before_frame=None, given_detections=None):
    """The three-stage clip pipeline with the backbone half run over frame PAIRS (Engine.pair_plan: one batch-2 pass for
    frames 2k, 2k+1 -- the layers below level 2 do not fill the GPU's SMs with one frame and cost the same for two).

      stream A   B(2k, 2k+1): input copies / test transform of both frames, ONE batch-2 backbone + FPN + RPN-head pass
      stream D   D(t): proposal selection, box head, per-class NMS of frame t (its image of the batched buffers)
      caller's   T(t): track stage, host solver H(t), next-frame memory

    Dependencies: D(t) after B(pair of t) and D(t-1) (stream order); T(t) after D(t) and H(t-1); B(pair p + 2) reuses the
    buffers of pair p, i.e. runs after T / H of its second frame (two pair slots).  B(p+1) is enqueued while frame 2p is
    in its track stage, so D(2p+1), T(2p), T(2p+1) run under it.  An odd last frame takes the single-frame plan.
    Results are identical to frame-by-frame calls (every kernel treats the images of a batch independently)."""
    n_frames = len(frames)
    results = []
    cur = torch.cuda.current_stream(eng.device)
    sA, sD = eng.side_stream(), eng.tail_stream()
    sA.wait_stream(cur)
    sD.wait_stream(cur)
    KP = 2                          # pair slots
    slot_free = [None] * KP         # event: every reader of the pair slot's buffers is enqueued-complete
    single_free = [None]
    plans = {}
    # Backbone units: frame 0 ALONE (the first result then waits for one backbone pass, not two: 0.55 ms less pipeline fill per
    # clip, 3 % of a 20-frame clip), then pairs, then an odd last frame alone.  unit = (first frame, frames, pair slot | None)
    units, t = [], 0
    if n_frames >= 3:
        units.append((0, 1, None))
        t = 1
    while t < n_frames:
        c = 2 if t + 1 < n_frames else 1
        units.append((t, c, (sum(1 for u in units if u[1] == 2) % KP) if c == 2 else None))
        t += c
    unit_of = {}
    for u, (f, c, _) in enumerate(units):
        for i in range(c):
            unit_of[f + i] = u

    def backbone(u):
        """Backbone half of unit u."""
        t0, count, pslot = units[u]
        with torch.cuda.stream(sA):
            if count == 2:
                if slot_free[pslot] is not None:
                    sA.wait_event(slot_free[pslot])
                PP = eng.run_backbone_pair(frames[t0], frames[t0 + 1], pslot)
                if PP.backbone_done is None:
                    PP.backbone_done = torch.cuda.Event()
                PP.backbone_done.record(sA)
                plans[t0], plans[t0 + 1] = PP.frames[0], PP.frames[1]
                PP.frames[0].backbone_done = PP.frames[1].backbone_done = PP.backbone_done
            else:
                if single_free[0] is not None:
                    sA.wait_event(single_free[0])
                P = (eng.run_static_raw(frames[t0], 0, part=0) if _is_raw_frame(frames[t0]) else eng.run_static(frames[t0], 0, part=0))
                if P.backbone_done is None:
                    P.backbone_done = torch.cuda.Event()
                P.backbone_done.record(sA)
                plans[t0] = P

    def detect(t):
        P = plans[t]
        with torch.cuda.stream(sD):
            sD.wait_event(P.backbone_done)
            eng.run_tail(P)
            if P.static_done is None:
                P.static_done = torch.cuda.Event()
            P.static_done.record(sD)

    deferred = []
    with torch.no_grad():
        backbone(0)
        detect(0)
        for t in range(n_frames):
            P = plans.pop(t)
            if before_frame is not None:
                before_frame(t)
            cur.wait_event(P.static_done)          # D(t) complete (hence B of its unit)
            pending = self.roi_heads.launch_frame(P, self._mem, given_detections[t] if given_detections is not None else None)
            _run_deferred(deferred, results)
            u = unit_of[t]
            t0, count, pslot = units[u]
            if t == t0 and u + 1 < len(units):
                backbone(u + 1)                    # its buffers held the unit before u (or nothing), whose last reader finished in iteration t-1
            if t + 1 < n_frames:
                detect(t + 1)
            result, mem = self.roi_heads.finish_frame(pending, next_P=plans.get(t + 1), defer=deferred)
            if t == t0 + count - 1:                # the unit's buffers are free for their next user
                ev = torch.cuda.Event()
                ev.record(cur)
                if pslot is not None:
                    slot_free[pslot] = ev
                else:
                    single_free[0] = ev
            self.__dict__["_mem"] = self.__dict__["track_memory"] = mem      # (plain attributes: bypass nn.Module.__setattr__)
            results.append(result)
        _run_deferred(deferred, results)
        cur.wait_stream(sA)
        cur.wait_stream(sD)
    return results


SiamMOT.forward_clip = _forward_clip


def build_siammot(cfg):
    return SiamMOT(cfg)
