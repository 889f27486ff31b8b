"""CPU stand-ins for the batched detection entry points of include/smot.h -- TEST INFRASTRUCTURE, never imported by the product.

Extends tests/cabi_emulator.py's FakeLib: each batched entry point runs every image through the single-image emulation at the
pointers the engine passes (image offsets as the batched kernels compute them), so the product's batched host code
(Engine.batch_plan, SiamMOT.forward on a (B,3,H,W) batch) runs end to end without a GPU.
"""
import ctypes as C

import cabi_emulator
from cabi_emulator import _a, _f32, _i32


class BatchedFakeLib(cabi_emulator.FakeLib):
    def smot_rpn_select_batched_workspace(self, num_levels, pre_nms_top_n, batch):
        return 64

    def smot_sort_nms_segmented_workspace(self, batch, ncls, n_max):
        return 64

    def smot_rpn_select_batched(self, levels, strides, batch, num_levels, pre_n, post_n, nms_thresh, min_size, fpn_post_n, img_w,
                                img_h, amodal, out_boxes, out_scores, out_count, ws, ws_bytes, st):
        self._count("smot_rpn_select_batched")
        for b in range(batch):
            lv = (type(levels[0]) * num_levels)()
            for l in range(num_levels):
                lv[l] = type(levels[l]).from_buffer_copy(levels[l])
                lv[l].head = _a(levels[l].head) + 4 * b * int(strides[l])
            self.smot_rpn_select(lv, num_levels, pre_n, post_n, nms_thresh, min_size, fpn_post_n, img_w, img_h, amodal,
                                 _a(out_boxes) + 16 * b * fpn_post_n, _a(out_scores) + 4 * b * fpn_post_n, _a(out_count) + 4 * b,
                                 ws, ws_bytes, st)
        return 0

    def smot_roi_align_batched(self, pref, strides, batch, rois, count, max_rois, Cc, res, sampling, out, dt, st):
        self._count("smot_roi_align_batched")
        p = pref._obj
        for b in range(batch):
            q = type(p).from_buffer_copy(p)
            for l in range(p.num_levels):
                q.feat[l] = _a(p.feat[l]) + 4 * b * int(strides[l])
            self.smot_roi_align(C.byref(q), _a(rois) + 16 * b * max_rois, None, _a(count) + 4 * b, max_rois, Cc, res, sampling,
                                _a(out) + 4 * b * max_rois * res * res * Cc, dt, st)
        return 0

    def smot_box_decode_batched(self, head, head_ld, rois, count, batch, n_max, ncls, w4ref, img_w, img_h, amodal, out_boxes,
                                out_scores, st):
        self._count("smot_box_decode_batched")
        for b in range(batch):
            self.smot_box_decode(_a(head) + 4 * b * n_max * head_ld, head_ld, _a(rois) + 16 * b * n_max, _a(count) + 4 * b, n_max,
                                 ncls, w4ref, img_w, img_h, amodal, None, _a(out_boxes) + 16 * b * n_max * ncls,
                                 _a(out_scores) + 4 * b * n_max * ncls, st)
        return 0

    def smot_sort_nms_segmented(self, boxes, scores, count, batch, n_max, ncls, min_score, thresh, max_keep, cap, out_boxes,
                                out_scores, out_block, ws, ws_bytes, st):
        """The per-class loop of the single-image tail (scores -1, count 0, then classes 1 .. ncls-1 appended), per image."""
        self._count("smot_sort_nms_segmented")
        for b in range(batch):
            ob, os_ = _a(out_boxes) + 16 * b * cap, _a(out_scores) + 4 * b * cap
            blk = _a(out_block) + 4 * b * (1 + cap)
            _f32(os_, cap)[:] = -1.0
            _i32(blk, 1)[0] = 0
            for j in range(1, ncls):
                self.smot_sort_nms(_a(boxes) + 16 * (b * n_max * ncls + j), 4 * ncls, _a(scores) + 4 * (b * n_max * ncls + j), ncls,
                                   _a(count) + 4 * b, n_max, min_score, thresh, max_keep, j, None, ob, os_, blk + 4, blk, ws, ws_bytes,
                                   st)
        return 0


def install(monkeypatch):
    """cabi_emulator.install() with the library routed to a BatchedFakeLib instead.  Returns it."""
    from siammot_b200 import _lib, engine, ops, preprocess
    cabi_emulator.install(monkeypatch)
    fake = BatchedFakeLib()
    for mod in (_lib, engine, ops, preprocess):
        monkeypatch.setattr(mod, "lib", lambda: fake)
    return fake
