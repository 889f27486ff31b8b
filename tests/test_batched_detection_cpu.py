"""Batched detection (Engine.batch_plan, SiamMOT.forward on a (B,3,H,W) batch of a detector-only model) without a GPU:

* the product's host code runs end to end over tests/batched_emulator.py (tests/cabi_emulator.py plus the batched entry
  points) and must reproduce what the reference's own detector-only model returns for one batched call
  (tests/golden/detect_batch3_192x320.pt), and equal per-image calls exactly;
* the calls the batch path refuses raise ValueError;
* the source of the kernels the batched entry points run, compiled over tests/cpu_cuda/shim.h, reproduces the single-image
  launches bit for bit (the batched ROIAlign and box decode) and the per-class append loop (the segmented NMS's scatter).
  The sort / mask / reduce kernels of the segmented NMS and the proposal selection use warp intrinsics the shim does not model;
  their batched instantiations (an image index in the grid, chosen at compile time) are compared with per-image calls by the
  `-m gpu` tests.
"""
import ctypes as C
import os
import sys

import pytest
import torch

import batched_emulator
import cabi_emulator
from helpers import CONFIG_DIR, YAML_MAP

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "cpu_cuda"))
GOLDEN = os.path.join(HERE, "golden", "detect_batch3_192x320.pt")
BOX_TOL, SCORE_TOL = 1e-3, 1e-3


def _inputs(track_on=False):
    from siammot_b200.config import get_cfg
    from siammot_b200.synth_clip import make_clip
    from siammot_b200.synthetic import make_state_dict
    gold = torch.load(GOLDEN, weights_only=False)
    sc = gold["spec"]
    cfg = get_cfg()
    cfg.merge_from_file(os.path.join(CONFIG_DIR, YAML_MAP[sc["yaml"]]))
    cfg.merge_from_list(sc["overrides"])
    cfg.MODEL.TRACK_ON = track_on
    cfg.DTYPE = "float32"
    clip = make_clip(sc["frames"], sc["H"], sc["W"], sc["n_obj"], sc["clip_seed"])
    batch = torch.stack([clip[t] for t in sc["pick"]])
    return cfg, make_state_dict(cfg, sc["weight_seed"]), batch, gold


def _model(cfg, sd):
    from siammot_b200.modelling import build_siammot
    model = build_siammot(cfg)
    model.load_state_dict(sd, strict=False)
    return model.eval()


def test_emulated_batched_forward_matches_reference_golden(monkeypatch):
    fake = batched_emulator.install(monkeypatch)
    cfg, sd, batch, gold = _inputs()
    out = _model(cfg, sd)(batch)
    assert len(out) == len(gold["images"]) == batch.shape[0]
    for i, (r, g) in enumerate(zip(out, gold["images"])):
        assert r.bbox.shape == g["boxes"].shape, "image %d: %d boxes vs %d" % (i, r.bbox.shape[0], g["boxes"].shape[0])
        assert torch.equal(r.get_field("labels"), g["labels"]), "image %d labels" % i
        assert torch.equal(r.get_field("ids"), torch.full_like(g["labels"], -1))
        assert float((r.bbox - g["boxes"]).abs().max()) <= BOX_TOL, "image %d boxes" % i
        assert float((r.get_field("scores") - g["scores"]).abs().max()) <= SCORE_TOL, "image %d scores" % i
    for name in ("smot_rpn_select_batched", "smot_roi_align_batched", "smot_box_decode_batched", "smot_sort_nms_segmented"):
        assert fake.calls.get(name) == 1, name


@pytest.mark.parametrize("on_host", [False, True])
def test_emulated_batched_forward_equals_per_image_calls(monkeypatch, on_host):
    batched_emulator.install(monkeypatch)
    cfg, sd, batch, _ = _inputs()
    model = _model(cfg, sd)
    model.results_on_host = on_host
    got = model(batch)
    for i in range(batch.shape[0]):
        one = model(batch[i:i + 1])[0]
        for field in ("scores", "ids", "labels"):
            assert torch.equal(got[i].get_field(field), one.get_field(field)), (i, field)
        assert torch.equal(got[i].bbox, one.bbox) and got[i].size == one.size == (batch.shape[3], batch.shape[2])
    again = model(batch[[2, 0]])   # another B: its own plan
    assert torch.equal(again[0].bbox, got[2].bbox) and torch.equal(again[1].bbox, got[0].bbox)


def test_batched_forward_refusals(monkeypatch):
    batched_emulator.install(monkeypatch)
    from siammot_b200.structures import BoxList
    cfg, sd, batch, _ = _inputs()
    model = _model(cfg, sd)

    class ImageList(object):
        def __init__(self, tensors, image_sizes):
            self.tensors, self.image_sizes = tensors, image_sizes

    H, W = batch.shape[2], batch.shape[3]
    ok = model(ImageList(batch, [(H, W)] * 3))
    assert len(ok) == 3
    with pytest.raises(ValueError, match="padded ImageList"):
        model(ImageList(batch, [(H, W), (H - 32, W), (H, W)]))
    det = BoxList(torch.tensor([[10.0, 10.0, 60.0, 80.0]]), (W, H), mode="xyxy")
    with pytest.raises(ValueError, match="given_detection"):
        model(batch, given_detection=[det])
    cfg_t, sd_t, _, _ = _inputs(track_on=True)
    with pytest.raises(ValueError, match="tracking model"):
        _model(cfg_t, sd_t)(batch)


# ---- kernel source under the CPU shim --------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def batched_kernels(tmp_path_factory):
    import re
    import cpu_cuda_build as cb
    repo = os.path.dirname(HERE)
    roi = open(os.path.join(repo, "siammot_b200", "csrc", "roi_align.cu")).read()
    sel = open(os.path.join(repo, "siammot_b200", "csrc", "select_nms.cu")).read()
    header = open(os.path.join(repo, "include", "smot.h")).read()
    pyramid = re.search(r"typedef struct \{\s*const void\* feat\[SMOT_MAX_LEVELS\];.*?\} smot_pyramid;", header, re.S).group(0)
    parts = ['#include "shim.h"', "#include <math.h>", "#define SMOT_MAX_LEVELS 5", pyramid, "namespace smot {",
             re.search(r"struct RoiArgs \{.*?\n\};", roi, re.S).group(0),
             re.search(r"constexpr int RAP_TP = \d+;[^\n]*", roi).group(0),
             re.search(r"constexpr float BBOX_XFORM_CLIP = [^\n]*", sel).group(0),
             cb._function_text(roi, r"__global__ void roi_align_kernel"),
             cb._rows_kernel_text(roi),
             cb._function_text(sel, r"__global__ void box_decode_kernel"),
             cb._function_text(sel, r"__global__ void __launch_bounds__\(256\) nms_scatter_segments_kernel"),
             "}  // namespace smot", """
using namespace smot;
// the launches of roi_align_nhwc (roi_align.cu): `rows` = 1 the row kernel with the product's rows-per-CTA rule, 0 the warp-per-bin one
extern "C" void cpu_roi_align_batched(const smot_pyramid* pyr, const long long* strides, int batch, const float* rois, const int* count,
                                      int max_rois, int channels, int res, int sampling, float* out, int rows) {
  RoiArgs a;
  a.pyr = *pyr, a.rois = rois, a.level_boxes = nullptr, a.count = count;
  a.max_rois = max_rois, a.channels = channels, a.res = res, a.sampling = sampling, a.batch = batch;
  for (int l = 0; l < SMOT_MAX_LEVELS; ++l) a.img_stride[l] = strides ? strides[l] : 0;
  int rpc = (64 + res - 1) / res;
  if (rpc > res) rpc = res;
  // strides: smot_roi_align_batched's BATCHED instantiations; none: smot_roi_align's
  const dim3 rgrid((res + rpc - 1) / rpc, batch * max_rois), wgrid((unsigned)(((long long)batch * max_rois * res * res * 32 + 255) / 256));
  if (rows && strides)
    cpu_launch(rgrid, dim3(256), [&] { roi_align_rows_kernel<float, false, 0, true>(a, out, rpc, 0); });
  else if (rows)
    cpu_launch(rgrid, dim3(256), [&] { roi_align_rows_kernel<float, false, 0>(a, out, rpc, 0); });
  else if (strides)
    cpu_launch(wgrid, dim3(256), [&] { roi_align_kernel<float, true>(a, out); });
  else
    cpu_launch(wgrid, dim3(256), [&] { roi_align_kernel<float>(a, out); });
}
extern "C" void cpu_box_decode(const float* head, int head_ld, const float* rois, const int* count, int batch, int n_max, int ncls,
                               const float* w, int img_w, int img_h, float* out_boxes, float* out_scores) {
  // batch > 1: smot_box_decode_batched's instantiation; 1: smot_box_decode's
  cpu_launch(dim3((batch * n_max + 127) / 128), dim3(128), [&] {
    if (batch > 1)
      box_decode_kernel<true>(head, head_ld, rois, count, n_max, batch, ncls, w[0], w[1], w[2], w[3], img_w, img_h, 0, nullptr, out_boxes, out_scores);
    else
      box_decode_kernel<false>(head, head_ld, rois, count, n_max, batch, ncls, w[0], w[1], w[2], w[3], img_w, img_h, 0, nullptr, out_boxes, out_scores);
  });
}
extern "C" void cpu_scatter(const float* boxes, const float* scores, int batch, int n_max, int ncls, const int* kept_index, const int* kept_n,
                            int cap, float* out_boxes, float* out_scores, int* out_block) {
  cpu_launch(dim3(batch * (ncls - 1)), dim3(64), [&] {
    nms_scatter_segments_kernel(boxes, scores, n_max, ncls, kept_index, kept_n, cap, out_boxes, out_scores, out_block);
  });
}
"""]
    d = tmp_path_factory.mktemp("batched_cpu")
    src = os.path.join(str(d), "batched_cpu.cpp")
    with open(src, "w") as f:
        f.write("\n".join(parts) + "\n")
    return C.CDLL(cb._compile(src, os.path.join(str(d), "batched_cpu.so")))


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _pyramid(maps, scales):
    from siammot_b200._lib import Pyramid
    p = Pyramid()
    p.num_levels, p.k_min = len(maps), 2
    for l, m in enumerate(maps):
        p.feat[l], p.H[l], p.W[l], p.ld[l], p.scale[l], p.pad[l] = m.data_ptr(), m.shape[1], m.shape[2], m.shape[3], scales[l], 0
    return p


def _rois(g, n, H, W):
    xy = torch.rand((n, 2), generator=g) * torch.tensor([W * 0.9, H * 0.9])
    wh = torch.rand((n, 2), generator=g) * torch.tensor([W * 0.6, H * 0.6]) + 2
    return torch.cat([xy, torch.minimum(xy + wh, torch.tensor([W - 1.0, H - 1.0]))], 1).float()


@pytest.mark.parametrize("rows", [1, 0])
def test_batched_roi_align_source_equals_per_image_launches(batched_kernels, rows):
    g = torch.Generator().manual_seed(7)
    B, n, Cc, res, H, W = 3, 20, 8, 7, 128, 192
    scales = [0.25, 0.125, 0.0625, 0.03125]
    maps = [torch.randn((B, H >> (l + 2), W >> (l + 2), Cc), generator=g) for l in range(4)]
    rois = torch.stack([_rois(g, n, H, W) for _ in range(B)]).contiguous()
    count = torch.tensor([n, 0, 13], dtype=torch.int32)      # a full segment, an empty one, a partial one
    strides = (C.c_longlong * 5)(*[m[0].numel() for m in maps], 0)
    out = torch.full((B * n, res, res, Cc), 7.0)
    batched_kernels.cpu_roi_align_batched(C.byref(_pyramid(maps, scales)), strides, B, _p(rois), _p(count), n, Cc, res, 2, _p(out), rows)
    for b in range(B):
        ref = torch.full((n, res, res, Cc), 7.0)
        one = [m[b:b + 1].contiguous() for m in maps]
        batched_kernels.cpu_roi_align_batched(C.byref(_pyramid(one, scales)), None, 1, _p(rois[b].contiguous()), _p(count[b:b + 1]), n,
                                              Cc, res, 2, _p(ref), rows)
        assert torch.equal(out[b * n:(b + 1) * n], ref), b
        assert float(out[b * n + int(count[b]):(b + 1) * n].abs().max() if count[b] < n else 0.0) == 0.0


def test_batched_box_decode_source_equals_per_image_launches(batched_kernels):
    g = torch.Generator().manual_seed(3)
    B, n, ncls, H, W = 3, 40, 3, 192, 320
    ld = ((5 * ncls + 3) // 4) * 4
    head = torch.randn((B * n, ld), generator=g)
    rois = torch.stack([_rois(g, n, H, W) for _ in range(B)]).contiguous()
    count = torch.tensor([n, 17, 0], dtype=torch.int32)
    w = torch.tensor([10.0, 10.0, 5.0, 5.0])
    ob, os_ = torch.full((B * n, ncls, 4), 9.0), torch.full((B * n, ncls), 9.0)
    batched_kernels.cpu_box_decode(_p(head), ld, _p(rois), _p(count), B, n, ncls, _p(w), W, H, _p(ob), _p(os_))
    for b in range(B):
        rb, rs = torch.full((n, ncls, 4), 9.0), torch.full((n, ncls), 9.0)
        batched_kernels.cpu_box_decode(_p(head[b * n:(b + 1) * n].contiguous()), ld, _p(rois[b].contiguous()), _p(count[b:b + 1]), 1, n,
                                       ncls, _p(w), W, H, _p(rb), _p(rs))
        assert torch.equal(ob[b * n:(b + 1) * n], rb) and torch.equal(os_[b * n:(b + 1) * n], rs), b
        assert bool((rs[int(count[b]):] == -1).all()) and bool((rb[int(count[b]):] == 0).all())


def test_segmented_scatter_source_equals_the_per_class_append_loop(batched_kernels):
    """The scatter of smot_sort_nms_segmented (per-image prefix over the class keep counts) against the emulator's per-class
    smot_sort_nms loop, which is the single-image tail's specification, on the same decoded boxes."""
    from oracle import prims
    g = torch.Generator().manual_seed(11)
    B, n, ncls = 4, 48, 4
    K, cap = ncls - 1, n * (ncls - 1)
    boxes = torch.cat([_rois(g, B * n * ncls, 192, 320)], 0).view(B * n, ncls, 4).contiguous()
    scores = torch.rand((B * n, ncls), generator=g)
    scores[n:2 * n] = 0.01           # image 1: nothing above the threshold
    boxes[2 * n:3 * n] = torch.tensor([float(i) * 50 for i in range(n)]).view(n, 1, 1) + torch.tensor([0.0, 0.0, 10.0, 10.0])
    scores[2 * n:3 * n] += 0.5
    count = torch.tensor([n, n, n, 30], dtype=torch.int32)   # image 2: disjoint boxes, every segment at capacity
    min_score, thresh = 0.05, 0.5
    kept_index = torch.zeros((B * K, n), dtype=torch.int32)
    kept_n = torch.zeros((B * K,), dtype=torch.int32)
    for b in range(B):
        m = int(count[b])
        for j in range(1, ncls):
            s = scores[b * n:b * n + m, j]
            cand = (s > min_score).nonzero().squeeze(1)
            keep = cand[prims.nms_legacy(boxes[b * n:b * n + m, j][cand], s[cand], thresh)][:n]
            kept_index[b * K + j - 1, :keep.numel()] = keep.to(torch.int32)
            kept_n[b * K + j - 1] = keep.numel()
    ob, os_, blk = torch.zeros((B, cap, 4)), torch.zeros((B, cap)), torch.zeros((B, 1 + cap), dtype=torch.int32)
    batched_kernels.cpu_scatter(_p(boxes), _p(scores), B, n, ncls, _p(kept_index), _p(kept_n), cap, _p(ob), _p(os_), _p(blk))
    fake = cabi_emulator.FakeLib()
    for b in range(B):
        rb, rs, rblk = torch.zeros((cap, 4)), torch.full((cap,), -1.0), torch.zeros((1 + cap,), dtype=torch.int32)
        for j in range(1, ncls):
            fake.smot_sort_nms(boxes.data_ptr() + 16 * (b * n * ncls + j), 4 * ncls, scores.data_ptr() + 4 * (b * n * ncls + j), ncls,
                               count[b:b + 1].data_ptr(), n, min_score, thresh, n, j, None, rb.data_ptr(), rs.data_ptr(),
                               rblk.data_ptr() + 4, rblk.data_ptr(), None, 0, None)
        k = int(rblk[0])
        assert int(blk[b, 0]) == k and torch.equal(blk[b, 1:1 + k], rblk[1:1 + k]), b
        assert torch.equal(ob[b, :k], rb[:k]) and torch.equal(os_[b], rs), b
    assert int(blk[1, 0]) == 0 and int(blk[2, 0]) == cap
