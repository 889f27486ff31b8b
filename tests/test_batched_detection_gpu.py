"""Batched detection on the H100: the batched entry points against per-image calls of the single-image ones (torch.equal, B in
{1, 2, 3, 8}), the batched forward of a detector-only model against the reference's batched call (tests/golden/
detect_batch3_192x320.pt) and, at 3x704x1280 in fp32 and fp16, against model(x[i:i+1]) bit for bit."""
import os

import pytest
import torch

from helpers import CONFIG_DIR, YAML_MAP

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "detect_batch3_192x320.pt")
BATCHES = [1, 2, 3, 8]


def _cfg(track_on=False, dtype="float32", yaml="DLA_34_FPN_EMM.yaml"):
    from siammot_b200.config import get_cfg
    cfg = get_cfg()
    cfg.merge_from_file(os.path.join(CONFIG_DIR, YAML_MAP[yaml]))
    cfg.MODEL.TRACK_ON = track_on
    cfg.DTYPE = dtype
    return cfg


def _model(cfg, seed=0):
    from siammot_b200.modelling import build_siammot
    from siammot_b200.synthetic import make_state_dict
    model = build_siammot(cfg)
    model.load_state_dict(make_state_dict(cfg, seed), strict=False)
    return model.to("cuda").eval()


def _rois(g, B, n, H, W):
    xy = torch.rand((B, n, 2), generator=g) * torch.tensor([W * 0.9, H * 0.9])
    wh = torch.rand((B, n, 2), generator=g) * torch.tensor([W * 0.7, H * 0.7]) + 2
    return torch.cat([xy, torch.minimum(xy + wh, torch.tensor([W - 1.0, H - 1.0]))], 2).float().cuda().contiguous()


# ---- entry points vs per-image calls ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", BATCHES)
def test_rpn_select_batched_equals_per_image(B):
    from siammot_b200 import ops
    from siammot_b200.engine import cell_anchors
    g = torch.Generator().manual_seed(B)
    H, W, A, ld = 704, 1280, 3, 16
    strides, sizes = (4, 8, 16, 32, 64), (32, 64, 128, 256, 512)
    cells = [cell_anchors(st, (sz,), (0.5, 1.0, 2.0)) for st, sz in zip(strides, sizes)]
    heads = []
    for l, st in enumerate(strides):
        h = torch.randn((B, -(-H // st), -(-W // st), ld), generator=g)
        h[..., A:5 * A] *= 0.2
        if B > 1:
            h[1, ..., :A] = torch.round(h[1, ..., :A] * 2) / 2      # image 1: heavy logit ties (anchor-index order decides)
        if B > 2:
            h[2, ..., :A] -= 6.0                                    # image 2: low objectness everywhere
        heads.append(h.cuda())
    n, post = 1000, 800                                             # pre_nms_top_n, post_nms_top_n 1000 / 800, top 1000 overall
    ws = ops.rpn_select_batched_workspace(5, 1000, B, "cuda")
    levels = ops.rpn_levels(heads, strides, cells)
    ob, os_, oc = torch.full((B, n, 4), 7.0, device="cuda"), torch.full((B, n), 7.0, device="cuda"), torch.zeros((B,), dtype=torch.int32, device="cuda")
    ops.rpn_select_batched(heads, levels, 1000, post, 0.7, 0.0, n, W, H, False, ob, os_, oc, ws)
    ws1 = ops.rpn_select_workspace(5, 1000, "cuda")
    for b in range(B):
        one = [h[b:b + 1] for h in heads]
        rb, rs, rc = torch.full((n, 4), 7.0, device="cuda"), torch.full((n,), 7.0, device="cuda"), torch.zeros((1,), dtype=torch.int32, device="cuda")
        ops.rpn_select(ops.rpn_levels(one, strides, cells), 1000, post, 0.7, 0.0, n, W, H, False, rb, rs, rc, ws1)
        k = int(rc[0])
        assert int(oc[b]) == k, b
        assert torch.equal(ob[b, :k], rb[:k]) and torch.equal(os_[b, :k], rs[:k]), b


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("B", BATCHES)
def test_roi_align_batched_equals_per_image(B, dtype):
    from siammot_b200 import ops
    g = torch.Generator().manual_seed(10 + B)
    H, W, Cc, n = 704, 1280, 128, 1000
    scales = (0.25, 0.125, 0.0625, 0.03125)
    feats = [torch.randn((B, H >> (l + 2), W >> (l + 2), Cc), generator=g).to("cuda", dtype) for l in range(4)]
    rois = _rois(g, B, n, H, W)
    count = torch.tensor([(n, 0, 517, n // 2)[b % 4] for b in range(B)], dtype=torch.int32, device="cuda")
    out = ops.roi_align_batched(feats, rois, count, scales, 7, 2)
    for b in range(B):
        ref = ops.roi_align([f[b:b + 1] for f in feats], rois[b], scales, 7, 2, count=count[b:b + 1])
        assert torch.equal(out[b * n:(b + 1) * n], ref), b


@pytest.mark.parametrize("B", BATCHES)
def test_box_decode_batched_equals_per_image(B):
    from siammot_b200 import ops
    g = torch.Generator().manual_seed(20 + B)
    n, ncls, H, W = 1000, 3, 704, 1280
    ld = ((5 * ncls + 3) // 4) * 4
    head = torch.randn((B * n, ld), generator=g).cuda()
    rois = _rois(g, B, n, H, W)
    count = torch.tensor([(n, 311, 0)[b % 3] for b in range(B)], dtype=torch.int32, device="cuda")
    w = (10.0, 10.0, 5.0, 5.0)
    ob, os_ = ops.box_decode_batched(head, rois, count, ncls, w, W, H, False)
    for b in range(B):
        rb, rs = ops.box_decode(head[b * n:(b + 1) * n], rois[b], ncls, w, W, H, False, count=count[b:b + 1])
        assert torch.equal(ob[b * n:(b + 1) * n], rb) and torch.equal(os_[b * n:(b + 1) * n], rs), b
        assert bool((rs[int(count[b]):] == -1).all())


@pytest.mark.parametrize("B", BATCHES)
def test_sort_nms_segmented_equals_the_per_class_loop(B):
    """Image 0: nothing above SCORE_THRESH; image 1: much fuller than the others, every segment at capacity (disjoint boxes, all
    scores high); the rest random."""
    from siammot_b200 import ops
    g = torch.Generator().manual_seed(30 + B)
    n, ncls, H, W = 1000, 3, 704, 1280
    K, cap = ncls - 1, n * (ncls - 1)
    boxes = _rois(g, B * n, ncls, H, W).view(B * n, ncls, 4).contiguous()
    scores = torch.rand((B * n, ncls), generator=g).cuda()
    count = torch.full((B,), n, dtype=torch.int32, device="cuda")
    scores[0:n] *= 0.04
    if B > 1:
        i = torch.arange(n, device="cuda", dtype=torch.float32)
        base = torch.stack([(i % 40) * 32, (i // 40) * 28, (i % 40) * 32 + 20, (i // 40) * 28 + 20], 1)
        boxes[n:2 * n] = base.view(n, 1, 4)
        scores[n:2 * n] = 0.5 + 0.4 * scores[n:2 * n]
    if B > 2:
        count[2] = 123
    ob = torch.zeros((B, cap, 4), device="cuda")
    os_ = torch.zeros((B, cap), device="cuda")
    blk = torch.zeros((B, 1 + cap), dtype=torch.int32, device="cuda")
    ops.sort_nms_segmented(boxes, scores, count, B, ncls, 0.05, 0.5, n, ob, os_, blk)
    ws = ops.sort_nms_workspace(n, "cuda")
    for b in range(B):
        rb = torch.zeros((cap, 4), device="cuda")
        rs = torch.full((cap,), -1.0, device="cuda")
        rblk = torch.zeros((1 + cap,), dtype=torch.int32, device="cuda")
        for j in range(1, ncls):
            ops.sort_nms(boxes[b * n:(b + 1) * n, j], scores[b * n:(b + 1) * n, j], rblk[0:1], n_max=n, count=count[b:b + 1],
                         min_score=0.05, thresh=0.5, max_keep=n, tag=j, out_boxes=rb, out_scores=rs, out_tag=rblk[1:],
                         workspace=ws, box_stride=4 * ncls, score_stride=ncls)
        k = int(rblk[0])
        assert int(blk[b, 0]) == k, b
        assert torch.equal(blk[b, 1:1 + k], rblk[1:1 + k]) and torch.equal(ob[b, :k], rb[:k]) and torch.equal(os_[b], rs), b
    assert int(blk[0, 0]) == 0
    if B > 1:
        assert int(blk[1, 0]) == cap


# ---- end to end --------------------------------------------------------------------------------------------------------------
def test_batched_forward_fp32_matches_reference_golden():
    from siammot_b200.synth_clip import make_clip
    gold = torch.load(GOLDEN, weights_only=False)
    sc = gold["spec"]
    cfg = _cfg()
    cfg.merge_from_list(sc["overrides"])
    model = _model(cfg, sc["weight_seed"])
    clip = make_clip(sc["frames"], sc["H"], sc["W"], sc["n_obj"], sc["clip_seed"])
    out = model(torch.stack([clip[t] for t in sc["pick"]]).cuda())
    assert len(out) == len(gold["images"])
    for i, (r, g) in enumerate(zip(out, gold["images"])):
        assert r.bbox.shape == g["boxes"].shape, "image %d: %d boxes vs %d" % (i, r.bbox.shape[0], g["boxes"].shape[0])
        assert torch.equal(r.get_field("labels").cpu(), g["labels"])
        assert float((r.bbox.cpu() - g["boxes"]).abs().max()) <= 1e-3
        assert float((r.get_field("scores").cpu() - g["scores"]).abs().max()) <= 1e-3


def _fields(r):
    return [r.bbox.cpu(), r.get_field("scores").cpu(), r.get_field("labels").cpu(), r.get_field("ids").cpu()]


@pytest.mark.parametrize("dtype", ["float32", "float16"])
def test_batched_forward_equals_single_image_calls_720p(dtype):
    from siammot_b200.synth_clip import make_clip
    model = _model(_cfg(dtype=dtype))
    x = torch.stack(list(make_clip(8, 704, 1280, 8, 5))).cuda()
    singles = [_fields(model(x[i:i + 1])[0]) for i in range(8)]
    assert sum(s[0].shape[0] for s in singles) > 0
    for B in (2, 3, 8):
        for on_host in (False, True):
            model.results_on_host = on_host
            first = model(x[:B])
            again = model(x[:B])                 # the second replay of the captured graph
            assert len(first) == B
            for i in range(B):
                a, b = _fields(first[i]), _fields(again[i])
                for u, v, w in zip(a, b, singles[i]):
                    assert torch.equal(u, w) and torch.equal(v, w), (dtype, B, on_host, i)
        model.results_on_host = False
    assert model.engine().plans[(704, 1280, "batch", 8)].graph is not None


def test_batched_forward_refusals_on_gpu():
    model = _model(_cfg(track_on=True))
    with pytest.raises(ValueError, match="tracking model"):
        model(torch.zeros((2, 3, 192, 320), device="cuda"))
