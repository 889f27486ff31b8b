"""Proposal selection, NMS and box decoding on the H100 at their size, tie and threshold edges, through siammot_b200.ops:
smot_sort_nms, smot_sort_nms_segmented, smot_rpn_select(_batched), smot_box_decode(_batched) against the references of
tests/select_cases.py (which documents the cases and derives the bounds).  Ids, counts and orders are exact; continuous
outputs are within the derived bounds."""
import pytest
import torch

import select_cases as sc

pytestmark = pytest.mark.gpu

DEV = "cuda"
N_VALUES = (1, 63, 64, 65, 127, 128, 129, 1024, 1185, 1186, 2048, 2049, 4095, 4096)


def ops():
    from siammot_b200 import ops as _ops
    return _ops


@pytest.mark.parametrize("n_max", N_VALUES)
def test_sort_nms_edges(n_max):
    calls, failures = sc.sort_nms_table(ops(), DEV, (n_max,))
    print("\nsort_nms n_max=%d: %d cases, IoU pairs where fp32 and exact disagree so far: %s" % (n_max, calls, sc.IOU_DISAGREEMENTS))
    assert not failures, failures[:5]


SEGMENTED = [(1, 2, 64), (1, 9, 1186), (3, 3, 65), (3, 9, 64), (8, 2, 1186), (8, 3, 65), (8, 9, 65), (3, 2, 1186), (1, 3, 64)]


def test_sort_nms_segmented_edges():
    calls, failures = sc.segmented_table(ops(), DEV, SEGMENTED)
    print("\nsort_nms_segmented: %d cases" % calls)
    assert not failures, failures[:5]


def test_sort_nms_segmented_refuses_too_many_segments():
    batch, ncls, n = 65536, 2, 1
    boxes = torch.zeros((batch * n, ncls, 4), device=DEV)
    scores = torch.ones((batch * n, ncls), device=DEV)
    count = torch.ones((batch,), dtype=torch.int32, device=DEV)
    ob = torch.full((batch, 1, 4), -7.0, device=DEV)
    os_ = torch.full((batch, 1), -7.0, device=DEV)
    blk = torch.full((batch, 2), -7, dtype=torch.int32, device=DEV)
    with pytest.raises(RuntimeError, match="65536 segments"):
        ops().sort_nms_segmented(boxes, scores, count, batch, ncls, 0.0, 0.5, 1, ob, os_, blk)
    torch.cuda.synchronize()
    assert bool((ob == -7).all()) and bool((os_ == -7).all()) and bool((blk == -7).all())


RPN_WORST = {}


@pytest.mark.parametrize("spec", sc.rpn_cases(), ids=lambda s: s["name"])
def test_rpn_select_edges(spec):
    logits_l, deltas_l, heads = sc.rpn_image(spec, 77)
    ref = sc.rpn_case_reference(spec, logits_l, deltas_l)
    ob, os_, oc = sc.run_rpn(ops(), DEV, spec, heads)
    err, ws, wb = sc.check_rpn(spec, ob[0], os_[0], int(oc[0]), ref)
    RPN_WORST[spec["name"]] = (ws, wb)
    print("\nrpn_select %s: %d rows, worst score |err|/bound %.3f, box %.3f" % (spec["name"], int(oc[0]), ws, wb))
    assert err is None, err


BATCHED_RPN = [
    dict(name="batched-small", shapes=[(15, 239), (56, 64), (1, 1)], kinds=["straddle", "pm_zero", "level_ties"], pre=1000, post=500,
         fpn=1200),
    dict(name="batched-21-chunks", shapes=[(224, 336), (1, 1)], kinds=["all_equal", "saturated", "pm_zero"], pre=1024, post=900,
         fpn=700, extreme=True),
]


@pytest.mark.parametrize("bspec", BATCHED_RPN, ids=lambda s: s["name"])
def test_rpn_select_batched_edges(bspec):
    """B = 3 images of one size with different tie structures; each image equals its own reference."""
    specs, refs, heads = [], [], []
    for b, kind in enumerate(bspec["kinds"]):
        spec = dict(bspec, levels=[s + (kind,) for s in bspec["shapes"]], nms=0.7, amodal=False, img=(333, 517))
        logits_l, deltas_l, h = sc.rpn_image(spec, 90 + b)
        specs.append(spec)
        refs.append(sc.rpn_case_reference(spec, logits_l, deltas_l))
        heads.append(h)
    cat = [torch.cat([h[l] for h in heads]) for l in range(len(bspec["shapes"]))]
    ob, os_, oc = sc.run_rpn(ops(), DEV, specs[0], cat, batched=True)
    for b in range(3):
        err, ws, wb = sc.check_rpn(specs[b], ob[b], os_[b], int(oc[b]), refs[b])
        RPN_WORST["%s/%d" % (bspec["name"], b)] = (ws, wb)
        print("\nrpn_select_batched %s image %d: %d rows, worst score |err|/bound %.3f, box %.3f" % (bspec["name"], b, int(oc[b]), ws, wb))
        assert err is None, (b, err)


def _check_decode(gb, gs, ref, rows):
    """Worst |err|/bound of scores and boxes; a zero bound (a track row's other classes) demands an exact 0."""
    p, pb, b, bb = ref
    de = (gs[rows].double() - p[rows]).abs()
    zero = pb[rows] == 0
    es = float((de[~zero] / pb[rows][~zero]).max()) if bool((de[zero] == 0).all()) else float("inf")
    eb = float(((gb[rows].double() - b[rows]).abs() / bb[rows]).max())
    return es, eb


@pytest.mark.parametrize("ncls", [2, 9])
@pytest.mark.parametrize("tracks,amodal", [(False, False), (True, False), (False, True)])
def test_box_decode_edges(ncls, tracks, amodal):
    n, ld = 300, 5 * ncls + 3
    w = (10.0, 10.0, 5.0, 5.0)
    head, rois = sc.box_decode_scene(n, ncls, ld, 40 + ncls)
    labels = torch.randint(1, ncls, (n,), generator=torch.Generator().manual_seed(5)).int() if tracks else None
    gb, gs = ops().box_decode(head.to(DEV), rois.to(DEV), ncls, w, 320, 192, amodal,
                              track_labels=labels.to(DEV) if tracks else None)
    ref = sc.box_decode_expected(head, rois, ncls, w, 320, 192, amodal, labels)
    es, eb = _check_decode(gb.cpu(), gs.cpu(), ref, slice(0, n))
    print("\nbox_decode ncls=%d tracks=%s amodal=%s: %d rows, worst score |err|/bound %.3f, box %.3f" % (ncls, tracks, amodal, n, es, eb))
    assert es <= 1.0 and eb <= 1.0
    if tracks:
        gs = gs.cpu()
        own = gs[torch.arange(n), labels.long()]
        assert bool((own >= 1.0).all())
        others = gs.clone()
        others[torch.arange(n), labels.long()] = 0.0
        assert bool((others == 0).all())
    else:
        assert bool((gs == 0).any())          # probabilities that underflow to 0


@pytest.mark.parametrize("ncls", [2, 9])
def test_box_decode_batched_edges(ncls):
    B, n, ld = 3, 200, 5 * ncls + 2
    w = (10.0, 10.0, 5.0, 5.0)
    head, rois = sc.box_decode_scene(B * n, ncls, ld, 60 + ncls)
    count = torch.tensor([n - 57, 0, n + 7], dtype=torch.int32)
    gb, gs = ops().box_decode_batched(head.to(DEV), rois.view(B, n, 4).to(DEV), count.to(DEV), ncls, w, 320, 192, False)
    gb, gs = gb.cpu(), gs.cpu()
    ref = sc.box_decode_expected(head, rois, ncls, w, 320, 192, False)
    for b in range(B):
        k = min(int(count[b]), n)
        rows = slice(b * n, b * n + k)
        if k:
            es, eb = _check_decode(gb, gs, ref, rows)
            print("\nbox_decode_batched ncls=%d image %d: %d rows, worst score |err|/bound %.3f, box %.3f" % (ncls, b, k, es, eb))
            assert es <= 1.0 and eb <= 1.0, b
        assert bool((gs[b * n + k:(b + 1) * n] == -1).all()) and bool((gb[b * n + k:(b + 1) * n] == 0).all()), b
