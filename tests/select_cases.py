"""Case generators and references for the proposal-selection kernels of csrc/select_nms.cu -- a helper module, not a test
file.  tests/test_select_edges_gpu.py runs the tables through siammot_b200.ops on the GPU; tests/test_select_kernels_on_cpu.py
runs smaller tables through the same kernels' source text on the host (tests/cpu_cuda/shim_warp.h), with `CpuOps` standing in
for siammot_b200.ops.

Every case places its inputs on one of the kernels' internal edges: the bitonic width (64 minimum), the 64-row blocks of the
suppression mask and of the reduction, the shared-memory bitmask limit (n_max 1185 staged, 1186 read from global memory), the
radix select's aggregated histogram and early exit, the 10752-anchor chunks, the shared (<= 20 chunks) and global (21) merge,
the cross-level rank merge, the BBOX_XFORM_CLIP clamp and the min_size filter; and on score / IoU ties and thresholds.

References
----------
* sort + NMS: ``prims.nms_legacy`` (fp32 ``_C.nms`` semantics, pinned against brute force in test_oracle_prims.py) on rows
  i < min(count, n_max) with score > min_score, truncated at max_keep; thresh <= 0 is sort only (smot.h).  Ids, boxes and
  scores must be exact.  ``iou_disagreements`` also recomputes every suppression decision with exact rationals (the boxes
  are integers) and records the pairs where fp32 and exact arithmetic disagree; that is reported, not asserted: the fp32
  rule is the contract.
* segmented NMS: the same reference per image and class, blocks assembled as the per-class loop would.
* RPN: ``oracle.rpn_select`` with cfg.MODEL.RPN overridden per case gives count, order and the fp32 scores; ``rpn_reference``
  restates it step by step so that it can also return each output row's logit, anchor and deltas (and asserts that its
  result equals the oracle's bit for bit).  Scores and boxes are then compared with float64 evaluations of the same
  formulas on the same fp32 inputs, within the bounds below.
* box decode: a float64 restatement of softmax + BoxCoder.decode + clip.

Bounds (u = 2^-24, the unit roundoff of fp32; first order in u, the second-order terms are below u^2 * 100 relative and are
covered by the factor 1 + 2^-10; expf / __expf of the CUDA math library has a documented maximum error of 2 ulp, i.e. a
relative error <= 4u, plus 2^-148 absolute where the result is subnormal; every other operation is one IEEE rounding:
<= u * |result| + 2^-150 absolute):
* sigmoid, s = 1 / (1 + expf(-x)) with a rounded add and a rounded division:
      |s' - s| <= s * (4u * e / (1 + e) + 2u),   e = exp(-x)
* decode of one coordinate (RPN weights 1; box head weights wx, wy, ww, wh: one rounded division each first):
      w = x2 - x1 + 1 (two roundings), c = x1 + 0.5 w, E = expf(min(d_w, CLIP)), pw = E * w, pc = d_x * w + c,
      x1' = pc - 0.5 pw, x2' = pc + 0.5 pw - 1;  the error of each is bounded by propagating |error| through these steps
      (``_decode_bound``); the clip to [0, img - 1] and the min with CLIP are 1-Lipschitz and add nothing.
* softmax, p_j = expf(x_j - m) / sum_k expf(x_k - m) (sequential sum, m = max): the error of x_j - m (u |x_j - m|) times
  the exp's slope, the exp's own 4u, ncls - 1 rounded adds of the sum and one rounded division (``_softmax_bound``).
  A track row's p + 1 adds one rounding.
"""
import ctypes as C
from fractions import Fraction

import numpy as np
import torch

from oracle import prims

U = 2.0 ** -24
SAFE = 1.0 + 2.0 ** -10
TINY = 2.0 ** -148
CLIP = float(np.float32(prims.BBOX_XFORM_CLIP))

SN_BLOCK = 64
SHARED_MASK_LIMIT = 1185      # largest n_max whose suppression bitmask nms_reduce_kernel stages in shared memory
RPN_CHUNK = 10752

IOU_DISAGREEMENTS = []        # (case, i, j, fp32 iou, exact iou, thresh): filled by iou_disagreements, reported by the tests


def f32(x):
    return np.float32(x)


# ---- sort + NMS ------------------------------------------------------------------------------------------------------------
SCORE_KINDS = ("distinct", "half_dup", "all_equal", "pm_zero", "at_min_score", "negative")
GEOMETRIES = ("random", "staircase", "cross_block", "clique", "degenerate", "iou_edges")
IOU_EDGE_THRESHOLDS = (0.4, 0.5, 0.6, 0.7)


def make_scores(kind, n, g):
    """(scores fp32 [n], min_score) for one of SCORE_KINDS."""
    if kind == "distinct":
        return (torch.randperm(n, generator=g).float() + 1.0) / (n + 1.0), -1e30
    if kind == "half_dup":
        s = torch.rand(n, generator=g)
        h = n // 2
        s[n - h:] = s[torch.randperm(h, generator=g)] if h else s[n - h:]   # every value of the first half appears twice
        return s, -1e30
    if kind == "all_equal":
        return torch.full((n,), 0.5), -1e30
    if kind == "pm_zero":   # mostly signed zeros, a few values on either side
        s = torch.tensor([0.0, -0.0, 0.0, -0.0, 0.0, -0.0, 0.25, -0.25])[torch.randint(0, 8, (n,), generator=g)]
        return s, -1.0
    if kind == "at_min_score":   # min_score equals a quarter of the scores: `score > min_score` drops them
        return torch.tensor([0.1, 0.2, 0.3, 0.4])[torch.randint(0, 4, (n,), generator=g)], float(np.float32(0.2))
    if kind == "negative":
        return -0.01 - torch.rand(n, generator=g), -1e30
    raise ValueError(kind)


def _rank_of_rows(scores):
    """Rank of every row in (score desc, index asc) order."""
    order = torch.sort(scores, descending=True, stable=True)[1]
    rank = torch.empty_like(order)
    rank[order] = torch.arange(order.numel())
    return rank


# Integer box pairs (inner [0,0,I-1,0] inside outer [0,0,U-1,0]: exact IoU(+1) = I/U) whose fp32 IoU, computed as the
# kernels do, I / ((I + U) - I), is fp32(thr), one ulp above and one ulp below (I, U, thr, fp32 IoU).  Near a simple fraction
# like 2/5 the next fractions are 1/(5U) apart, so U runs up to 2^24.  Found by scanning U with I = rint(target * U);
# verified below.
IOU_EDGE_PAIRS = [
    (2, 5, 0.4, 0.4000000059604645), (1579033, 3947582, 0.4, 0.40000003576278687), (2064889, 5162223, 0.4, 0.3999999761581421),
    (1, 2, 0.5, 0.5), (2796204, 5592407, 0.5, 0.5000000596046448), (5592405, 11184811, 0.5, 0.4999999701976776),
    (3, 5, 0.6, 0.6000000238418579), (1059614, 1766023, 0.6, 0.6000000834465027), (1830244, 3050407, 0.6, 0.5999999642372131),
    (7, 10, 0.7, 0.699999988079071), (903390, 1290557, 0.7, 0.7000000476837158), (690832, 986903, 0.7, 0.6999999284744263),
]
for _I, _U, _thr, _iou in IOU_EDGE_PAIRS:
    assert f32(_I) / ((f32(_I) + f32(_U)) - f32(_I)) == f32(_iou)
assert [np.float32(p[3]) - f32(p[2]) for p in IOU_EDGE_PAIRS[:3]] == [0, np.nextafter(f32(0.4), f32(1)) - f32(0.4),
                                                                        np.nextafter(f32(0.4), f32(0)) - f32(0.4)]


def make_boxes(geom, scores, g):
    """Boxes fp32 [n, 4] (integer coordinates except 'random') for one of GEOMETRIES; the chains follow the score order."""
    n = scores.numel()
    rank = _rank_of_rows(scores).float()
    if geom == "random":
        xy = torch.rand(n, 2, generator=g) * 300
        return torch.cat([xy, xy + torch.rand(n, 2, generator=g) * 120 + 2], 1)
    if geom == "staircase":   # box k+1 overlaps box k by 70/130 > 0.5, box k+2 by 40/160: greedy keeps every other box
        x = 30.0 * rank
        return torch.stack([x, torch.zeros(n), x + 99, torch.full((n,), 99.0)], 1)
    if geom == "cross_block":   # rank r's only suppressor is rank r - 64 (previous block); r - 128 is too far
        col, blk = torch.remainder(rank, SN_BLOCK), torch.div(rank, SN_BLOCK, rounding_mode="floor")
        x, y = 30.0 * blk, 200.0 * col
        return torch.stack([x, y, x + 99, y + 99], 1)
    if geom == "clique":
        return torch.tensor([[10.0, 20.0, 50.0, 70.0]]).repeat(n, 1)
    if geom == "degenerate":   # zero width (x2 = x1 - 1), negative width (x2 < x1 - 1), and ordinary boxes, all overlapping
        k = torch.remainder(torch.arange(n), 3)
        x1 = 10.0 + torch.remainder(torch.arange(n), 7).float()
        x2 = torch.where(k == 0, x1 - 1, torch.where(k == 1, x1 - 5, x1 + 20))
        return torch.stack([x1, torch.full((n,), 5.0), x2, torch.full((n,), 40.0)], 1)
    if geom == "iou_edges":   # the edge pairs on rows 0..23 (one per 10 pixels in y), disjoint unit boxes after them
        b = torch.zeros(n, 4)
        for p, (I, Uu, _, _) in enumerate(IOU_EDGE_PAIRS):
            for r, w in ((2 * p, I), (2 * p + 1, Uu)):
                if r < n:
                    b[r] = torch.tensor([0.0, 10.0 * p, w - 1.0, 10.0 * p])
        x = -1000.0 - 4 * torch.arange(min(2 * len(IOU_EDGE_PAIRS), n), n).float()
        b[min(2 * len(IOU_EDGE_PAIRS), n):] = torch.stack([x, torch.zeros_like(x), x + 1, torch.ones_like(x)], 1)
        return b
    raise ValueError(geom)


def nms_expected(boxes, scores, count, n_max, min_score, thresh, max_keep):
    """Kept row indices (list) of smot_sort_nms over rows i < min(count, n_max)."""
    n = max(0, min(count, n_max))
    live = torch.nonzero(scores[:n] > np.float32(min_score)).squeeze(1)
    if live.numel() == 0 or max_keep <= 0:
        return []
    b, s = boxes[live], scores[live]
    if thresh <= 0:
        keep = torch.sort(s, descending=True, stable=True)[1]
    else:
        keep = prims.nms_legacy(b, s, thresh)
    return live[keep[:max_keep]].tolist()


def iou_disagreements(case, boxes, scores, count, n_max, min_score, thresh):
    """Pairs (higher-ranked i, j) among the candidates whose fp32 IoU(+1) > thresh decision differs from the exact one
    (integer boxes only; pairs with both areas positive).  Appended to IOU_DISAGREEMENTS; returns how many were found."""
    if thresh <= 0:
        return 0
    n = max(0, min(count, n_max))
    live = torch.nonzero(scores[:n] > np.float32(min_score)).squeeze(1)
    b = boxes[live].double().numpy()
    if b.shape[0] < 2 or not np.all(b == np.round(b)):
        return 0
    x1, y1, x2, y2 = b.T
    area = (x2 - x1 + 1) * (y2 - y1 + 1)
    found = 0
    for i in range(b.shape[0] - 1):
        w = np.maximum(np.minimum(x2[i], x2[i + 1:]) - np.maximum(x1[i], x1[i + 1:]) + 1, 0)
        h = np.maximum(np.minimum(y2[i], y2[i + 1:]) - np.maximum(y1[i], y1[i + 1:]) + 1, 0)
        inter = w * h
        union = area[i] + area[i + 1:] - inter
        ok = (inter > 0) & (area[i] > 0) & (area[i + 1:] > 0)
        near = np.nonzero(ok & (np.abs(inter / np.where(union > 0, union, 1) - thresh) < 1e-5))[0]
        for jj in near:
            I, Uu = int(inter[jj]), int(union[jj])
            exact = Fraction(I, Uu) > Fraction(thresh).limit_denominator(10 ** 9)
            fp = f32(I) / f32(Uu)
            if bool(fp > f32(thresh)) != exact:
                IOU_DISAGREEMENTS.append((case, int(live[i]), int(live[i + 1 + jj]), float(fp), I / Uu, thresh))
                found += 1
    return found


def sort_nms_cases(n_values):
    """The sort + NMS table: per n_max, every geometry once (with count n_max - 1, n_max or n_max + 5 and the score kinds
    cycled), plus count 0 and count 1."""
    cases = []
    for ni, n_max in enumerate(n_values):
        picks = [(GEOMETRIES[i], ("n", "n+5", "n-1")[(i + ni) % 3], SCORE_KINDS[(i + 2 * ni) % len(SCORE_KINDS)])
                 for i in range(len(GEOMETRIES))]
        picks += [("staircase", "zero", "distinct"), ("clique", "one", SCORE_KINDS[ni % len(SCORE_KINDS)])]
        for geom, ck, sk in picks:
            count = {"zero": 0, "one": 1, "n-1": n_max - 1, "n": n_max, "n+5": n_max + 5}[ck]
            cases.append(dict(name="n%d-c%s-%s-%s" % (n_max, ck, sk, geom), n_max=n_max, count=count, scores=sk, geom=geom,
                              seed=1000 + len(cases), strided=len(cases) % 2 == 0))
    return cases


def sort_nms_scene(case):
    """Rows n_max + 5 (the count may exceed n_max; rows past n_max must be ignored), fp32 boxes / scores."""
    g = torch.Generator().manual_seed(case["seed"])
    n = case["n_max"] + 5
    scores, min_score = make_scores(case["scores"], n, g)
    boxes = make_boxes(case["geom"], scores[:case["n_max"]], g)
    boxes = torch.cat([boxes, torch.tensor([[0.0, 0.0, 1e4, 1e4]]).repeat(5, 1)])   # out-of-range rows: would suppress all
    scores[case["n_max"]:] = 2.0
    thresholds = IOU_EDGE_THRESHOLDS if case["geom"] == "iou_edges" else (0.5,)
    return boxes, scores.float(), min_score, thresholds


def max_keep_values(kept):
    return sorted({0, 1, 63, 64, 65, max(kept - 1, 0), kept, kept + 10})


def run_sort_nms(ops, dev, boxes, scores, count, n_max, min_score, thresh, max_keep, strided, tag=3):
    """One smot_sort_nms call on fresh sentinel-filled outputs.  strided: rows of 8 floats / scores every 3rd float and 7
    rows already in the output (appended behind them).  Returns (index, boxes, scores, tags, out_count, base) on the host."""
    n = boxes.shape[0]
    if strided:
        bx = torch.full((n, 8), 777.0)
        bx[:, :4] = boxes
        sc = torch.full((n, 3), 777.0)
        sc[:, 0] = scores
        bx, sc, box_stride, score_stride, base = bx.to(dev), sc.to(dev), 8, 3, 7
    else:
        bx, sc, box_stride, score_stride, base = boxes.to(dev), scores.to(dev), 4, 1, 0
    cap = base + n_max + 16
    out_count = torch.tensor([base], dtype=torch.int32, device=dev)
    oi = torch.full((cap,), -7, dtype=torch.int32, device=dev)
    ob = torch.full((cap, 4), -7.0, device=dev)
    os_ = torch.full((cap,), -7.0, device=dev)
    ot = torch.full((cap,), -7, dtype=torch.int32, device=dev)
    cnt = torch.tensor([count], dtype=torch.int32, device=dev)
    ops.sort_nms(bx, sc, out_count, n_max=n_max, count=cnt, min_score=min_score, thresh=thresh, max_keep=max_keep, tag=tag,
                 out_index=oi, out_boxes=ob, out_scores=os_, out_tag=ot, box_stride=box_stride, score_stride=score_stride)
    return oi.cpu(), ob.cpu(), os_.cpu(), ot.cpu(), int(out_count.cpu()[0]), base


def check_sort_nms(got, keep, boxes, scores, tag=3):
    """Exact ids, boxes, scores, tags and count; output rows outside the appended range untouched.  Returns an error string
    or None."""
    oi, ob, os_, ot, cnt, base = got
    k = len(keep)
    if cnt != base + k:
        return "out_count %d, expected %d" % (cnt, base + k)
    if oi[base:base + k].tolist() != keep:
        bad = next(i for i, (a, b) in enumerate(zip(oi[base:base + k].tolist(), keep)) if a != b)
        return "index list differs at %d: %s vs %s" % (bad, oi[base + bad:base + bad + 4].tolist(), keep[bad:bad + 4])
    kt = torch.as_tensor(keep, dtype=torch.int64)
    if not (torch.equal(ob[base:base + k], boxes[kt]) and torch.equal(os_[base:base + k], scores[kt])):
        return "boxes / scores differ"
    if not bool((ot[base:base + k] == tag).all()):
        return "tags differ"
    for t, sentinel in ((oi, -7), (ob, -7.0), (os_, -7.0), (ot, -7)):
        if not (bool((t[:base] == sentinel).all()) and bool((t[base + k:] == sentinel).all())):
            return "rows outside the appended range were written"
    return None


# ---- segmented NMS ---------------------------------------------------------------------------------------------------------
def segmented_scene(batch, ncls, n_max, counts, seed):
    """boxes [batch*n_max][ncls][4], scores [batch*n_max][ncls]: class columns with different tie / geometry structures."""
    g = torch.Generator().manual_seed(seed)
    boxes = torch.zeros(batch * n_max, ncls, 4)
    scores = torch.zeros(batch * n_max, ncls)
    for b in range(batch):
        for j in range(ncls):
            kind = SCORE_KINDS[(b + 2 * j) % len(SCORE_KINDS)]
            s, _ = make_scores(kind, n_max, g)
            geom = GEOMETRIES[(3 * b + j) % 5]          # iou_edges needs its own thresholds
            scores[b * n_max:(b + 1) * n_max, j] = s.abs() * 0.9 + 0.05 if kind != "pm_zero" else s
            boxes[b * n_max:(b + 1) * n_max, j] = make_boxes(geom, scores[b * n_max:(b + 1) * n_max, j], g)
    return boxes, scores, torch.tensor(counts, dtype=torch.int32)


def segmented_expected(boxes, scores, counts, batch, n_max, ncls, min_score, thresh, max_keep):
    """Per image: [(kept row index, class)] in block order (class 1's survivors, then class 2's, ...)."""
    out = []
    for b in range(batch):
        rows = []
        for j in range(1, ncls):
            keep = nms_expected(boxes[b * n_max:(b + 1) * n_max, j], scores[b * n_max:(b + 1) * n_max, j], int(counts[b]), n_max,
                                min_score, thresh, max_keep)
            rows += [(i, j) for i in keep]
        out.append(rows)
    return out


def check_segmented(ob, os_, blk, expected, boxes, scores, n_max, cap):
    B = len(expected)
    if not (bool((ob[B:] == -7).all()) and bool((os_[B:] == -7).all()) and bool((blk[B:] == -7).all())):
        return "written past the last image's block"
    for b, rows in enumerate(expected):
        k = len(rows)
        if int(blk[b, 0]) != k:
            return "image %d: count %d, expected %d" % (b, int(blk[b, 0]), k)
        if blk[b, 1:1 + k].tolist() != [j for _, j in rows]:
            return "image %d: labels differ" % b
        r = torch.as_tensor([b * n_max + i for i, _ in rows], dtype=torch.int64)
        c = torch.as_tensor([j for _, j in rows], dtype=torch.int64)
        if k and not (torch.equal(ob[b, :k], boxes[r, c]) and torch.equal(os_[b, :k], scores[r, c])):
            return "image %d: boxes / scores differ" % b
        if not bool((os_[b, k:] == -1).all()):
            return "image %d: the tail past the count is not -1" % b
        if not (bool((ob[b, k:] == -7).all()) and bool((blk[b, 1 + k:] == -7).all())):
            return "image %d: rows past the count were written" % b
    return None


def run_segmented(ops, dev, boxes, scores, counts, batch, n_max, ncls, min_score, thresh, max_keep, cap):
    """The outputs have one more image than the call sees: a block written past its capacity lands there (and fails the
    comparison) instead of past the allocation."""
    ob = torch.full((batch + 1, cap, 4), -7.0, device=dev)
    os_ = torch.full((batch + 1, cap), -7.0, device=dev)
    blk = torch.full((batch + 1, 1 + cap), -7, dtype=torch.int32, device=dev)
    ops.sort_nms_segmented(boxes.to(dev), scores.to(dev), counts.to(dev), batch, ncls, min_score, thresh, max_keep, ob[:batch],
                           os_[:batch], blk[:batch])
    return ob.cpu(), os_.cpu(), blk.cpu()


# ---- the tables (GPU and host runs) ---------------------------------------------------------------------------------------
def sort_nms_table(ops_, dev, n_values, extra=(-1.0, 0.0, 1.0), max_keeps=max_keep_values, stop_at_first=False):
    """Runs the sort + NMS table (thresh 1.0 only up to n_max 1186); returns (calls, failures [(case, thresh, max_keep,
    error)])."""
    calls, failures = 0, []
    for case in sort_nms_cases(n_values):
        boxes, scores, min_score, thresholds = sort_nms_scene(case)
        for thresh in thresholds + tuple(t for t in extra if t != 1.0 or case["n_max"] <= SHARED_MASK_LIMIT + 1):
            full = nms_expected(boxes, scores, case["count"], case["n_max"], min_score, thresh, 1 << 30)
            if case["n_max"] <= SHARED_MASK_LIMIT + 1 or case["geom"] == "iou_edges":
                iou_disagreements(case["name"], boxes, scores, case["count"], case["n_max"], min_score, thresh)
            for max_keep in max_keeps(len(full)):
                got = run_sort_nms(ops_, dev, boxes, scores, case["count"], case["n_max"], min_score, thresh, max_keep,
                                      case["strided"])
                calls += 1
                err = check_sort_nms(got, full[:max_keep], boxes, scores)
                if err:
                    failures.append((case["name"], thresh, max_keep, err))
                    if stop_at_first:
                        return calls, failures
    return calls, failures


def segmented_table(ops_, dev, combos, stop_at_first=False):
    calls, failures = 0, []
    for ci, (batch, ncls, n_max) in enumerate(combos):
        counts = [(n_max, 0, n_max + 9, n_max // 2, 1)[(b + ci) % 5] for b in range(batch)]
        boxes, scores, cnt = segmented_scene(batch, ncls, n_max, counts, 500 + ci)
        for max_keep in (0, 5, n_max):
            full = segmented_expected(boxes, scores, cnt, batch, n_max, ncls, -1.0, 0.5, max_keep)
            exact = (ncls - 1) * min(max_keep, n_max)
            for cap in (exact, exact + 17):
                if cap == 0:
                    continue
                ob, os_, blk = run_segmented(ops_, dev, boxes, scores, cnt, batch, n_max, ncls, -1.0, 0.5, max_keep, cap)
                calls += 1
                err = check_segmented(ob, os_, blk, full, boxes, scores, n_max, cap)
                if err:
                    failures.append(((batch, ncls, n_max, max_keep, cap), err))
                    if stop_at_first:
                        return calls, failures
    return calls, failures


# ---- RPN ---------------------------------------------------------------------------------------------------------------------
def _rpn_cfg(pre, post, fpn_post, nms_thresh, min_size, strides, sizes, amodal):
    from siammot_b200.config import get_cfg
    cfg = get_cfg()
    R = cfg.MODEL.RPN
    R.PRE_NMS_TOP_N_TEST, R.POST_NMS_TOP_N_TEST, R.FPN_POST_NMS_TOP_N_TEST = pre, post, fpn_post
    R.NMS_THRESH, R.MIN_SIZE = nms_thresh, min_size
    R.ANCHOR_STRIDE, R.ANCHOR_SIZES = tuple(strides), tuple(sizes)
    cfg.INPUT.AMODAL = amodal
    return cfg


def rpn_reference(cfg, logits_l, deltas_l, img_w, img_h):
    """oracle.rpn_select, restated so that each output row also carries its logit, anchor and deltas; asserts that the
    restatement's boxes and scores equal the oracle's bit for bit.  Returns boxes, scores, logits, anchors, deltas."""
    from oracle import siammot_oracle as orc
    R = cfg.MODEL.RPN
    per_level = []
    for lvl, (logits, deltas) in enumerate(zip(logits_l, deltas_l)):
        _, A, H, W = logits.shape
        logit = logits[0].permute(1, 2, 0).reshape(-1)
        reg = deltas[0].view(A, 4, H, W).permute(2, 3, 0, 1).reshape(-1, 4)
        k = min(R.PRE_NMS_TOP_N_TEST, logit.numel())
        idx = torch.sort(logit, descending=True, stable=True)[1][:k]
        obj = logit[idx].sigmoid()
        cell = prims.cell_anchors(R.ANCHOR_STRIDE[lvl], (R.ANCHOR_SIZES[lvl],), R.ASPECT_RATIOS)
        anchors = prims.grid_anchors(cell, R.ANCHOR_STRIDE[lvl], H, W)[idx]
        prop = prims.box_decode(reg[idx], anchors, (1.0, 1.0, 1.0, 1.0))
        if not cfg.INPUT.AMODAL:
            prop = prims.clip_boxes(prop, img_w, img_h)
        keep = prims.remove_small_mask(prop, R.MIN_SIZE).nonzero().squeeze(1)
        keep = keep[prims.nms_legacy(prop[keep], obj[keep], R.NMS_THRESH)[:R.POST_NMS_TOP_N_TEST]]
        per_level.append((prop[keep], obj[keep], logit[idx][keep], anchors[keep], reg[idx][keep]))
    cat = [torch.cat([p[i] for p in per_level]) for i in range(5)]
    k = min(R.FPN_POST_NMS_TOP_N_TEST, cat[1].numel())
    inds = torch.sort(cat[1], descending=True, stable=True)[1][:k]
    out = [c[inds] for c in cat]
    ob, os_ = orc.rpn_select(cfg, logits_l, deltas_l, img_w, img_h)
    assert torch.equal(ob, out[0]) and torch.equal(os_, out[1]), "rpn_reference no longer restates oracle.rpn_select"
    return out


def sigmoid_bound(x):
    x = x.double()
    e = torch.exp(-x)
    s = 1.0 / (1.0 + e)
    return s, s * (4 * U * e / (1 + e) + 2 * U) * SAFE + TINY


def _decode_bound(d, a, weights, img_w, img_h, amodal):
    """Float64 decode of fp32 deltas d [n, 4] on fp32 boxes a [n, 4] and the per-coordinate bound of the fp32 kernel
    (module docstring).  Returns (boxes64 [n, 4], bound [n, 4])."""
    d, a = d.double(), a.double()
    wx, wy, ww, wh = (float(np.float32(w)) for w in weights)
    out, bnd = torch.zeros(d.shape[0], 4, dtype=torch.float64), torch.zeros(d.shape[0], 4, dtype=torch.float64)
    for axis, (wc, ws) in enumerate(((wx, ww), (wy, wh))):
        lo, hi = a[:, axis], a[:, axis + 2]
        t = hi - lo
        w = t + 1
        e_w = U * t.abs() + U * w.abs()
        c = lo + 0.5 * w
        e_c = U * c.abs() + 0.5 * e_w
        dc = d[:, axis] / wc
        e_dc = U * dc.abs() if wc != 1.0 else torch.zeros_like(dc)
        dsz = d[:, axis + 2] / ws
        e_dsz = U * dsz.abs() if ws != 1.0 else torch.zeros_like(dsz)
        dsz = torch.clamp(dsz, max=CLIP)
        E = torch.exp(dsz)
        e_E = E * e_dsz + 4 * U * E + TINY
        pw = E * w
        e_pw = U * pw.abs() + E * e_w + w.abs() * e_E
        dw_ = dc * w
        pc = dw_ + c
        e_pc = U * dw_.abs() + dc.abs() * e_w + w.abs() * e_dc + U * pc.abs() + e_c
        x1 = pc - 0.5 * pw
        x2 = pc + 0.5 * pw - 1
        e1 = U * x1.abs() + e_pc + 0.5 * e_pw
        e2 = U * (pc + 0.5 * pw).abs() + U * x2.abs() + e_pc + 0.5 * e_pw
        if not amodal:
            lim = (img_w if axis == 0 else img_h) - 1.0
            x1, x2 = x1.clamp(0, lim), x2.clamp(0, lim)
        out[:, axis], out[:, axis + 2] = x1, x2
        bnd[:, axis], bnd[:, axis + 2] = e1 * SAFE + TINY, e2 * SAFE + TINY
    return out, bnd


def rpn_level_heads(spec, g):
    """One image's levels from a case spec: [(H, W, logit kind)], shared A = 3.  Returns logits_l (1,A,H,W), deltas_l
    (1,4A,H,W) and the NHWC heads (1,H,W,16)."""
    A = 3
    logits_l, deltas_l, heads = [], [], []
    for lvl, (H, W, kind) in enumerate(spec["levels"]):
        n = H * W * A
        lg = torch.round(torch.randn(n, generator=g) * 16) / 8          # quantized: distinct sigmoids are far apart
        if kind == "all_equal":
            lg[:] = 0.75
        elif kind == "straddle":                                        # equal logits across the top-k cut
            top = min(spec["pre"], n)
            order = torch.sort(lg, descending=True, stable=True)[1]
            lo, hi = max(top // 2, 0), min(top + top // 2 + 3, n)
            lg[order[lo:hi]] = float(lg[order[lo]])
        elif kind == "pm_zero":                                         # the top k are signed zeros: the index decides
            lg = torch.tensor([0.0, -0.0, 0.0, -0.0, -1.0, -2.0])[torch.randint(0, 6, (n,), generator=g)]
        elif kind == "saturated":                                       # sigmoid(30) = sigmoid(31) = sigmoid(40) = 1 in fp32
            lg = torch.tensor([30.0, 31.0, 40.0, -30.0, -31.0, 2.0])[torch.randint(0, 6, (n,), generator=g)]
        elif kind == "level_ties":                                      # few values: exact score ties across levels
            lg = torch.tensor([1.5, 1.0, 0.5, -0.5])[torch.randint(0, 4, (n,), generator=g)]
        dl = torch.round(torch.randn(n, 4, generator=g) * 8) / 16
        if spec.get("extreme"):                                         # past the clip / exp underflow
            pick = torch.randint(0, 8, (n, 4), generator=g)
            dl = torch.where(pick == 0, torch.full_like(dl, 6.0), torch.where(pick == 1, torch.full_like(dl, -60.0), dl))
        if spec.get("exact_min_size"):                                  # every third anchor decodes to itself exactly
            dl[::3] = 0.0
        # (h, w, a) flat order -> NCHW logits / A x 4 delta channels
        logits_l.append(lg.view(H, W, A).permute(2, 0, 1).unsqueeze(0).contiguous())
        deltas_l.append(dl.view(H, W, A, 4).permute(2, 3, 0, 1).reshape(1, 4 * A, H, W).contiguous())
        head = torch.zeros(1, H, W, 16)
        head[..., :A] = lg.view(1, H, W, A)
        head[..., A:5 * A] = dl.view(1, H, W, 4 * A)
        heads.append(head)
    return logits_l, deltas_l, heads


STRIDES, SIZES = (4, 8, 16, 32, 64), (32, 64, 128, 256, 512)


def rpn_cells(nlev):
    return [prims.cell_anchors(STRIDES[l], (SIZES[l],), (0.5, 1.0, 2.0)) for l in range(nlev)]


def rpn_cases(big=True):
    """RPN specs.  Level shapes (A = 3): 56x64 = 10752 anchors (one chunk), 15x239 = 10755 (a second chunk of 3), 1x1,
    224x320 = 20 chunks (shared-memory merge), 224x336 = 21 chunks (global-memory merge)."""
    one, two, tiny = (56, 64), (15, 239), (1, 1)
    c20, c21 = (224, 320), (224, 336)
    cases = [
        dict(name="one-chunk-distinct", levels=[one + ("random",), tiny + ("random",)], pre=1000, post=300, fpn=300),
        dict(name="chunk+3-straddle", levels=[two + ("straddle",), one + ("straddle",), tiny + ("random",)], pre=1000, post=800, fpn=2000),
        dict(name="pm-zero", levels=[two + ("pm_zero",), one + ("pm_zero",), tiny + ("pm_zero",)], pre=1000, post=300, fpn=500),
        dict(name="pm-zero-top1", levels=[one + ("pm_zero",), tiny + ("pm_zero",)], pre=1, post=1, fpn=2),
        dict(name="saturated-extreme", levels=[two + ("saturated",), one + ("saturated",)], pre=1024, post=800, fpn=1000, extreme=True),
        dict(name="level-ties-min-size", levels=[one + ("level_ties",), two + ("level_ties",), (30, 40, "level_ties"), tiny + ("level_ties",)],
             pre=1024, post=700, fpn=100, exact_min_size=True, min_size="anchor"),
        dict(name="amodal-extreme", levels=[one + ("random",), two + ("straddle",)], pre=1000, post=400, fpn=3000, extreme=True, amodal=True),
        dict(name="top1-ties", levels=[one + ("level_ties",), two + ("level_ties",), tiny + ("level_ties",)], pre=1, post=1, fpn=1),
    ]
    if big:
        cases += [
            dict(name="20-chunks-straddle", levels=[c20 + ("straddle",), one + ("random",), tiny + ("random",)], pre=1000, post=600, fpn=1000),
            dict(name="21-chunks-all-equal", levels=[c21 + ("all_equal",), two + ("level_ties",), tiny + ("random",)], pre=1024, post=800, fpn=5000),
            dict(name="21-chunks-pm-zero", levels=[c21 + ("pm_zero",), tiny + ("pm_zero",)], pre=1000, post=1000, fpn=800, extreme=True),
        ]
    for c in cases:
        c.setdefault("nms", 0.7)
        c.setdefault("amodal", False)
        c.setdefault("img", (700, 1000) if c["amodal"] else (333, 517))   # smaller than the anchor grids: boxes clip
    return cases


def rpn_min_size(spec):
    if spec.get("min_size") == "anchor":    # the width + 1 of the 1:1 anchor of level 0: those boxes sit exactly on the limit
        a = rpn_cells(1)[0][1]
        return float(a[2] - a[0] + 1)
    return 0.0


def rpn_case_reference(spec, logits_l, deltas_l):
    nlev = len(logits_l)
    img_w, img_h = spec["img"]
    cfg = _rpn_cfg(spec["pre"], spec["post"], spec["fpn"], spec["nms"], rpn_min_size(spec), STRIDES[:nlev], SIZES[:nlev],
                   spec["amodal"])
    return rpn_reference(cfg, logits_l, deltas_l, img_w, img_h)


def check_rpn(spec, ob, os_, cnt, ref):
    """Count exact; row r's score and box within the derived bounds of the reference's row r, which fixes the order (rows
    swapped across a tie show up as boxes far outside their bounds).  Returns (error or None, worst score |err|/bound,
    worst box |err|/bound)."""
    rb, rs, rlogit, ranchor, rdelta = ref
    k = rs.numel()
    if cnt != k:
        return "count %d, expected %d" % (cnt, k), 0.0, 0.0
    s64, sb = sigmoid_bound(rlogit)
    serr = (os_[:k].double() - s64).abs() / sb
    b64, bb = _decode_bound(rdelta, ranchor, (1.0, 1.0, 1.0, 1.0), spec["img"][0], spec["img"][1], spec["amodal"])
    berr = (ob[:k].double() - b64).abs() / bb
    ws = float(serr.max()) if k else 0.0
    wb = float(berr.max()) if k else 0.0
    if ws > 1.0:
        i = int(serr.argmax())
        return "score %d: %r vs %r (bound %.3g)" % (i, float(os_[i]), float(s64[i]), float(sb[i])), ws, wb
    if wb > 1.0:
        i = int(berr.max(1).values.argmax())
        return "box %d: %s vs %s" % (i, ob[i].tolist(), b64[i].tolist()), ws, wb
    return None, ws, wb


# ---- box decode --------------------------------------------------------------------------------------------------------------
def box_decode_scene(n, ncls, ld, seed, img_w=320, img_h=192):
    """head [n, ld] (logits spread +-80, deltas past the clip), rois partly outside the image and zero-width rows."""
    g = torch.Generator().manual_seed(seed)
    head = torch.full((n, ld), 123.0)
    lg = torch.randn(n, ncls, generator=g) * 3
    spread = torch.rand(n, generator=g) < 0.5
    lg[spread] = (torch.rand(int(spread.sum()), ncls, generator=g) * 160 - 80)
    head[:, :ncls] = lg
    d = torch.randn(n, 4 * ncls, generator=g) * 2
    d[::4, 2::4] = 30.0             # dw / ww = 6 > CLIP
    d[1::4, 3::4] = 25.0
    d[2::4, 2::4] = -400.0          # exp underflows to 0
    head[:, ncls:5 * ncls] = d
    xy = torch.rand(n, 2, generator=g) * torch.tensor([img_w * 1.4, img_h * 1.4]) - torch.tensor([img_w * 0.2, img_h * 0.2])
    wh = torch.rand(n, 2, generator=g) * 150
    rois = torch.cat([xy, xy + wh], 1)
    rois[::5, 2] = rois[::5, 0] - 1     # zero width
    return head, rois


def softmax_bound(lg):
    lg = lg.double()
    m = lg.max(1, keepdim=True).values
    t = lg - m
    e = torch.exp(t)
    den = e.sum(1, keepdim=True)
    p = e / den
    e_e = e * (U * t.abs() + 4 * U) + TINY
    ncls = lg.shape[1]
    e_den = e_e.sum(1, keepdim=True) + (ncls - 1) * U * den
    e_p = U * p + e_e / den + p * e_den / den + TINY
    return p, e_p * SAFE


def box_decode_expected(head, rois, ncls, weights, img_w, img_h, amodal, labels=None):
    """Float64 (scores [n, ncls], score bound, boxes [n, ncls, 4], box bound)."""
    n = head.shape[0]
    p, pb = softmax_bound(head[:, :ncls])
    if labels is not None:
        lab = labels.long()
        q = torch.zeros_like(p)
        qb = torch.zeros_like(pb)
        ar = torch.arange(n)
        q[ar, lab] = p[ar, lab] + 1.0
        qb[ar, lab] = pb[ar, lab] + U * (p[ar, lab] + 1.0) * SAFE
        p, pb = q, qb
    d = head[:, ncls:5 * ncls].reshape(n * ncls, 4)
    a = rois.repeat_interleave(ncls, 0)
    b, bb = _decode_bound(d, a, weights, img_w, img_h, amodal)
    return p, pb, b.view(n, ncls, 4), bb.view(n, ncls, 4)


# ---- host stand-in for siammot_b200.ops over the CPU build of csrc/select_nms.cu ---------------------------------------------
class CpuOps:
    """The siammot_b200.ops entry points this module uses, calling the host build of select_nms.cu (the same C ABI) on CPU
    tensors."""

    def __init__(self, path):
        from siammot_b200._lib import RpnLevel
        self.lib = C.CDLL(path)
        vp, i, f, sz = C.c_void_p, C.c_int, C.c_float, C.c_size_t
        sigs = {
            "smot_sort_nms": [vp, i, vp, i, vp, i, f, f, i, i, vp, vp, vp, vp, vp, vp, sz, vp],
            "smot_sort_nms_segmented": [vp, vp, vp, i, i, i, f, f, i, i, vp, vp, vp, vp, sz, vp],
            "smot_rpn_select": [C.POINTER(RpnLevel), i, i, i, f, f, i, i, i, i, vp, vp, vp, vp, sz, vp],
            "smot_rpn_select_batched": [C.POINTER(RpnLevel), vp, i, i, i, i, f, f, i, i, i, i, vp, vp, vp, vp, sz, vp],
        }
        for name, args in sigs.items():
            getattr(self.lib, name).argtypes = args
            getattr(self.lib, name).restype = i
        for name, args in (("smot_sort_nms_workspace", [i]), ("smot_sort_nms_segmented_workspace", [i, i, i]),
                           ("smot_rpn_select_workspace", [i, i]), ("smot_rpn_select_batched_workspace", [i, i, i])):
            getattr(self.lib, name).argtypes = args
            getattr(self.lib, name).restype = sz
        self.lib.cpu_last_error.restype = C.c_char_p

    def launches(self):
        return self.lib.cpu_launch_count()

    def _check(self, rc, what):
        if rc != 0:
            raise RuntimeError("%s failed (code %d): %s" % (what, rc, self.lib.cpu_last_error().decode()))

    @staticmethod
    def _p(t):
        return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)

    def sort_nms(self, boxes, scores, out_count, n_max=None, count=None, min_score=-1e30, thresh=0.5, max_keep=None, tag=0,
                 out_index=None, out_boxes=None, out_scores=None, out_tag=None, workspace=None, box_stride=4, score_stride=1):
        n_max = scores.shape[0] if n_max is None else n_max
        max_keep = n_max if max_keep is None else max_keep
        ws = torch.empty(max(self.lib.smot_sort_nms_workspace(n_max), 8), dtype=torch.uint8)
        p = self._p
        self._check(self.lib.smot_sort_nms(p(boxes), box_stride, p(scores), score_stride, p(count), n_max, min_score, thresh,
                                           max_keep, tag, p(out_index), p(out_boxes), p(out_scores), p(out_tag), p(out_count),
                                           p(ws), ws.numel(), None), "smot_sort_nms")

    def sort_nms_segmented(self, boxes, scores, count, batch, ncls, min_score, thresh, max_keep, out_boxes, out_scores,
                           out_block, workspace=None):
        n = boxes.shape[0] // batch
        ws = torch.empty(max(self.lib.smot_sort_nms_segmented_workspace(batch, ncls, n), 8), dtype=torch.uint8)
        p = self._p
        self._check(self.lib.smot_sort_nms_segmented(p(boxes), p(scores), p(count), batch, n, ncls, min_score, thresh, max_keep,
                                                     out_scores.shape[1], p(out_boxes), p(out_scores), p(out_block), p(ws),
                                                     ws.numel(), None), "smot_sort_nms_segmented")

    def rpn_levels(self, heads, strides, cell_anchors):
        from siammot_b200 import ops
        return ops.rpn_levels(heads, strides, cell_anchors)

    def rpn_select_workspace(self, num_levels, pre, device=None):
        return torch.empty(self.lib.smot_rpn_select_workspace(num_levels, pre), dtype=torch.uint8)

    def rpn_select_batched_workspace(self, num_levels, pre, batch, device=None):
        return torch.empty(self.lib.smot_rpn_select_batched_workspace(num_levels, pre, batch), dtype=torch.uint8)

    def rpn_select(self, levels, pre, post, nms_thresh, min_size, fpn_post, img_w, img_h, amodal, out_boxes, out_scores,
                   out_count, workspace):
        p = self._p
        self._check(self.lib.smot_rpn_select(levels, len(levels), pre, post, nms_thresh, float(min_size), fpn_post, img_w, img_h,
                                             int(amodal), p(out_boxes), p(out_scores), p(out_count), p(workspace),
                                             workspace.numel(), None), "smot_rpn_select")

    def rpn_select_batched(self, heads, levels, pre, post, nms_thresh, min_size, fpn_post, img_w, img_h, amodal, out_boxes,
                           out_scores, out_count, workspace):
        from siammot_b200 import ops
        p = self._p
        self._check(self.lib.smot_rpn_select_batched(levels, ops.image_strides(heads), heads[0].shape[0], len(levels), pre, post,
                                                     nms_thresh, float(min_size), fpn_post, img_w, img_h, int(amodal),
                                                     p(out_boxes), p(out_scores), p(out_count), p(workspace), workspace.numel(),
                                                     None), "smot_rpn_select_batched")


def run_rpn(ops, dev, spec, heads, batched=False):
    """smot_rpn_select (one image: heads (1,H,W,16)) or smot_rpn_select_batched (heads (B,H,W,16)).  Returns host
    (boxes [B, fpn, 4], scores [B, fpn], count [B])."""
    nlev = len(heads)
    B = heads[0].shape[0]
    dheads = [h.to(dev).contiguous() for h in heads]
    levels = ops.rpn_levels(dheads, STRIDES[:nlev], rpn_cells(nlev))
    fpn = spec["fpn"]
    ob = torch.full((B, fpn, 4), -7.0, device=dev)
    os_ = torch.full((B, fpn), -7.0, device=dev)
    oc = torch.zeros((B,), dtype=torch.int32, device=dev)
    args = (spec["pre"], spec["post"], spec["nms"], rpn_min_size(spec), fpn, spec["img"][0], spec["img"][1], spec["amodal"])
    if batched:
        ws = ops.rpn_select_batched_workspace(nlev, spec["pre"], B, dev)
        ops.rpn_select_batched(dheads, levels, *args, ob, os_, oc, ws)
    else:
        ws = ops.rpn_select_workspace(nlev, spec["pre"], dev)
        ops.rpn_select(levels, *args, ob[0], os_[0], oc, ws)
    return ob.cpu(), os_.cpu(), oc.cpu()


def rpn_image(spec, seed):
    g = torch.Generator().manual_seed(seed)
    return rpn_level_heads(spec, g)

