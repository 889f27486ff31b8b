"""tests/launch_check.py without a GPU: the step-by-step checker walks the fp32 launch lists of the benchmarked geometry
(704x1280) built over host buffers, with the C-ABI emulation (tests/cabi_emulator.py) doing the launches, and its conv bound
flags the ways a convolution kernel actually goes wrong while passing clean fp16 results."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import launch_check as lc

H, W = 704, 1280


def _model(monkeypatch, track_on=True, batched=False):
    import batched_emulator
    import cabi_emulator
    import fp16_scene
    from siammot_b200.modelling import build_siammot
    fake = batched_emulator.install(monkeypatch) if batched else cabi_emulator.install(monkeypatch)
    scene = fp16_scene.build_scene(1, 2, 3)
    cfg = scene["cfg"].clone()
    cfg.DTYPE = "float32"
    if not track_on:
        cfg.merge_from_list(["MODEL.TRACK_ON", False])
    model = build_siammot(cfg)
    model.load_state_dict(scene["sd"], strict=False)
    model.eval()
    return model, model.engine(), fake, scene


def _walk(name, steps, fake):
    recs = lc.check_steps(steps, lc.Memory("cpu"), lib=fake)
    head, expected, text = lc.report(name, steps, recs)
    print(text)
    assert sum(r["checked"] for r in recs) == expected
    assert all(r["checked"] or r["tag"] in lc.HOST_STEPS for r in recs)
    return recs


def test_static_and_track_plans_decode_and_pass(monkeypatch):
    model, eng, fake, scene = _model(monkeypatch)
    clip = scene["clip"]
    P = eng.plan(H, W)
    P.img_in.copy_(clip[0])
    recs = _walk("fp32 plan(704, 1280)", P.steps, fake)
    assert sum(r["entry"] == "smot_conv2d" for r in recs) >= 50
    assert [r["tag"] for r in recs if not r["checked"]] == ["det_init"]
    pool = model.roi_heads.track.track_pool
    import fp16_scene
    table = fp16_scene.track_table(80, H, W).numpy()
    for n in (0, 1, 30, 80):
        pool.reset()
        ids = np.array([pool.start_track() for _ in range(n)], dtype=np.int64)
        mem = model.roi_heads._build_memory(P, table[:n], ids, np.ones(n, dtype=np.int64))
        tp = eng.track_plan(P, n)
        if n:
            tp.tmpl.copy_(mem.feat.view(tp.tmpl.shape))
        recs = _walk("fp32 track plan n=%d" % n, tp.steps, fake)
        entries = {r["entry"] for r in recs}
        assert {"smot_track_combine", "smot_sort_nms"} <= entries
        if n:
            assert {"smot_roi_align", "smot_xcorr", "smot_groupnorm_relu", "smot_emm_decode", "smot_box_decode"} <= entries


def test_pair_plan_decodes_and_passes(monkeypatch):
    model, eng, fake, scene = _model(monkeypatch)
    PP = eng.pair_plan(H, W, 0)
    PP.img_batch[0].copy_(scene["clip"][0])
    PP.img_batch[1].copy_(scene["clip"][1])
    recs = _walk("fp32 pair_plan(704, 1280)", PP.steps, fake)
    assert all(r["conv"].startswith("b2 ") for r in recs if r["conv"])
    F0 = PP.frames[1]
    _walk("fp32 pair frame 1 tail", F0.steps[F0.split_index():], fake)


def test_batch_plan_decodes_and_passes(monkeypatch):
    model, eng, fake, scene = _model(monkeypatch, track_on=False, batched=True)
    P = eng.batch_plan(H, W, 3)
    P.img_batch.copy_(scene["clip"][:3])
    recs = _walk("fp32 batch_plan(704, 1280, 3)", P.steps, fake)
    entries = {r["entry"] for r in recs}
    assert {"smot_rpn_select_batched", "smot_roi_align_batched", "smot_box_decode_batched", "smot_sort_nms_segmented"} <= entries


def test_coverage_guard_fails_on_an_unchecked_entry_point():
    def smot_new_kernel(*a):
        return 0

    with pytest.raises(AssertionError, match="no checker"):
        lc.check_steps([(smot_new_kernel, (), "new", None)], lc.Memory("cpu"))
    # the host-side lambda is the listed exception: it runs and is reported as not checked
    ran = []
    recs = lc.check_steps([(lambda st: ran.append(1), (), "det_init", None), ("fork", 2, None, None), ("join", None, None, None)],
                          lc.Memory("cpu"))
    assert ran == [1] and len(recs) == 1 and not recs[0]["checked"]


# ---- sensitivity of the conv bound: seeded faults at real plan shapes ---------------------------------------------------
# level-5 3x3 (22x40x512 -> 512, K = 4608; its last tile row of 8 is ragged: 22 = 2 x 8 + 6) and fc6 (300 rows x 6272 -> 1024)
SHAPES = {"level5": dict(H=22, W=40, Cin=512, Cout=512, k=3), "fc6": dict(H=1, W=300, Cin=6272, Cout=1024, k=1)}


class _Layer(object):
    """A fp16 conv descriptor over host buffers; residual read from a channel slice (pitch 2 Cout) of a wider buffer."""

    def __init__(self, H, W, Cin, Cout, k, seed=0):
        from siammot_b200 import _lib
        g = torch.Generator().manual_seed(seed)
        self.x = torch.randn(1, H, W, Cin, generator=g).half()
        self.w = (torch.randn(Cout, k, k, Cin, generator=g) / math.sqrt(k * k * Cin)).half()
        self.scale = 0.5 + torch.rand(Cout, generator=g)
        self.bias = 0.5 * torch.randn(Cout, generator=g)
        self.resbuf = torch.randn(1, H, W, 2 * Cout, generator=g).half()
        self.out = torch.zeros(1, H, W, Cout, dtype=torch.float16)
        d = self.d = _lib.ConvDesc()
        d.inp, d.weight, d.scale, d.bias = self.x.data_ptr(), self.w.data_ptr(), self.scale.data_ptr(), self.bias.data_ptr()
        d.residual, d.out = self.resbuf.data_ptr(), self.out.data_ptr()
        d.batch, d.H, d.W, d.Cin, d.in_ld = 1, H, W, Cin, Cin
        d.OH, d.OW, d.Cout, d.out_ld, d.res_ld = H, W, Cout, Cout, 2 * Cout
        d.KH = d.KW = k
        d.stride, d.pad, d.relu, d.in_dtype, d.out_dtype = 1, k // 2, 1, 1, 1

    def result(self, w=None, res_ld=None, bias=None, extra=None):
        """fp32 computation of the layer (optionally with a faulty operand), rounded to fp16."""
        w = self.w if w is None else w
        acc = F.conv2d(self.x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), None, 1, self.d.pad)
        if extra is not None:
            acc = acc + extra
        Cout = self.d.Cout
        res = self.resbuf[..., :Cout] if res_ld is None else \
            self.resbuf.view(-1)[:self.d.OH * self.d.OW * res_ld].view(1, self.d.OH, self.d.OW, res_ld)[..., :Cout]
        b = self.bias if bias is None else bias
        y = acc * self.scale.view(1, -1, 1, 1) + b.view(1, -1, 1, 1) + res.float().permute(0, 3, 1, 2)
        return F.relu(y).permute(0, 2, 3, 1).half()

    def check(self, y):
        return lc.check_conv(lc.Memory("cpu"), self.d, lambda: self.out.copy_(y))


def _faults(L):
    clean = L.result()
    Cout, K = L.d.Cout, L.d.KH * L.d.KW * L.d.Cin
    faults = {}
    # a ragged edge tile's last row written one pixel off
    y = clean.clone()
    if L.d.H > 1:
        y[0, L.d.H - 1, 1:] = clean[0, L.d.H - 1, :-1]
    else:
        y[0, 0, 257:] = clean[0, 0, 256:-1]
    faults["ragged_row_shift"] = y
    # one 64-channel K chunk of one tap dropped
    w = L.w.clone()
    w[:, L.d.KH // 2, L.d.KW // 2, 64:128] = 0
    faults["k_chunk_dropped"] = L.result(w=w)
    # the residual read with the output's pitch instead of its own
    faults["residual_pitch"] = L.result(res_ld=Cout)
    # the bias of one channel missing
    b = L.bias.clone()
    b[int(L.bias.abs().argmax())] = 0
    faults["bias_missing"] = L.result(bias=b)
    # split-K over 8 CTAs: one partial sum added twice
    wp = torch.zeros_like(L.w).view(Cout, K)
    wp[:, 3 * K // 8:4 * K // 8] = L.w.view(Cout, K)[:, 3 * K // 8:4 * K // 8]
    part = F.conv2d(L.x.float().permute(0, 3, 1, 2), wp.view_as(L.w).float().permute(0, 3, 1, 2), None, 1, L.d.pad)
    faults["split_k_partial_twice"] = L.result(extra=part)
    return clean, faults


@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_conv_bound_flags_seeded_faults_and_passes_clean(shape):
    L = _Layer(**SHAPES[shape])
    clean, faults = _faults(L)
    ok = L.check(clean)
    print("%s clean: max |err| %.3e, worst |err|/bound %.3f" % (shape, ok.max_err, ok.max_ratio))
    assert ok.max_ratio <= 1.0
    for name, y in faults.items():
        ck = L.check(y)
        print("%s %s: worst |err|/bound %.1f at %s" % (shape, name, ck.max_ratio, ck.where))
        assert ck.max_ratio > 1.0, "%s: fault %s not flagged" % (shape, name)


def test_ulp_matches_the_storage_types():
    r = torch.tensor([0.0, 1.0, 1.5, 2.0 ** -20, 65504.0, -3.0], dtype=torch.float64)
    assert lc.ulp(r, torch.float16).tolist() == [2.0 ** -24, 2.0 ** -10, 2.0 ** -10, 2.0 ** -24, 32.0, 2.0 ** -9]
    assert lc.ulp(r, torch.float32).tolist()[:3] == [2.0 ** -149, 2.0 ** -23, 2.0 ** -23]
    # the bound of a clean fp16 rounding is met, one ulp more is not
    x = torch.randn(1000, dtype=torch.float64)
    y = x.half().double()
    assert bool(((y - x).abs() <= lc.ulp(x, torch.float16) / 2).all())
