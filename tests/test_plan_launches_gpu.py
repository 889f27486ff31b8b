"""Every launch of the benchmarked plans, one step at a time, against float64 (tests/launch_check.py): the fp16 DLA-34-FPN + EMM
static plan at 704x1280 on a clip frame, its track plans for 0 / 1 / 30 / 80 tracks, the frame-pair and batch-3 plans, the
fp32 plan and its 30-track plan, the R-50-FPN plan and the DLA-60 DCN scenario.  Each case checks every step but the listed
host-side one and prints the per-step report.  The static plans and the 30-track plan also compare the CUDA graph's result,
buffer by buffer, with the serialised walk: kernels are deterministic and split-K factors fixed per layer, so any difference
is a race (programmatic dependent launch, parallel graph branches)."""
import ctypes
import math
import time

import numpy as np
import pytest
import torch

import fp16_scene
import launch_check as lc

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
H, W = 704, 1280


def _model(cfg, sd, dtype, track_on=True):
    from siammot_b200.modelling import build_siammot
    cfg = cfg.clone()
    cfg.DTYPE = dtype
    if not track_on:
        cfg.merge_from_list(["MODEL.TRACK_ON", False])
    model = build_siammot(cfg)
    model.load_state_dict(sd, strict=False)
    return model.to(DEV).eval()


def _walk(name, steps):
    from siammot_b200 import _lib
    t0 = time.time()
    recs = lc.check_steps(steps, lc.Memory(DEV), lib=_lib.lib(), strict=False)
    head, expected, text = lc.report(name, steps, recs)
    print(text)
    print("%s: walk %.1f s" % (name, time.time() - t0))
    bad = [r for r in recs if r["checked"] and not r["max_ratio"] <= 1.0]
    assert not bad, "steps over their bound:\n" + "\n".join(lc.format_record(r) for r in bad)
    assert sum(r["checked"] for r in recs) == expected
    assert all(r["checked"] or r["tag"] in lc.HOST_STEPS for r in recs)
    return recs


def _static_outputs(P):
    out = {"buf%d" % i: b for i, b in enumerate(P.bufs)}
    for k in ("props", "prop_scores", "prop_count", "det_boxes", "det_scores", "det_block"):
        if hasattr(P, k):
            out[k] = getattr(P, k)
    for k, v in getattr(P, "box", {}).items():
        if torch.is_tensor(v):
            out["box." + k] = v
    return out


def _track_outputs(tp):
    out = {"res": tp.res, "cat_boxes": tp.cat_boxes}
    if tp.n:
        for k in ("srp", "srf", "resp", "tower", "maps", "tb", "conf", "valid"):
            if hasattr(tp, k) and getattr(tp, k) is not None:
                out[k] = getattr(tp, k)
        for k, v in tp.box.items():
            if torch.is_tensor(v):
                out["box." + k] = v
    return out


def _assert_same(graph, walked, what):
    diff = [k for k in graph if not torch.equal(graph[k], walked[k])]
    assert not diff, "%s: the CUDA graph and the serialised walk differ in %s" % (what, diff)


def _graph_then_walk(name, run_graph, outputs, steps):
    run_graph()
    run_graph()
    torch.cuda.synchronize()
    graph = {k: v.clone() for k, v in outputs().items()}
    recs = _walk(name, steps)
    _assert_same(graph, outputs(), name)
    return recs


@pytest.fixture(scope="module")
def scene():
    return fp16_scene.build_scene(1, 2, 3, workload="720p30")


def _memories(model, P, counts, table):
    """Memories of n tracks on plan P's current features, built the way fp16_scene.run_engine builds them."""
    pool = model.roi_heads.track.track_pool
    mems = {}
    for n in counts:
        pool.reset()
        ids = np.array([pool.start_track() for _ in range(n)], dtype=np.int64)
        mems[n] = model.roi_heads._build_memory(P, table[:n], ids, np.ones(n, dtype=np.int64))
    return mems


def _stage(eng, P, mem, n):
    tp = eng.track_plan(P, n)
    if n:
        mem.stage(tp)
        tp.staged_mem = mem
        tp.inputs.copy_(tp.inputs_host)
        tp.tmpl.copy_(mem.feat.view(tp.tmpl.shape))
    torch.cuda.synchronize()
    return tp


def _static_and_tracks(scene, dtype, counts, graph_n):
    model = _model(scene["cfg"], scene["sd"], dtype)
    eng = model.engine()
    clip = scene["clip"]
    P = eng.plan(H, W)
    P.img_in.copy_(clip[0].to(DEV))
    recs = _graph_then_walk("%s plan(704, 1280)" % dtype, P.run, lambda: _static_outputs(P), P.steps)
    assert sum(r["entry"] == "smot_conv2d" for r in recs) >= 50
    # the memory from frame 0, the track stage on frame 1 (the same plan: the templates live in their own tensors)
    mems = _memories(model, P, counts, fp16_scene.track_table(max(counts), H, W).numpy())
    P.img_in.copy_(clip[1].to(DEV))
    P.run()
    torch.cuda.synchronize()
    for n in counts:
        tp, mem = _stage(eng, P, mems[n], n), mems[n]
        name = "%s track plan n=%d" % (dtype, n)
        if n == graph_n:
            recs = _graph_then_walk(name, lambda: tp.run(mem.feat), lambda: _track_outputs(tp), tp.steps)
        else:
            recs = _walk(name, tp.steps)
        entries = {r["entry"] for r in recs}
        if n and dtype == "float16":
            assert {"smot_roi_align_planar", "smot_xcorr_planar_mode"} <= entries
        if n and dtype == "float32":
            assert {"smot_roi_align", "smot_xcorr"} <= entries


def test_fp16_static_and_track_plans(scene):
    _static_and_tracks(scene, "float16", (0, 1, 30, 80), 30)


def test_fp32_static_and_30_track_plans(scene):
    _static_and_tracks(scene, "float32", (30,), 30)


def test_fp16_pair_plan(scene):
    model = _model(scene["cfg"], scene["sd"], "float16")
    eng = model.engine()
    PP = eng.pair_plan(H, W, 0)
    PP.img_batch[0].copy_(scene["clip"][1].to(DEV))
    PP.img_batch[1].copy_(scene["clip"][2].to(DEV))
    recs = _graph_then_walk("float16 pair_plan(704, 1280)", lambda: PP.run_part(0), lambda: _static_outputs(PP), PP.steps)
    assert all(r["conv"].startswith("b2 ") for r in recs if r["conv"])
    F1 = PP.frames[1]
    _walk("float16 pair frame 1 tail", F1.steps[F1.split_index():])


def test_fp16_batch_plan(scene):
    model = _model(scene["cfg"], scene["sd"], "float16", track_on=False)
    eng = model.engine()
    P = eng.batch_plan(H, W, 3)
    P.img_batch.copy_(scene["clip"][:3].to(DEV))
    recs = _graph_then_walk("float16 batch_plan(704, 1280, 3)", P.run, lambda: _static_outputs(P), P.steps)
    assert {"smot_rpn_select_batched", "smot_roi_align_batched", "smot_box_decode_batched",
            "smot_sort_nms_segmented"} <= {r["entry"] for r in recs}


def test_fp16_r50_plan():
    sc = fp16_scene.build_scene(1, 2, 1, workload="r50_720p30")
    model = _model(sc["cfg"], sc["sd"], "float16")
    P = model.engine().plan(H, W)
    P.img_in.copy_(sc["clip"][0].to(DEV))
    recs = _graph_then_walk("float16 R-50-FPN plan(704, 1280)", P.run, lambda: _static_outputs(P), P.steps)
    assert "smot_maxpool3x3s2" in {r["entry"] for r in recs}


def test_fp16_dla60_dcn_plan():
    from helpers import scenario_inputs
    cfg, sd, clip = scenario_inputs("emm_dla60_dcn_192x320")
    model = _model(cfg, sd, "float16")
    P = model.engine().plan(clip.shape[2], clip.shape[3])
    P.img_in.copy_(clip[0].to(DEV))
    recs = _graph_then_walk("float16 DLA-60 DCN plan(%d, %d)" % (clip.shape[2], clip.shape[3]), P.run,
                            lambda: _static_outputs(P), P.steps)
    assert "smot_deform_im2col3x3" in {r["entry"] for r in recs}


# ---- the ring depths the plans do not reach: SMOT_TC_STAGES forces them (read on every call) -----------------------------
# BN is the widest N tile with tiles * Cout / BN >= 96: 88x160 is 110 tiles of 16x8, so Cout 256 -> BN 256, 128 -> 128, 64 -> 64.
# Forced depth 2 / 4 / 6 gives BN 256: 3, 4, 4; BN 128: 2, 3, 6; BN 64: 2, 4, 8 -- all 8 conv_tc_kernel<BN, STAGES>.
@pytest.mark.parametrize("cout", [256, 128, 64])
def test_forced_ring_depths_meet_the_bound(cout, monkeypatch):
    from siammot_b200 import _lib, ops
    g = torch.Generator().manual_seed(cout)
    Cin = 128
    x = torch.randn(1, 88, 160, Cin, generator=g).half().to(DEV)
    w = (torch.randn(cout, 3, 3, Cin, generator=g) / math.sqrt(9 * Cin)).half().to(DEV)
    scale = (0.5 + torch.rand(cout, generator=g)).to(DEV)
    bias = torch.randn(cout, generator=g).to(DEV)
    res = torch.randn(1, 88, 160, cout, generator=g).half().to(DEV)
    results = {}
    for st in ("2", "4", "6"):
        monkeypatch.setenv("SMOT_TC_STAGES", st)
        out = torch.zeros(1, 88, 160, cout, dtype=torch.float16, device=DEV)
        d = ops.conv_desc(x, w, out, scale, bias, res, 1, 1, True)
        assert _lib.lib().smot_conv2d_algo(ctypes.byref(d)) == _lib.CONV_TCGEN05
        ck = lc.check_conv(lc.Memory(DEV), d, lambda: (ops.conv2d(x, w, scale, bias, res, 1, 1, True, out=out),
                                                        torch.cuda.synchronize()))
        print("Cout %d, SMOT_TC_STAGES=%s: max |err| %.3e, worst |err|/bound %.3f" % (cout, st, ck.max_err, ck.max_ratio))
        assert ck.max_ratio <= 1.0, ck.where
        results[st] = out
    assert torch.equal(results["2"], results["4"]) and torch.equal(results["4"], results["6"])
