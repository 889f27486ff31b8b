"""Further GPU parity cases: more configuration switches, bodies and pipeline modes (plain tests, so a regression
fails the suite).  Expected outputs
come from the reference itself (tests/golden/make_golden.py, ORACLE_SCENARIOS); the CPU oracle is pinned to the same fixtures
in tests/test_oracle_golden.py."""
import pytest
import torch

from helpers import load_golden
from scenarios import ORACLE_SCENARIOS
from test_e2e_gpu import BOX_TOL, SCORE_TOL, run_engine_scenario

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", list(ORACLE_SCENARIOS))
def test_engine_fp32_matches_reference_golden_more_switches(name):
    """Two foreground classes; TRACKTOR scoring + centerness off; the AOT geometry (7x7 templates, 35x35 search windows,
    29x29 responses, PAD_PIXELS 256) -- expected outputs from the reference itself."""
    gold = load_golden(name)["frames"]
    got = run_engine_scenario(name, "float32")
    assert len(got) == len(gold)
    for t, (g, o) in enumerate(zip(gold, got)):
        assert o["boxes"].shape == g["boxes"].shape, "frame %d: %d boxes vs %d" % (t, o["boxes"].shape[0], g["boxes"].shape[0])
        assert torch.equal(o["ids"], g["ids"]), "frame %d: track ids differ" % t
        assert torch.equal(o["labels"], g["labels"])
        assert float((o["boxes"] - g["boxes"]).abs().max()) <= BOX_TOL, "frame %d boxes" % t
        assert float((o["scores"] - g["scores"]).abs().max()) <= SCORE_TOL, "frame %d scores" % t
        assert o["active"] == g["active"] and o["dormant"] == g["dormant"]


def test_track_combine_grouped_matches_its_cpu_specification():
    """The CUDA kernel against tests/cabi_emulator.py's restatement of roi_heads.py:60-84 over class-grouped tracks."""
    import ctypes as C

    import numpy as np

    import cabi_emulator as ce
    from siammot_b200 import _lib
    spec = ce.FakeLib()
    L = _lib.lib()
    rng = np.random.default_rng(0)

    def p(t):
        return C.c_void_p(t.data_ptr())

    for trial in range(40):
        n, ncap, ncls = int(rng.integers(1, 90)), int(rng.integers(0, 40)), int(rng.integers(3, 6))
        tracktor = int(rng.integers(0, 2))
        host = dict(det_boxes=torch.rand(max(ncap, 1), 4), det_scores=torch.rand(max(ncap, 1)), dec_boxes=torch.rand(n, ncls, 4),
                    dec_scores=torch.rand(n, ncls), labels=torch.tensor(rng.integers(1, ncls, n), dtype=torch.int32),
                    conf=torch.rand(n), valid=torch.tensor(rng.integers(0, 2, n), dtype=torch.int32),
                    active=torch.tensor(rng.integers(0, 2, n), dtype=torch.float32))
        out_h = dict(cb=torch.full((ncap + n, 4), 9.), cs=torch.full((ncap + n,), 9.), zc=torch.tensor([5], dtype=torch.int32),
                     perm=torch.full((n,), 7, dtype=torch.int32))
        dev = {k: v.cuda() for k, v in host.items()}
        out_d = {k: v.cuda() for k, v in out_h.items()}
        for src, out, fn in ((host, out_h, spec.smot_track_combine_grouped), (dev, out_d, L.smot_track_combine_grouped)):
            rc = fn(p(src["det_boxes"]), p(src["det_scores"]), ncap, p(src["dec_boxes"]), p(src["dec_scores"]), ncls, p(src["labels"]),
                    p(src["conf"]), p(src["valid"]), p(src["active"]), n, tracktor, p(out["cb"]), p(out["cs"]), p(out["zc"]),
                    p(out["perm"]), None)
            assert rc == 0
        torch.cuda.synchronize()
        for k in out_h:
            assert torch.equal(out_d[k].cpu(), out_h[k]), (trial, k)




@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_maxpool3x3s2_matches_torch(dtype):
    import torch.nn.functional as F
    from siammot_b200 import ops
    from test_ops_gpu import DEV, nchw, nhwc, q
    g = torch.Generator().manual_seed(5)
    for shape in ((1, 64, 352, 640), (2, 8, 7, 9), (1, 16, 1, 5)):
        x = q(torch.randn(*shape, generator=g), dtype)
        ref = F.max_pool2d(x, 3, 2, 1)
        got = ops.maxpool3x3s2(nhwc(x, dtype))
        assert torch.equal(nchw(got), ref), shape            # a max of storage-type values is exact
    # channel-slice operands (pitch > channels) on both sides
    x = q(torch.randn(1, 24, 10, 12, generator=g), dtype)
    wide_in = nhwc(x, dtype)
    wide_out = torch.zeros((1, 5, 6, 32), dtype=dtype, device=DEV)
    ops.maxpool3x3s2(wide_in[..., 8:24], out=wide_out[..., 4:20])
    assert torch.equal(nchw(wide_out[..., 4:20]), F.max_pool2d(x[:, 8:24], 3, 2, 1))
    assert float(wide_out[..., :4].abs().max()) == 0.0 and float(wide_out[..., 20:].abs().max()) == 0.0


def test_r50_body_features_match_oracle_fp32_and_fp16():
    """FPN maps of the R-50-FPN plan against the oracle (fp32: summation-order tolerance; fp16 storage: 2e-2 of the map's scale
    through 53 convolutions)."""
    from oracle.siammot_oracle import OracleSiamMOT
    from test_e2e_gpu import build_model
    for dtype, tol_ in (("float32", 1e-4), ("float16", 2e-2)):
        cfg, model, clip = build_model("emm_r50_192x320", dtype)
        eng = model.engine()
        P = eng.run_static(clip[0].to("cuda"))
        torch.cuda.synchronize()
        sd = {k: v.detach().cpu() for k, v in model.state_dict().items()}
        ref = OracleSiamMOT(cfg, sd).features(clip[0])
        for l, (got, want) in enumerate(zip(P.feats, ref)):
            got = got.permute(0, 3, 1, 2).float().cpu()
            assert got.shape == want.shape
            err = float((got - want).abs().max() / want.abs().max())
            assert err <= tol_, "%s FPN level %d: relative error %g" % (dtype, l, err)


def test_r50_fp16_tracks_close_to_reference():
    from test_e2e_gpu import run_engine_scenario
    name = "emm_r50_192x320"
    gold = load_golden(name)["frames"]
    got = run_engine_scenario(name, "float16")
    g0, o0 = gold[0], got[0]
    n = min(len(g0["ids"]), len(o0["ids"]))
    assert abs(len(g0["ids"]) - len(o0["ids"])) <= max(3, len(g0["ids"]) // 10)
    assert int((g0["ids"][:n] == o0["ids"][:n]).sum()) >= 0.8 * n


@pytest.mark.parametrize("slots", ["2", "3"])
def test_three_stage_clip_equals_frame_by_frame(slots, monkeypatch):
    """SMOT_CLIP_SPLIT=1: backbone half of frame t+1 / detection tail of frame t / track stage of frame t on three streams,
    K plan copies, one CUDA graph per half -- exactly the per-frame results, twice in a row (graph capture, then replay)."""
    from test_e2e_gpu import build_model
    name = "emm_256x384"
    monkeypatch.setenv("SMOT_CLIP_SPLIT", "0")
    cfg, model, clip = build_model(name, "float32")
    model.reset_siammot_status()
    ref = [model(f.to("cuda"))[0] for f in clip]
    monkeypatch.setenv("SMOT_CLIP_SPLIT", "1")
    monkeypatch.setenv("SMOT_CLIP_SLOTS", slots)
    cfg, model, clip = build_model(name, "float32")
    assert model.engine().clip_split and model.engine().clip_slots == int(slots)
    for _ in range(2):
        model.reset_siammot_status()
        got = model.forward_clip([f.to("cuda") for f in clip])
        torch.cuda.synchronize()
        assert len(got) == len(ref)
        for a, b in zip(ref, got):
            assert torch.equal(a.bbox, b.bbox) and torch.equal(a.get_field("ids"), b.get_field("ids"))
            assert torch.equal(a.get_field("scores"), b.get_field("scores"))


@pytest.mark.parametrize("dtype", ["float32"])
def test_tracker_plugin_contract_on_the_gpu(dtype):
    """EMM.extract_cache / EMM.forward through the SIAMESE_TRACKER registry object, against the oracle."""
    from helpers import scenario_inputs
    from siammot_b200.modelling import build_siammot
    from test_engine_emulated_cpu import _plugin_contract_check
    cfg, sd, clip = scenario_inputs("emm_256x384")
    cfg.DTYPE = dtype
    model = build_siammot(cfg)
    model.load_state_dict(sd, strict=False)
    model = model.to("cuda").eval()
    _plugin_contract_check(model, cfg, sd, clip, to_dev=lambda t: t.to("cuda"))


def test_public_detection_clip_equals_reference_golden():
    from test_engine_emulated_cpu import BOX_TOL, _given_scenario
    from siammot_b200.modelling import build_siammot
    cfg, sd, clip, given = _given_scenario()
    model = build_siammot(cfg)
    model.load_state_dict(sd, strict=False)
    model = model.to("cuda").eval()
    model.reset_siammot_status()
    gold = load_golden("given_det_192x320")["frames"]
    given = [[g[0].to("cuda")] for g in given]
    results = model.forward_clip([clip[t].to("cuda") for t in range(len(gold))], given_detections=given)
    for t, (r, g) in enumerate(zip(results, gold)):
        assert r.bbox.shape == g["boxes"].shape and torch.equal(r.get_field("ids").cpu(), g["ids"]), "frame %d" % t
        if g["boxes"].numel():
            assert float((r.bbox.cpu() - g["boxes"]).abs().max()) <= BOX_TOL


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("stride", [1, 2])
def test_deform_im2col_plus_gemm_matches_torchvision(stride, dtype):
    from torchvision.ops import deform_conv2d
    from siammot_b200 import ops
    from test_ops_gpu import DEV, nhwc, q, rel_err
    g = torch.Generator().manual_seed(stride)
    Cc, H, W, Cout = 64, 44, 80, 64
    OH, OW = (H - 1) // stride + 1, (W - 1) // stride + 1
    x = q(torch.randn(1, Cc, H, W, generator=g), dtype)
    w = q(torch.randn(Cout, Cc, 3, 3, generator=g) / 24., dtype)
    off = torch.randn(1, 18, OH, OW, generator=g) * 2.0
    ref = deform_conv2d(x, off, w, None, stride=stride, padding=1)
    offs = torch.zeros((1, OH, OW, 20), device=DEV)
    offs[..., :18] = off.permute(0, 2, 3, 1).to(DEV)
    cols = ops.deform_im2col3x3(nhwc(x, dtype), offs, stride)
    wq = w.permute(0, 2, 3, 1).reshape(Cout, 1, 1, 9 * Cc).contiguous().to(DEV, dtype)
    got = ops.conv2d(cols, wq)                                     # the deformable conv proper: a GEMM over the columns
    torch.cuda.synchronize()
    assert rel_err(got.permute(0, 3, 1, 2).float().cpu(), ref) <= (2e-5 if dtype == torch.float32 else 4e-3)


def test_frame_overlap_changes_nothing(monkeypatch):
    from test_e2e_gpu import build_model

    def run(flag):
        monkeypatch.setenv("SMOT_FRAME_OVERLAP", flag)
        cfg, model, clip = build_model("emm_256x384", "float32")
        assert model.engine().frame_overlap == (flag == "1")
        outs = []
        for _ in range(2):                                  # second pass: the per-half CUDA graphs are replayed
            model.reset_siammot_status()
            outs = [model(f.to("cuda"))[0] for f in clip]
        return outs

    for a, b in zip(run("0"), run("1")):
        assert torch.equal(a.bbox, b.bbox) and torch.equal(a.get_field("ids"), b.get_field("ids"))
        assert torch.equal(a.get_field("scores"), b.get_field("scores"))


# (kept last: the only pending cases that launch a kernel with asynchronous copies for the first time)
# ---- channel-planar search-window exchange (developer switch SMOT_XCORR_PLANAR, DESIGN.md section 5.2) -------------------


def _planar_to_nhwc(p, res, row_pitch):
    """(n, C, plane) planar windows -> (n, res, res, C)."""
    n, C, plane = p.shape
    rows = p[:, :, :res * row_pitch].reshape(n, C, res, row_pitch)[..., :res]
    return rows.permute(0, 2, 3, 1).contiguous()


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_roi_align_planar_equals_roi_align(dtype):
    """Same arithmetic, different layout: the planar variant must reproduce smot_roi_align exactly, pads untouched."""
    from siammot_b200 import _lib, ops
    from test_ops_gpu import DEV, _pyramid
    from oracle import siammot_oracle as orc
    g = torch.Generator().manual_seed(21)
    C, H, W = 128, 48, 80
    _, dfeats = _pyramid(g, C, H, W, dtype)
    scales = (0.25, 0.125, 0.0625, 0.03125)
    boxes = torch.tensor([[10., 20., 60., 150.], [100., 30., 180., 190.], [5., 5., 300., 185.], [250., 60., 290., 160.],
                          [-30., -20., 40., 50.], [0., 0., 319., 191.], [200., 100., 201., 101.], [310., 180., 400., 260.]])
    pad = 64
    sr = orc.search_region(boxes, pad, 1.0, 0)
    pads = [int(pad / ((2 ** i) * 4)) for i in range(4)]
    ref = ops.roi_align(dfeats, sr.to(DEV), scales, 30, 2, level_boxes=boxes.to(DEV), pads=pads)
    got = ops.roi_align_planar(dfeats, sr.to(DEV), scales, 30, 2, level_boxes=boxes.to(DEV), pads=pads)
    assert got.shape == (8, C, _lib.XCORR_PLANE)
    assert torch.equal(_planar_to_nhwc(got, 30, _lib.XCORR_ROW_PITCH), ref)
    mask = torch.ones(_lib.XCORR_PLANE, dtype=torch.bool)
    for r in range(30):
        mask[r * _lib.XCORR_ROW_PITCH:r * _lib.XCORR_ROW_PITCH + 30] = False
    assert float(got[:, :, mask.to(DEV)].abs().max()) == 0.0, "the planar kernel wrote outside the windows"
    # other geometry (template-sized windows, tight pitches) and the device-side count
    ref = ops.roi_align(dfeats, boxes.to(DEV), scales, 15, 2)
    got = ops.roi_align_planar(dfeats, boxes.to(DEV), scales, 15, 2, row_pitch=16, plane_pitch=15 * 16)
    assert torch.equal(_planar_to_nhwc(got, 15, 16), ref)
    cnt = torch.tensor([3], dtype=torch.int32, device=DEV)
    got = ops.roi_align_planar(dfeats, boxes.to(DEV), scales, 15, 2, count=cnt, row_pitch=16, plane_pitch=15 * 16)
    assert float(got[3:].abs().max()) == 0.0 and torch.equal(_planar_to_nhwc(got, 15, 16)[:3], ref[:3])


@pytest.mark.parametrize("n,C", [(30, 128), (3, 32), (80, 128), (5, 256)])
def test_xcorr_planar_equals_xcorr(n, C):
    """Bulk-copy staging, identical MMA phase: bit-identical to smot_xcorr on the same windows; oracle within the fp16 bar."""
    from siammot_b200 import _lib, ops
    from test_ops_gpu import DEV, nchw, nhwc, q, rel_err, tol
    from oracle import siammot_oracle as orc
    g = torch.Generator().manual_seed(n + C)
    dt = torch.float16
    x = q(torch.randn(n, C, 30, 30, generator=g), dt)
    k = q(torch.randn(n, C, 15, 15, generator=g) / 15., dt)
    dx, dk = nhwc(x, dt), nhwc(k, dt)
    xp = torch.zeros((n, C, _lib.XCORR_PLANE), dtype=dt, device=DEV)
    xp[:, :, :30 * _lib.XCORR_ROW_PITCH].view(n, C, 30, _lib.XCORR_ROW_PITCH)[..., :30] = x.to(DEV, dt)
    xp[:, :, 30 * _lib.XCORR_ROW_PITCH:] = 7.0          # the plane's 8 trailing halves are never read
    xp.view(n, C, -1)[:, :, :30 * _lib.XCORR_ROW_PITCH].view(n, C, 30, _lib.XCORR_ROW_PITCH)[..., 32:] = 7.0   # nor columns 32..39
    ref = ops.xcorr(dx, dk)
    for _ in range(3):                                   # back-to-back launches chain through PDL
        got = ops.xcorr_planar(xp, dk, mma_mode=0)       # the untrimmed MMA phase: xcorr_mma_kernel's, instruction for instruction
    torch.cuda.synchronize()
    assert torch.equal(got, ref)
    assert rel_err(nchw(got), orc.xcorr_depthwise(x, k)) <= tol(dt)
    # trimmed MMA phase (the default: SMOT_XCORR_PLANAR=2 / mma_mode 1): another accumulation order -> the oracle bar, not bit equality
    trim = ops.xcorr_planar(xp, dk, mma_mode=1)
    assert rel_err(nchw(trim), orc.xcorr_depthwise(x, k)) <= tol(dt)
    assert rel_err(trim.float(), ref.float()) <= 2e-3
    # planes per CTA (the grid's granularity) never change the bits: every plane is one warp's work in a fixed order
    # (0 = the flat form: one CTA per SM, 4-plane units dealt evenly; only while the planes fit one wave of 28 per SM)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for cg in (2, 4, 8, 16) + ((0,) if n * C <= 28 * sms else ()):
        for mode, want in ((0, ref), (1, trim)):
            out = torch.full_like(ref, float("nan"))
            for _ in range(2):
                ops.xcorr_planar(xp, dk, out=out, mma_mode=mode, channel_group=cg)
            assert torch.equal(out, want), "channel group %d, mma_mode %d" % (cg, mode)


def test_engine_planar_switch_changes_nothing(monkeypatch):
    """fp16 engine with the planar exchange and the untrimmed MMA phase (SMOT_XCORR_PLANAR=1): same boxes / scores / ids as the
    NHWC exchange (SMOT_XCORR_PLANAR=0), frame by frame and as a clip; the default (=2, trimmed MMA phase) tracks the same ids."""
    from test_e2e_gpu import build_model

    def run(flag, clip_api):
        monkeypatch.setenv("SMOT_XCORR_PLANAR", flag)
        cfg, model, clip = build_model("emm_256x384", "float16")
        assert model.engine().xcorr_planar_ok() == (flag != "0") and model.engine().xcorr_planar_mode == (0 if flag == "1" else 1)
        model.reset_siammot_status()
        frames = [f.to("cuda") for f in clip]
        return model.forward_clip(frames) if clip_api else [model(f)[0] for f in frames]

    ref = run("0", False)
    assert sum(int((r.get_field("ids") >= 0).sum()) for r in ref) > 0
    for clip_api in (False, True):
        got = run("1", clip_api)
        for a, b in zip(ref, got):
            assert torch.equal(a.bbox, b.bbox) and torch.equal(a.get_field("scores"), b.get_field("scores"))
            assert torch.equal(a.get_field("ids"), b.get_field("ids"))
    got = run("2", False)                                    # the default: fp32 accumulation in another order (fp16 ulp of the response)
    for a, b in zip(ref[:2], got[:2]):
        assert a.bbox.shape == b.bbox.shape and float((a.bbox - b.bbox).abs().max()) <= 0.5
