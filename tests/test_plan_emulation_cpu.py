"""Host-side wiring of the static launch plan, checked without a GPU: the plan is built over host buffers and its backbone +
FPN calls are interpreted with torch CPU ops (tests/plan_emulator.py), then compared with the oracle's FPN maps.  The DLA-34
case (whose GPU execution is validated by the e2e parity tests) validates the interpreter; the R-50-FPN case is the check of
the wiring written without GPU access."""
import pytest
import torch

from helpers import scenario_inputs
from plan_emulator import build_engine_on_host, run_backbone


@pytest.mark.parametrize("name", ["emm_amodal_expire_192x320", "emm_r50_192x320"])
def test_backbone_and_fpn_wiring_matches_oracle(name, monkeypatch):
    from oracle.siammot_oracle import OracleSiamMOT
    cfg, sd, clip = scenario_inputs(name)
    cfg.DTYPE = "float32"
    eng = build_engine_on_host(cfg, sd, monkeypatch)
    image = clip[0]
    P = eng.plan(image.shape[1], image.shape[2])
    n = run_backbone(P, image)
    assert n >= 50, n
    ref = OracleSiamMOT(cfg, sd).features(image)
    assert len(P.feats) == len(ref) == 5
    for l, (got, want) in enumerate(zip(P.feats, ref)):
        got = got.permute(0, 3, 1, 2)
        assert got.shape == want.shape, (l, got.shape, want.shape)
        err = float((got - want).abs().max() / want.abs().max())
        assert err <= 1e-4, "FPN level %d: relative error %g" % (l, err)


def test_concurrent_stages_use_disjoint_split_k_scratch(monkeypatch):
    """forward_clip runs the backbone half of frame t+1, the detection tail of frame t and the track stage of frame t on three
    streams (SMOT_CLIP_SPLIT) -- or the first two on one and the third on another (default).  The emulated convs do not touch
    the split-K scratch, so tests/stream_sim.py cannot see a conflict there: check the assignment itself."""
    import cabi_emulator
    from siammot_b200 import engine
    cabi_emulator.install(monkeypatch)          # the track plan's arena also creates events / pinned blocks
    cfg, sd, clip = scenario_inputs("emm_amodal_expire_192x320")
    cfg.DTYPE = "float32"
    eng = engine.Engine(cfg, device="cpu", use_graph=False)
    eng.load_state_dict(sd)
    P = eng.plan(clip[0].shape[1], clip[0].shape[2])
    k = P.split_index()

    def scratch(steps):
        out = set()
        for st in steps:
            if getattr(st[0], "__name__", None) == "smot_conv2d":
                out.add(st[1][0]._obj.workspace)
        return out

    backbone, tail = scratch(P.steps[:k]), scratch(P.steps[k:])
    tp = eng.track_plan(P, 5)
    track = scratch(tp.steps)
    allowed_backbone = {eng.conv_ws.data_ptr()} | {w.data_ptr() for w in eng._branch_ws.values()}
    assert backbone <= allowed_backbone and len(backbone) >= 2      # main line + parallel branches
    assert tail == {eng.conv_ws_det.data_ptr()}
    assert track == {eng.conv_ws_track.data_ptr()}
    assert not (backbone & tail) and not (backbone & track) and not (tail & track)
    # parallel branches of one fork never share scratch with each other or with the main line
    per_branch = {}
    for fn, args, tag, branch in P.steps[:k]:
        if getattr(fn, "__name__", None) == "smot_conv2d" and branch is not None:
            per_branch.setdefault(branch, set()).add(args[0]._obj.workspace)
    assert all(len(v) == 1 for v in per_branch.values())
    assert len({next(iter(v)) for v in per_branch.values()}) == len(per_branch)
    assert eng.conv_ws.data_ptr() not in {next(iter(v)) for v in per_branch.values()}
    # a frame PAIR's backbone pass (batch 2) and the detection tails of its two frame plans keep the same separation
    PP = eng.pair_plan(clip[0].shape[1], clip[0].shape[2], 0)
    assert scratch(PP.steps) <= allowed_backbone and PP.split_index() == len(PP.steps)
    for F in PP.frames:
        assert scratch(F.steps[F.split_index():]) == {eng.conv_ws_det.data_ptr()}
        assert all(a.data_ptr() == b[F.view_index:F.view_index + 1].data_ptr() for a, b in zip(F.bufs, PP.bufs))


DLA_FAMILY = {"DLA-46-C-FPN": (64, 64, 128, 256), "DLA-60-FPN": (128, 256, 512, 1024), "DLA-102-FPN": (128, 256, 512, 1024),
              "DLA-169-FPN": (128, 256, 512, 1024)}


@pytest.mark.parametrize("arch", sorted(DLA_FAMILY) + ["DLA-60-FPN+DCN", "DLA-102-FPN+DCN"])
def test_dla_family_wiring_matches_oracle(arch, monkeypatch):
    """The general concat-free DlaTree plan (bottleneck blocks, nests up to five deep, residual roots, level-2 nests) against
    the oracle, which tests/test_oracle_dla_family_cpu.py pins to the reference's own dla.py modules."""
    _check_dla_wiring(arch, monkeypatch)


def test_dla34_wiring_matches_oracle(monkeypatch):
    """DLA-34 (basic blocks, two-level nests), whose GPU execution the e2e parity tests validate, through the same builder."""
    _check_dla_wiring("DLA-34-FPN", monkeypatch)


def _check_dla_wiring(arch, monkeypatch):
    import os
    from helpers import CONFIG_DIR
    from oracle.siammot_oracle import OracleSiamMOT
    from siammot_b200.config import get_cfg
    from siammot_b200.synthetic import make_state_dict
    cfg = get_cfg()
    cfg.merge_from_file(os.path.join(CONFIG_DIR, "dla34_emm.yaml"))
    if arch.endswith("+DCN"):                      # MODEL.DLA.STAGE_WITH_DCN on levels 3..5 (the reference's "-DCN" models)
        arch = arch[:-4]
        cfg.merge_from_list(["MODEL.DLA.STAGE_WITH_DCN", (False, False, False, True, True, True)])
    stages = DLA_FAMILY.get(arch, (64, 128, 256, 512))
    cfg.merge_from_list(["MODEL.BACKBONE.CONV_BODY", arch, "MODEL.DLA.DLA_STAGE2_OUT_CHANNELS", stages[0],
                         "MODEL.DLA.DLA_STAGE3_OUT_CHANNELS", stages[1], "MODEL.DLA.DLA_STAGE4_OUT_CHANNELS", stages[2],
                         "MODEL.DLA.DLA_STAGE5_OUT_CHANNELS", stages[3]])
    cfg.DTYPE = "float32"
    sd = make_state_dict(cfg, 3)
    eng = build_engine_on_host(cfg, sd, monkeypatch)
    P = eng.plan(64, 96)
    image = torch.randn(3, 64, 96, generator=torch.Generator().manual_seed(2))
    assert run_backbone(P, image) >= 40
    ref = OracleSiamMOT(cfg, sd).features(image)
    for l, (got, want) in enumerate(zip(P.feats, ref)):
        got = got.permute(0, 3, 1, 2)
        assert got.shape == want.shape
        err = float((got - want).abs().max() / want.abs().max())
        assert err <= 1e-4, "%s FPN level %d: relative error %g" % (arch, l, err)


def test_r101_wiring_matches_oracle(monkeypatch):
    """upstream "R-101-FPN" (stage specs 3, 4, 23, 3) through the same bottleneck plan."""
    import os
    from helpers import CONFIG_DIR
    from oracle.siammot_oracle import OracleSiamMOT
    from siammot_b200.config import get_cfg
    from siammot_b200.synthetic import make_state_dict
    cfg = get_cfg()
    cfg.merge_from_file(os.path.join(CONFIG_DIR, "r50_emm.yaml"))
    cfg.merge_from_list(["MODEL.BACKBONE.CONV_BODY", "R-101-FPN"])
    cfg.DTYPE = "float32"
    sd = make_state_dict(cfg, 2)
    eng = build_engine_on_host(cfg, sd, monkeypatch)
    P = eng.plan(64, 96)
    image = torch.randn(3, 64, 96, generator=torch.Generator().manual_seed(5))
    assert run_backbone(P, image) >= 100
    for l, (got, want) in enumerate(zip(P.feats, OracleSiamMOT(cfg, sd).features(image))):
        err = float((got.permute(0, 3, 1, 2) - want).abs().max() / want.abs().max())
        assert err <= 1e-4, "R-101 FPN level %d: relative error %g" % (l, err)
