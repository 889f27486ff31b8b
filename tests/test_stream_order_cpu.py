"""Stream / event ordering of the engine's host orchestration under adversarial (but CUDA-legal) schedules, without a GPU
(tests/stream_sim.py): per-frame calls, the two-stream clip pipeline and the three-stage clip pipeline must reproduce the
reference golden whatever the interleaving; a deliberately removed edge must NOT (the detector detects)."""
import pytest
import torch

import stream_sim
from helpers import load_golden, scenario_inputs
from test_engine_emulated_cpu import _compare

POLICIES = ["lazy", "eager", "workers_eager", "default_eager", ("random", 1), ("random", 2), ("random", 3)]
NAME = "emm_amodal_expire_192x320"


def _run_sim(monkeypatch, policy, mode, env=None, sabotage=None, n_frames=None):
    from siammot_b200.modelling import build_siammot
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    sim, fake = stream_sim.install(monkeypatch, policy)
    if sabotage:
        sabotage(monkeypatch)
    cfg, sd, clip = scenario_inputs(NAME)
    cfg.DTYPE = "float32"
    model = build_siammot(cfg)
    model.load_state_dict(sd, strict=False)
    model.eval()
    model.results_on_host = True
    model.reset_siammot_status()
    pool = model.roi_heads.track.track_pool
    frames = list(clip)
    if n_frames is not None:      # a longer clip: the scenario's frames over and over (the tracks persist, slots get reused)
        frames = [frames[i % len(frames)] for i in range(n_frames)]
    states = []
    sim.active = True
    try:
        if mode == "frame":
            results = []
            for f in frames:
                results.append(model(f)[0])
                states.append((sorted(pool.get_active_ids()), sorted(pool._dormant_ids)))
        else:
            results = model.forward_clip(frames, before_frame=lambda t: states.append((sorted(pool.get_active_ids()), sorted(pool._dormant_ids))))
            states = states[1:] + [(sorted(pool.get_active_ids()), sorted(pool._dormant_ids))]
        sim.sync_all()
    finally:
        sim.active = False
    assert sim.executed > 100
    return [dict(boxes=r.bbox, scores=r.get_field("scores"), ids=r.get_field("ids"), labels=r.get_field("labels"), active=a, dormant=d)
            for r, (a, d) in zip(results, states)]


@pytest.mark.parametrize("policy", POLICIES, ids=str)
def test_per_frame_and_two_stream_clip_are_schedule_independent(policy, monkeypatch):
    gold = load_golden(NAME)["frames"]
    _compare(gold, _run_sim(monkeypatch, policy, "frame"))
    _compare(gold, _run_sim(monkeypatch, policy, "clip"))


@pytest.mark.parametrize("pairs", ["0", "1"])
@pytest.mark.parametrize("slots", ["2", "3"])
@pytest.mark.parametrize("policy", POLICIES, ids=str)
def test_three_stage_clip_is_schedule_independent(policy, slots, pairs, monkeypatch):
    """pairs = 1 (the default): the backbone half runs over frame pairs (batch-2 plan, two pair slots); 0: one frame per pass."""
    gold = load_golden(NAME)["frames"]
    env = {"SMOT_CLIP_SPLIT": "1", "SMOT_CLIP_SLOTS": slots, "SMOT_CLIP_PAIRS": pairs}
    _compare(gold, _run_sim(monkeypatch, policy, "clip", env=env))


def _differs(gold, got):
    try:
        _compare(gold, got)
    except AssertionError:
        return True
    return False


def test_the_detector_detects_a_missing_edge(monkeypatch):
    """Remove one edge at a time from the three-stage pipeline: some legal schedule must then break the results."""
    gold = load_golden(NAME)["frames"]
    env = {"SMOT_CLIP_SPLIT": "1", "SMOT_CLIP_SLOTS": "2"}

    def no_wait_on(attr):
        # Stream.wait_event ignores the events stored under P.<attr> (B -> D edge, or D -> T edge)
        def sabotage(mp):
            orig = stream_sim.VStream.wait_event

            def wait_event(self, ev):
                if getattr(ev, "_tag", None) == attr:
                    return
                orig(self, ev)
            mp.setattr(stream_sim.VStream, "wait_event", wait_event)
            from siammot_b200 import engine
            orig_setattr = engine._Plan.__setattr__

            def tagging_setattr(self, name, value):
                if name == attr and value is not None:
                    value._tag = attr
                orig_setattr(self, name, value)
            mp.setattr(engine._Plan, "__setattr__", tagging_setattr)
        return sabotage

    for attr in ("backbone_done", "static_done"):
        broken = False
        for policy in POLICIES:
            with pytest.MonkeyPatch.context() as mp:
                try:
                    got = _run_sim(mp, policy, "clip", env=env, sabotage=no_wait_on(attr))
                    broken = broken or _differs(gold, got)
                except Exception:
                    broken = True
            if broken:
                break
        assert broken, "removing the %s edge went unnoticed under every schedule" % attr


@pytest.mark.parametrize("split", ["0", "1"])
@pytest.mark.parametrize("policy", ["lazy", "workers_eager", ("random", 4)], ids=str)
def test_public_detection_clip_is_schedule_independent(policy, split, monkeypatch):
    """forward_clip(frames, given_detections=...): the per-frame box head over external boxes runs on the caller's stream between
    the detection stage and the track stage of the same frame."""
    from siammot_b200.modelling import build_siammot
    from test_engine_emulated_cpu import BOX_TOL, _given_scenario
    monkeypatch.setenv("SMOT_CLIP_SPLIT", split)
    sim, fake = stream_sim.install(monkeypatch, policy)
    cfg, sd, clip, given = _given_scenario()
    model = build_siammot(cfg)
    model.load_state_dict(sd, strict=False)
    model.eval()
    model.results_on_host = True
    model.reset_siammot_status()
    gold = load_golden("given_det_192x320")["frames"]
    sim.active = True
    try:
        results = model.forward_clip([clip[t] for t in range(len(gold))], given_detections=given)
        sim.sync_all()
    finally:
        sim.active = False
    for t, (r, g) in enumerate(zip(results, gold)):
        assert r.bbox.shape == g["boxes"].shape and torch.equal(r.get_field("ids"), g["ids"]), "frame %d" % t
        if g["boxes"].numel():
            assert float((r.bbox - g["boxes"]).abs().max()) <= BOX_TOL


@pytest.mark.parametrize("policy", ["lazy", "workers_eager", ("random", 6)], ids=str)
def test_device_resident_results_are_schedule_independent(policy, monkeypatch):
    """results_on_host = False (the reference contract): every frame's BoxList fields are views of a device block filled by an
    asynchronous copy from ONE pinned buffer that the next frame rewrites -- the copy must have run before that rewrite."""
    from siammot_b200.modelling import build_siammot
    gold = load_golden(NAME)["frames"]
    for mode in ("frame", "clip"):
        with pytest.MonkeyPatch.context() as mp:
            sim, fake = stream_sim.install(mp, policy)
            cfg, sd, clip = scenario_inputs(NAME)
            cfg.DTYPE = "float32"
            model = build_siammot(cfg)
            model.load_state_dict(sd, strict=False)
            model.eval()
            model.reset_siammot_status()
            sim.active = True
            try:
                res = [model(f)[0] for f in clip] if mode == "frame" else model.forward_clip(list(clip))
                sim.sync_all()
            finally:
                sim.active = False
            for t, (r, g) in enumerate(zip(res, gold)):
                assert r.bbox.shape == g["boxes"].shape and torch.equal(r.get_field("ids"), g["ids"]), (mode, t)
                if g["boxes"].numel():
                    assert float((r.bbox - g["boxes"]).abs().max()) <= 1e-3, (mode, t)


@pytest.mark.parametrize("policy", POLICIES, ids=str)
def test_frame_overlap_is_schedule_independent(policy, monkeypatch):
    """SMOT_FRAME_OVERLAP=1: model(frame) with the detection tail on a second stream under the EMM half of the track stage."""
    gold = load_golden(NAME)["frames"]
    _compare(gold, _run_sim(monkeypatch, policy, "frame", env={"SMOT_FRAME_OVERLAP": "1"}))


def test_frame_overlap_detector_detects_the_missing_wait(monkeypatch):
    """Without the wait on the detection tail before the candidate assembly some schedule must break the results."""
    gold = load_golden(NAME)["frames"]
    from siammot_b200 import engine
    broken = False
    for policy in POLICIES:
        with pytest.MonkeyPatch.context() as mp:
            orig = engine._TrackPlan.run_split
            mp.setattr(engine._TrackPlan, "run_split", lambda self, feat, between: orig(self, feat, lambda: None))
            try:
                broken = broken or _differs(gold, _run_sim(mp, policy, "frame", env={"SMOT_FRAME_OVERLAP": "1"}))
            except Exception:
                broken = True
        if broken:
            break
    assert broken


@pytest.mark.parametrize("n_frames", [7, 8])
@pytest.mark.parametrize("policy", ["lazy", "workers_eager", "default_eager", ("random", 1), ("random", 4)], ids=str)
def test_long_pair_clip_reuses_its_slots_safely(policy, n_frames, monkeypatch):
    """Frame 0 alone, then pairs on two alternating pair slots, then (8 frames) an odd last frame on the single-frame plan
    again: 7 / 8 frames reuse every buffer set at least once.  The adversarial schedule must give what per-frame calls give
    (same emulated kernels, no overlap), row for row and bit for bit."""
    ref = _run_sim(monkeypatch, "eager", "frame", n_frames=n_frames)
    got = _run_sim(monkeypatch, policy, "clip", env={"SMOT_CLIP_SPLIT": "1", "SMOT_CLIP_SLOTS": "3", "SMOT_CLIP_PAIRS": "1"}, n_frames=n_frames)
    assert len(ref) == len(got) == n_frames
    assert sum(int((r["ids"] >= 0).sum()) for r in ref) > 0
    for t, (a, b) in enumerate(zip(ref, got)):
        assert torch.equal(a["ids"], b["ids"]) and torch.equal(a["labels"], b["labels"]), t
        assert torch.equal(a["boxes"], b["boxes"]) and torch.equal(a["scores"], b["scores"]), t
        assert a["active"] == b["active"] and a["dormant"] == b["dormant"], t
