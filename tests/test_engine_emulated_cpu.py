"""The engine's host side, end to end, without a GPU: build_siammot(cfg) -> model(frame) runs over tests/cabi_emulator.py
(every libsmot entry point emulated with the oracle's primitives on the pointers the engine passes) and must reproduce the
goldens the reference itself produced -- ids / labels bit-exact, boxes <= 1e-3 px -- on every scenario, including the ones
whose GPU run is still pending (two foreground classes, TRACKTOR, AOT geometry, R-50-FPN body).  This pins launch plans,
arenas, result-block packing, the host solver and the next-frame memory; the CUDA kernels are what the `-m gpu` tests pin."""
import pytest
import torch

import cabi_emulator
from helpers import load_golden, scenario_inputs
from scenarios import ORACLE_SCENARIOS, SCENARIOS, inject_boxes

BOX_TOL, SCORE_TOL = 1e-3, 1e-3


def _run(name, monkeypatch, clip_api=False, env=None):
    from siammot_b200.modelling import build_siammot
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    fake = cabi_emulator.install(monkeypatch)
    sc = SCENARIOS.get(name) or ORACLE_SCENARIOS[name]
    cfg, sd, clip = scenario_inputs(name)
    cfg.DTYPE = "float32"
    model = build_siammot(cfg)
    model.load_state_dict(sd, strict=False)
    model.eval()
    model.reset_siammot_status()
    out, start = [], 0
    pool = model.roi_heads.track.track_pool
    if sc["inject"] is not None:
        eng = model.engine()
        P = eng.run_static(clip[0])
        pool.reset()
        boxes = inject_boxes(sc["inject"])
        ids = torch.tensor([pool.start_track() for _ in range(len(boxes))])
        model.flush_memory(model.roi_heads._build_memory(P, boxes.numpy(), ids.numpy(), torch.ones(len(boxes), dtype=torch.int64).numpy()))
        pool.increment_frame()
        start = 1
    frames = [clip[t] for t in range(start, sc["frames"])]
    if clip_api:
        states = []
        results = model.forward_clip(frames, before_frame=lambda t: states.append((sorted(pool.get_active_ids()), sorted(pool._dormant_ids))))
        states = states[1:] + [(sorted(pool.get_active_ids()), sorted(pool._dormant_ids))]
    else:
        results, states = [], []
        for f in frames:
            results.append(model(f)[0])
            states.append((sorted(pool.get_active_ids()), sorted(pool._dormant_ids)))
    for r, (act, dor) in zip(results, states):
        out.append(dict(boxes=r.bbox, scores=r.get_field("scores"), ids=r.get_field("ids"), labels=r.get_field("labels"),
                        active=act, dormant=dor))
    return out, fake


def _compare(gold, got):
    assert len(got) == len(gold)
    for t, (g, o) in enumerate(zip(gold, got)):
        assert o["boxes"].shape == g["boxes"].shape, "frame %d: %d boxes vs %d" % (t, o["boxes"].shape[0], g["boxes"].shape[0])
        assert torch.equal(o["ids"], g["ids"]), "frame %d: track ids differ" % t
        assert torch.equal(o["labels"], g["labels"]), "frame %d: labels differ" % t
        if g["boxes"].numel():
            assert float((o["boxes"] - g["boxes"]).abs().max()) <= BOX_TOL, "frame %d boxes" % t
            assert float((o["scores"] - g["scores"]).abs().max()) <= SCORE_TOL, "frame %d scores" % t
        assert o["active"] == g["active"] and o["dormant"] == g["dormant"], "frame %d pool state" % t


SMALL = [n for n in list(SCENARIOS) + list(ORACLE_SCENARIOS) if n != "pair_720p_4tracks"]


@pytest.mark.parametrize("name", SMALL)
def test_emulated_engine_matches_reference_golden(name, monkeypatch):
    got, fake = _run(name, monkeypatch)
    _compare(load_golden(name)["frames"], got)
    assert fake.calls.get("smot_xcorr", 0) > 0 and fake.calls.get("smot_sort_nms", 0) > 0


def test_emulated_engine_720p_pair_with_injected_tracks(monkeypatch):
    """BASELINE.json configs[0] (704x1280, four injected tracks on FPN levels 0,1,2,0)."""
    got, _ = _run("pair_720p_4tracks", monkeypatch)
    _compare(load_golden("pair_720p_4tracks")["frames"], got)


def test_emulated_forward_clip_equals_golden(monkeypatch):
    """The clip API's bookkeeping (double-buffered plans, next_P for the memory) on the host."""
    got, _ = _run("emm_amodal_expire_192x320", monkeypatch, clip_api=True)
    _compare(load_golden("emm_amodal_expire_192x320")["frames"], got)


def test_emulated_planar_window_exchange_wiring(monkeypatch):
    """Host wiring of the SMOT_XCORR_PLANAR switch (arena buffer, the two planar calls in the track plan): same goldens.
    The emulation is fp32, so the dtype condition of the switch is lifted for this test only."""
    from siammot_b200 import engine
    monkeypatch.setattr(engine.Engine, "xcorr_planar_ok", lambda self: self.xcorr_planar and self.s_res == 30 and self.t_res == 15)
    got, fake = _run("emm_256x384", monkeypatch, env={"SMOT_XCORR_PLANAR": "1"})
    _compare(load_golden("emm_256x384")["frames"], got)
    assert fake.calls.get("smot_xcorr_planar", 0) > 0 and fake.calls.get("smot_roi_align_planar", 0) > 0
    assert fake.calls.get("smot_xcorr", 0) == 0


@pytest.mark.parametrize("slots", ["2", "3"])
def test_emulated_three_stage_clip_equals_golden(slots, monkeypatch):
    """SMOT_CLIP_SPLIT=1: the static plan cut at the proposal selection, K plan copies -- same results (this checks the
    bookkeeping: plan slices, slot rotation, next_P; the stream / event ordering can only be exercised on a GPU)."""
    env = {"SMOT_CLIP_SPLIT": "1", "SMOT_CLIP_SLOTS": slots}
    for name in ("emm_amodal_expire_192x320", "emm_256x384"):
        got, fake = _run(name, monkeypatch, clip_api=True, env=env)
        _compare(load_golden(name)["frames"], got)


def _plugin_contract_check(model, cfg, sd, clip, to_dev=lambda t: t):
    """EMM.extract_cache / EMM.forward (the SIAMESE_TRACKER plugin contract, track_core.py:28-98) against the oracle."""
    from oracle import siammot_oracle as orc
    from siammot_b200.structures import BoxList
    T = cfg.MODEL.TRACK_HEAD
    H, W = clip[0].shape[1], clip[0].shape[2]
    eng = model.engine()
    tracker = model.roi_heads.track.tracker
    boxes = inject_boxes([(60., 80., 40., 90.), (150., 100., 70., 120.), (250., 90., 100., 160.), (300., 150., 30., 60.)])
    ids = torch.tensor([0, 1, 2, 3])
    labels = torch.ones(4, dtype=torch.int64)
    det = BoxList(to_dev(boxes.clone()), (W, H), "xyxy")
    det.add_field("ids", to_dev(ids))
    det.add_field("labels", to_dev(labels))
    det.add_field("scores", to_dev(torch.full((4,), 0.9)))
    P0 = eng.run_static(to_dev(clip[0]))
    x, sr, dets = tracker.extract_cache(P0, det)
    o = orc.OracleSiamMOT(cfg, sd)
    feats0 = o.features(clip[0])
    ref_x = orc.pool_rois(feats0, boxes, boxes, T.POOLER_SCALES, T.POOLER_RESOLUTION, T.POOLER_SAMPLING_RATIO)
    ref_sr = orc.search_region(boxes, T.PAD_PIXELS, T.SEARCH_REGION - 1.0, T.MINIMUM_SREACH_REGION)
    assert tuple(x.shape) == (4, T.POOLER_RESOLUTION, T.POOLER_RESOLUTION, eng.C)
    assert float((x.permute(0, 3, 1, 2).float().cpu() - ref_x).abs().max()) <= 2e-5 * float(ref_x.abs().max())
    assert len(sr) == 1 and torch.equal(sr[0].bbox.cpu(), ref_sr) and tuple(sr[0].size) == (W + 2 * T.PAD_PIXELS, H + 2 * T.PAD_PIXELS)
    assert dets[0] is det
    from siammot_b200.modelling.rcnn import FeaturesView
    x2, sr2, _ = tracker.extract_cache(FeaturesView(P0), det)          # the reference's argument form: a sequence of NCHW maps
    assert torch.equal(x2, x) and torch.equal(sr2[0].bbox, sr[0].bbox)
    # next frame: propagate the four tracks
    P1 = eng.run_static(to_dev(clip[1]))
    extra, out, losses = tracker(P1, [det], sr, template_features=x)
    assert extra == {} and losses == {} and len(out) == 1
    ref = orc.emm_forward(o.P, cfg, o.features(clip[1]), dict(feat=ref_x, sr=ref_sr, boxes=boxes, ids=ids, labels=labels), W, H)
    got = out[0]
    assert torch.equal(got.get_field("ids").cpu(), ref["ids"]) and torch.equal(got.get_field("labels").cpu(), ref["labels"])
    assert float((got.bbox.cpu() - ref["boxes"]).abs().max()) <= BOX_TOL
    assert float((got.get_field("scores").cpu() - ref["scores"]).abs().max()) <= SCORE_TOL
    # the reference's argument forms (track_core.py:28,81-98): `features` a sequence of NCHW maps, templates NCHW
    fv = FeaturesView(P1)
    ref_feats = o.features(clip[1])
    assert len(fv) == len(ref_feats) == 5 and len(fv[1:3]) == 2
    for l, (a, b) in enumerate(zip(fv, ref_feats)):
        assert tuple(a.shape) == tuple(b.shape), l                      # (1, C, H_l, W_l): what a reference-style tracker indexes
        assert float((a.float().cpu() - b).abs().max()) <= 1e-4 * float(b.abs().max())
    import torchvision
    third_party = torchvision.ops.roi_align(fv[0].float(), [det.bbox.float()], 7, 0.25, 2, False)    # any torch op takes the view
    want = torchvision.ops.roi_align(ref_feats[0], [boxes], 7, 0.25, 2, False)
    assert float((third_party.cpu() - want).abs().max()) <= 1e-4 * float(want.abs().max())
    _, out2, _ = tracker(fv, [det], sr, template_features=x.permute(0, 3, 1, 2))
    assert torch.equal(out2[0].bbox, got.bbox) and torch.equal(out2[0].get_field("scores"), got.get_field("scores"))


def test_emulated_tracker_plugin_contract(monkeypatch):
    from siammot_b200.modelling import build_siammot
    cabi_emulator.install(monkeypatch)
    cfg, sd, clip = scenario_inputs("emm_256x384")
    cfg.DTYPE = "float32"
    model = build_siammot(cfg)
    model.load_state_dict(sd, strict=False)
    model.eval()
    _plugin_contract_check(model, cfg, sd, clip)


@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
def test_emulated_flush_memory_accepts_the_reference_memory_tuple(layout, monkeypatch):
    """SiamMOT.flush_memory(cache) with the reference's (template_features, [sr], [boxes]) tuple (rcnn.py:34, track_head.py:54-110),
    templates in the reference's NCHW layout or in the engine's NHWC one: the next frame must come out exactly as in the normal
    flow, where the engine carries its own memory object."""
    from siammot_b200.modelling import build_siammot
    cabi_emulator.install(monkeypatch)
    name = "emm_256x384"
    cfg, sd, clip = scenario_inputs(name)
    cfg.DTYPE = "float32"

    def fresh():
        m = build_siammot(cfg)
        m.load_state_dict(sd, strict=False)
        m.eval()
        m.reset_siammot_status()
        return m

    ref_model = fresh()
    ref = [ref_model(clip[t])[0] for t in range(3)]
    model = fresh()
    for t in range(2):
        model(clip[t])
    mem = model.track_memory                       # the engine's own memory after frame 1
    W, H = clip[0].shape[2], clip[0].shape[1]
    feats, sr_l, boxes_l = mem.as_reference_tuple((W, H), cfg.MODEL.TRACK_HEAD.PAD_PIXELS)
    # ... which is also what unpacking ``model.track_memory`` the reference way (track_head.py:54-110) yields
    f2, s2, b2 = model.track_memory
    assert len(model.track_memory) == 3 and torch.equal(f2, feats) and torch.equal(s2[0].bbox, sr_l[0].bbox) and tuple(s2[0].size) == tuple(sr_l[0].size)
    assert torch.equal(b2[0].bbox, boxes_l[0].bbox) and torch.equal(b2[0].get_field("ids"), boxes_l[0].get_field("ids")) and tuple(b2[0].size) == (W, H)
    assert torch.equal(model.track_memory[2][0].get_field("labels"), boxes_l[0].get_field("labels"))
    sr, boxes = sr_l[0], boxes_l[0]
    assert tuple(feats.shape[1:]) == (128, 15, 15) and tuple(sr.size) == (W + 1024, H + 1024)
    if layout == "nhwc":
        feats = mem.feat
    model.flush_memory((feats, [sr], [boxes]))
    got = model(clip[2])[0]
    assert len(got) == len(ref[2]) and int((ref[2].get_field("ids") >= 0).sum()) > 0
    assert torch.equal(got.bbox, ref[2].bbox) and torch.equal(got.get_field("ids"), ref[2].get_field("ids"))
    assert torch.equal(got.get_field("scores"), ref[2].get_field("scores"))
    with pytest.raises(ValueError):
        model.flush_memory((feats[:, :3], [sr], [boxes]))


def _given_scenario():
    import os
    from helpers import CONFIG_DIR, YAML_MAP
    from scenarios import GIVEN_SCENARIOS, given_boxes
    from siammot_b200.config import get_cfg
    from siammot_b200.structures import BoxList
    from siammot_b200.synth_clip import make_clip
    from siammot_b200.synthetic import make_state_dict
    sc = GIVEN_SCENARIOS["given_det_192x320"]
    cfg = get_cfg()
    cfg.merge_from_file(os.path.join(CONFIG_DIR, YAML_MAP[sc["yaml"]]))
    cfg.merge_from_list(sc["overrides"])
    cfg.DTYPE = "float32"
    clip = make_clip(sc["frames"], sc["H"], sc["W"], sc["n_obj"], sc["clip_seed"])
    given = []
    for boxes in given_boxes(sc):
        n = boxes.shape[0]
        bl = BoxList(boxes.clone(), (sc["W"], sc["H"]), mode="xyxy")
        bl.add_field("labels", torch.ones(n, dtype=torch.int64))
        bl.add_field("scores", torch.ones(n))
        bl.add_field("ids", torch.full((n,), -1, dtype=torch.int64))
        given.append([bl])
    return cfg, make_state_dict(cfg, sc["weight_seed"]), clip, given


@pytest.mark.parametrize("mode", ["frame", "clip", "clip3"])
def test_emulated_public_detections_match_reference_golden(mode, monkeypatch):
    """given_detection every frame (one frame with none at all) -- per-frame calls and the clip API's given_detections."""
    from siammot_b200.modelling import build_siammot
    if mode == "clip3":
        monkeypatch.setenv("SMOT_CLIP_SPLIT", "1")
    cabi_emulator.install(monkeypatch)
    cfg, sd, clip, given = _given_scenario()
    model = build_siammot(cfg)
    model.load_state_dict(sd, strict=False)
    model.eval()
    model.reset_siammot_status()
    gold = load_golden("given_det_192x320")["frames"]
    if mode == "frame":
        results = [model(clip[t], given_detection=given[t])[0] for t in range(len(gold))]
    else:
        results = model.forward_clip([clip[t] for t in range(len(gold))], given_detections=given)
    for t, (r, g) in enumerate(zip(results, gold)):
        assert r.bbox.shape == g["boxes"].shape, "frame %d" % t
        assert torch.equal(r.get_field("ids"), g["ids"]) and torch.equal(r.get_field("labels"), g["labels"]), "frame %d" % t
        if g["boxes"].numel():
            assert float((r.bbox - g["boxes"]).abs().max()) <= BOX_TOL and float((r.get_field("scores") - g["scores"]).abs().max()) <= SCORE_TOL
    pool = model.roi_heads.track.track_pool
    assert sorted(pool.get_active_ids()) == gold[-1]["active"] and sorted(pool._dormant_ids) == gold[-1]["dormant"]


def test_emulated_reset_between_videos_and_resolution_change(monkeypatch):
    """reset_siammot_status() between videos (inferencer.py:157-159): ids restart, results repeat exactly; a video of another
    resolution gets its own launch plan and arena and leaves the first one's results unchanged when it comes back."""
    from siammot_b200.modelling import build_siammot
    from siammot_b200.synth_clip import make_clip
    cabi_emulator.install(monkeypatch)
    cfg, sd, clip = scenario_inputs("emm_amodal_expire_192x320")
    cfg.DTYPE = "float32"
    model = build_siammot(cfg)
    model.load_state_dict(sd, strict=False)
    model.eval()

    def run(frames):
        model.reset_siammot_status()
        return [model(f)[0] for f in frames]

    a = run(clip[:4])
    other = make_clip(3, 128, 224, 4, 11)
    b = run(other)
    assert all(r.size == (224, 128) for r in b)
    a2 = run(clip[:4])
    assert max(int(r.get_field("ids").max()) for r in a if len(r)) >= 0
    for x, y in zip(a, a2):
        assert torch.equal(x.bbox, y.bbox) and torch.equal(x.get_field("ids"), y.get_field("ids"))
        assert torch.equal(x.get_field("scores"), y.get_field("scores"))
    # 4-D batch-of-one input and an object with .tensors (ImageList) are the same call
    model.reset_siammot_status()
    r4 = model(clip[0][None])[0]

    class ImageListLike(object):
        tensors = clip[0][None]
    model.reset_siammot_status()
    rl = model(ImageListLike())[0]
    assert torch.equal(r4.bbox, a[0].bbox) and torch.equal(rl.bbox, a[0].bbox)
    with pytest.raises(ValueError):
        model(torch.zeros(2, 3, 192, 320))


@pytest.mark.parametrize("clip_api", [False, True])
def test_emulated_detector_only_model(clip_api, monkeypatch):
    """MODEL.TRACK_ON False (roi_heads.py:36,92): no track head, no solver -- the box head's detections with id -1, per frame and
    through the clip API; the parameter tree has no roi_heads.track.* entries, like the reference's."""
    from oracle import siammot_oracle as orc
    from siammot_b200.modelling import build_siammot
    cabi_emulator.install(monkeypatch)
    cfg, sd, clip = scenario_inputs("emm_3class_192x320")
    cfg.merge_from_list(["MODEL.TRACK_ON", False])
    cfg.DTYPE = "float32"
    model = build_siammot(cfg)
    assert not any(k.startswith("roi_heads.track.") for k in model.state_dict())
    assert "track" not in model.roi_heads and "solver" not in model.roi_heads
    model.load_state_dict({k: v for k, v in sd.items() if not k.startswith("roi_heads.track.")}, strict=False)
    model.eval()
    model.reset_siammot_status()
    frames = [clip[t] for t in range(3)]
    results = model.forward_clip(frames) if clip_api else [model(f)[0] for f in frames]
    o = orc.OracleSiamMOT(cfg, sd)
    for f, r in zip(frames, results):
        feats = o.features(f)
        props, _ = orc.rpn_forward(o.P, cfg, feats, f.shape[2], f.shape[1])
        ref = orc.box_head_forward(o.P, cfg, feats, props, f.shape[2], f.shape[1])
        assert len(r) == ref["boxes"].shape[0] > 0
        assert torch.equal(r.get_field("labels"), ref["labels"]) and bool((r.get_field("ids") == -1).all())
        assert float((r.bbox - ref["boxes"]).abs().max()) <= BOX_TOL and float((r.get_field("scores") - ref["scores"]).abs().max()) <= SCORE_TOL
    assert model.track_memory is None


@pytest.mark.parametrize("override", [["MODEL.ROI_BOX_HEAD.FEATURE_EXTRACTOR", "FPNXconv1fcFeatureExtractor"], ["MODEL.FPN.USE_GN", True],
                                      ["MODEL.RPN.USE_FPN", False], ["MODEL.BACKBONE.CONV_BODY", "DLA-46-XC-FPN"],
                                      ["MODEL.RPN.ANCHOR_STRIDE", (16,)]])
def test_unsupported_configuration_alternatives_fail_loudly(override, monkeypatch):
    from siammot_b200 import engine
    cabi_emulator.install(monkeypatch)
    cfg, sd, clip = scenario_inputs("emm_256x384")
    cfg.merge_from_list(override)
    with pytest.raises(NotImplementedError):
        engine.Engine(cfg, device="cpu", use_graph=False)


def test_emulated_frame_overlap_equals_golden(monkeypatch):
    """SMOT_FRAME_OVERLAP=1 (split static plan + split track plan in model(frame)): same results on two scenarios."""
    for name in ("emm_amodal_expire_192x320", "emm_3class_192x320"):
        got, fake = _run(name, monkeypatch, env={"SMOT_FRAME_OVERLAP": "1"})
        _compare(load_golden(name)["frames"], got)
