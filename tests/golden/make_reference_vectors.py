"""Generate tests/golden/reference_vectors.pt.gz: what the reference's own modules produce for the seeded inputs of the tests that
compare against them (state-dict layouts, xcorr, the DLA family, result egress), so that those tests run without the
reference tree.  Large outputs are stored as a fixed, seeded sample of elements plus full-tensor float64 sums.

  SIAMMOT_REFERENCE_ROOT=<reference checkout> python tests/golden/make_reference_vectors.py
"""
import gzip
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
for p in (REPO, os.path.join(REPO, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

OUT = os.path.join(HERE, "reference_vectors.pt.gz")


def sample(t):
    """A fixed sample of a tensor's elements (helpers.sample_index) and its float64 sums."""
    from helpers import sample_index
    flat = t.detach().reshape(-1).float()
    return {"shape": tuple(t.shape), "val": flat[sample_index(flat.numel())].clone(), "sum": float(flat.double().sum()),
            "abs_sum": float(flat.double().abs().sum()), "abs_max": float(flat.abs().max())}


def state_dicts(cfg0, build, root):
    from scenarios import ORACLE_SCENARIOS, SCENARIOS
    out = {}
    for name in ("emm_256x384", "emm_r50_192x320", "emm_dla102_192x320", "emm_dla60_dcn_192x320"):
        sc = SCENARIOS.get(name) or ORACLE_SCENARIOS[name]
        rcfg = cfg0.clone()
        rcfg.merge_from_file(os.path.join(root, "configs", "dla", sc["yaml"]))
        rcfg.merge_from_list(sc["overrides"])
        rcfg.MODEL.DEVICE = "cpu"
        out[name] = [(k, tuple(v.shape)) for k, v in build(rcfg).state_dict().items()]
    rcfg = cfg0.clone()
    rcfg.merge_from_file(os.path.join(root, "configs", "dla", "DLA_34_FPN_EMM.yaml"))
    rcfg.merge_from_list(["MODEL.TRACK_ON", False])
    rcfg.MODEL.DEVICE = "cpu"
    out["detector_only"] = [(k, tuple(v.shape)) for k, v in build(rcfg).state_dict().items()]
    return out


def xcorr():
    from siammot.modelling.track_head.EMM.xcorr import xcorr_depthwise
    from test_oracle_golden import xcorr_inputs
    return sample(xcorr_depthwise(*xcorr_inputs()))


def dla_family():
    from siammot.modelling.backbone import dla as ref_dla
    from test_oracle_dla_family_cpu import CASES, fill_weights
    out = {}
    for arch, dcn in CASES:
        torch.manual_seed(0)
        net = ref_dla.BACKBONE[arch](dcn).eval()
        sd = net.state_dict()
        x = fill_weights(sd)
        with torch.no_grad():
            ref = net(x)
        out[(arch, dcn)] = {"keys": [(k, tuple(v.shape)) for k, v in sd.items()], "out": [sample(t) for t in ref]}
    return out


def egress():
    from maskrcnn_benchmark.structures.bounding_box import BoxList as RefBoxList
    from siammot.utils.boxlists_to_entities import boxlists_to_entities
    from siammot_b200 import egress as eg
    import test_egress_cpu as te
    out = {}
    for video in te.VIDEOS:
        ents = []
        for t, r in enumerate(te._random_results(video[0])):
            rb = RefBoxList(r.bbox.clone(), r.size, "xyxy")
            for f in r.fields():
                rb.add_field(f, r.get_field(f))
            o = rb.resize([video[0], video[1]]).convert("xywh").to(torch.device("cpu"))
            ents += boxlists_to_entities([o], 100 + t, [0.04 * (100 + t)], class_table=["person", "vehicle"])
        out[video] = [te.entity_tuple(e) for e in ents]
    fn, DataSample = te._reference_postprocess()
    tracks = eg.clip_to_tracks(te._random_results(7, n_frames=40), 1280, 720)
    sample_ = DataSample("v", entities=eg.to_entities(tracks, ["person", "vehicle"]))
    out["postprocess"] = sorted(te.entity_key(e) for e in fn(te.PostprocessSelf(), sample_).entities)
    return out


def main():
    from oracle import reference_loader
    cfg0, build = reference_loader.load()
    vec = {"state_dict": state_dicts(cfg0, build, reference_loader.REFERENCE_ROOT), "xcorr": xcorr(), "dla": dla_family(),
           "egress": egress()}
    with gzip.GzipFile(OUT, "wb", mtime=0) as f:
        torch.save(vec, f)
    print("wrote %s (%d bytes)" % (OUT, os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
