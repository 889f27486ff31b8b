"""Generate tests/golden/detect_batch3_192x320.pt: the reference's detector-only model (MODEL.TRACK_ON False) called ONCE on
a batch of three distinct frames, as do_inference does with INFERENCE.CLIP_LEN > 1 (inferencer.py:60-68).

Run in the authoring container only (the reference tree does not exist on the GPU box):

    python tests/golden/make_batch_golden.py

The reference is the UNMODIFIED upstream model over the maskrcnn_benchmark stand-in in oracle/shim (see make_golden.py), with
the seeded weights of the other scenarios.  Stored: the spec (the frames are a function of its seeds) and the three BoxLists (boxes / scores /
labels) the batched call returns, in image order.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))

from oracle import reference_loader  # noqa: E402
from siammot_b200.synth_clip import make_clip  # noqa: E402
from siammot_b200.synthetic import make_state_dict  # noqa: E402

NAME = "detect_batch3_192x320"
# three distinct frames: frames 0, 2 and 4 of a seeded clip (objects move between them)
SPEC = dict(yaml="DLA_34_FPN_EMM.yaml", overrides=["MODEL.TRACK_ON", False], H=192, W=320, frames=5, n_obj=5, clip_seed=1,
            weight_seed=0, pick=(0, 2, 4))
PATH = os.path.join(HERE, NAME + ".pt")


def build_reference(sc):
    """make_golden.build_reference for a model without a track head: the seeded weights minus the track head's."""
    cfg0, build = reference_loader.load()
    cfg = cfg0.clone()
    cfg.merge_from_file(os.path.join(reference_loader.REFERENCE_ROOT, "configs", "dla", sc["yaml"]))
    cfg.merge_from_list(sc["overrides"])
    cfg.MODEL.DEVICE = "cpu"
    model = build(cfg).eval()
    sd = model.state_dict()
    sd.update({k: v for k, v in make_state_dict(cfg, sc["weight_seed"]).items() if k in sd})
    model.load_state_dict(sd)
    return cfg, model


def run():
    cfg, model = build_reference(SPEC)
    clip = make_clip(SPEC["frames"], SPEC["H"], SPEC["W"], SPEC["n_obj"], SPEC["clip_seed"])
    batch = torch.stack([clip[t] for t in SPEC["pick"]])
    model.reset_siammot_status()
    with torch.no_grad():
        out = model(batch)
    assert len(out) == batch.shape[0]
    images = []
    for i, r in enumerate(out):
        images.append(dict(boxes=r.bbox.clone(), scores=r.get_field("scores").clone(), labels=r.get_field("labels").clone()))
        print(NAME, "image", i, "boxes", len(r))
    torch.save(dict(scenario=NAME, spec=SPEC, torch=torch.__version__, images=images), PATH)


if __name__ == "__main__":
    run()
