"""demos/demo.py for the engine, minus video decoding and visualisation (both out of scope, DESIGN.md section 8):
decoded RGB uint8 frames in -> tracks out, through the calls a siam-mot user switches to.

    python tools/demo_clip.py --frames clip.npy --weights model.pth --out tracks.json        # (T, H, W, 3) uint8 frames
    python tools/demo_clip.py --synthetic 64 --out tracks.json                               # synthetic clip, synthetic weights

Flow (reference counterpart): build_siammot(cfg) + checkpoint (demo_inference.py:84-96) -> model.forward_clip(frames)
(process_frame_sequence :112-123, one blocking call per frame there) with the test transform on the device (:74-82) ->
egress.clip_to_tracks (results.resize(...).convert('xywh') :107-108) -> egress.postprocess_tracks (inferencer.py:134-153) ->
JSON records {frame_num, id, label, confidence, bbox [x, y, w, h]}.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--frames", help=".npy file with decoded RGB uint8 frames (T, H, W, 3)")
    src.add_argument("--synthetic", type=int, metavar="T", help="use a synthetic 720p clip of T frames")
    ap.add_argument("--config", default=os.path.join(REPO, "siammot_b200", "configs", "dla34_emm.yaml"))
    ap.add_argument("--weights", default=None, help="reference checkpoint (.pth with a 'model' entry or a plain state dict); "
                                                    "default: seeded synthetic weights")
    ap.add_argument("--dtype", default="float16", choices=["float16", "float32"])
    ap.add_argument("--size", default="720x1280", help="synthetic frame size HxW")
    ap.add_argument("--track-len", type=int, default=5)
    ap.add_argument("--track-conf", type=float, default=0.7)
    ap.add_argument("--out", default=None, help="write the kept tracks as JSON")
    args = ap.parse_args(argv)

    from siammot_b200 import egress
    from siammot_b200.config import get_cfg
    from siammot_b200.modelling import build_siammot
    cfg = get_cfg()
    cfg.merge_from_file(args.config)
    cfg.DTYPE = args.dtype
    if args.frames:
        frames = np.load(args.frames)
        if frames.dtype != np.uint8 or frames.ndim != 4 or frames.shape[3] != 3:
            raise SystemExit("--frames: expected uint8 (T, H, W, 3), got %s %s" % (frames.dtype, frames.shape))
        frames = torch.from_numpy(frames)
    else:
        from siammot_b200.synth_clip import make_clip_u8
        h, w = (int(v) for v in args.size.lower().split("x"))
        frames = make_clip_u8(args.synthetic, h, w, n_obj=10, seed=0, mean=cfg.INPUT.PIXEL_MEAN, std=cfg.INPUT.PIXEL_STD)
    model = build_siammot(cfg)
    if args.weights:
        sd = torch.load(args.weights, map_location="cpu")
        model.load_state_dict(sd.get("model", sd), strict=False)
    else:
        from siammot_b200.synthetic import make_state_dict
        model.load_state_dict(make_state_dict(cfg, 1), strict=False)
    model = model.to("cuda").eval()
    model.results_on_host = True
    model.reset_siammot_status()
    frames = frames.pin_memory()
    results = model.forward_clip([frames[t] for t in range(frames.shape[0])])
    tracks = egress.clip_to_tracks(results, frames.shape[2], frames.shape[1])
    kept = egress.postprocess_tracks(tracks, args.track_len, args.track_conf)
    print("frames %d, boxes %d, tracked ids %d, kept after the track filter: %d boxes of %d ids"
          % (frames.shape[0], len(tracks), len(set(tracks.id[tracks.id >= 0].tolist())), len(kept), len(set(kept.id.tolist()))))
    if args.out:
        recs = [dict(frame_num=int(f), id=int(i), label=int(l), confidence=float(c), bbox=[float(v) for v in b])
                for f, i, l, c, b in zip(kept.frame_num, kept.id, kept.label, kept.confidence, kept.bbox)]
        with open(args.out, "w") as fh:
            json.dump(recs, fh)
    return kept


if __name__ == "__main__":
    main()
