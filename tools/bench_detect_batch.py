"""Throughput of the batched detection stage: a detector-only DLA-34 model (MODEL.TRACK_ON False), fp16, 3x704x1280, over 32
distinct device-resident frames, called as model(x) on batches of B in {1, 2, 4, 8} (B = 1 is the per-frame path).

Per B: warm-up (plan build, graph capture), then at least --images images timed with CUDA events around whole model() calls --
launch, the one device-to-host copy, the host wait and the BoxLists.  Also reported: kernel launches per image of the plan the
calls replay (C-ABI calls x kernels per call, _lib.KERNELS_PER_CALL; memsets and the split-K reduce kernels not counted).
Prints one JSON line with the card's name and power limit.

    python tools/bench_detect_batch.py [--images 256] [--batches 1,2,4,8]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True,
                             timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def launches_per_image(P):
    from siammot_b200 import _lib
    n = 0
    for fn, _args, tag, _branch in P.steps:
        if fn in ("fork", "join"):
            continue
        name = getattr(fn, "__name__", "")
        if name in _lib.KERNELS_PER_CALL:
            n += _lib.KERNELS_PER_CALL[name]
        elif tag == "det_init":
            n += 2                      # the per-frame tail's two fills of the detection block
        else:
            n += 1
    return n / P.batch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=256, help="timed images per batch size (at least 200)")
    ap.add_argument("--batches", default="1,2,4,8")
    ap.add_argument("--frames", type=int, default=32)
    args = ap.parse_args()
    from siammot_b200.config import get_cfg
    from siammot_b200.modelling import build_siammot
    from siammot_b200.synth_clip import make_clip
    from siammot_b200.synthetic import make_state_dict
    cfg = get_cfg()
    cfg.merge_from_file(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "siammot_b200", "configs",
                                     "dla34_emm.yaml"))
    cfg.MODEL.TRACK_ON = False
    cfg.DTYPE = "float16"
    model = build_siammot(cfg)
    model.load_state_dict(make_state_dict(cfg, 0), strict=False)
    model = model.to("cuda").eval()
    frames = torch.stack(list(make_clip(args.frames, 704, 1280, 8, 0))).cuda()
    eng = model.engine()
    results = []
    for B in [int(b) for b in args.batches.split(",")]:
        starts = list(range(0, args.frames - B + 1, B))
        for s in starts[:3]:                                    # warm-up: plan build + graph capture + a few replays
            model(frames[s:s + B])
        calls = -(-max(args.images, 200) // B)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for c in range(calls):
            s = starts[c % len(starts)]
            model(frames[s:s + B])
        e1.record()
        e1.synchronize()
        ms = e0.elapsed_time(e1)
        P = eng.plans[(704, 1280, 0)] if B == 1 else eng.plans[(704, 1280, "batch", B)]
        results.append(dict(B=B, images=calls * B, ms=round(ms, 3), images_per_s=round(calls * B / (ms / 1e3), 1),
                            launches_per_image=round(launches_per_image(P), 2)))
    print(json.dumps(dict(metric="detector_only_dla34_fp16_704x1280_images_per_s", gpu=torch.cuda.get_device_name(),
                          power_limit_w=power_limit_w(), frames=args.frames, results=results)))


if __name__ == "__main__":
    main()
