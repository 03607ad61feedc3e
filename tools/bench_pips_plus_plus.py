"""SamPt with ViT-H + PIPS++ on the C2 clip (50 frames 480x854, 8 positive points).

  python tools/bench_pips_plus_plus.py [--steps K] [--warmup W]

Prints one JSON line with
  - fps: frames/s of SamPt._forward with the clip resident on the GPU (CUDA events over K steps after W warm-up steps),
  - tracker_ms_per_clip: PipsPlusPlusPointTracker alone on the same clip and points (encoder, both directions, 16 iterations
    per window; CUDA events over K calls after the warm-up),
  - the card's name and power limit, read in the same run.
Weights are seeded synthetic checkpoints (sampt_b200.synth); nothing is written into the tree."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "sam-pt_b200"), os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import torch  # noqa: E402


def timed(fn, steps):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return sum(a.elapsed_time(b) for a, b in ev) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pips_plus_plus needs a CUDA device")
    import bench
    from bench_tinyvit import card
    from sampt_b200 import factory, synth

    name, power = card()
    T, H, W, P = 50, 480, 854, 8
    dev = torch.device("cuda", 0)
    video = synth.make_video_dict(T, H, W, P, seed=72)
    frames_dev = torch.stack(video["image"]).to(dev)
    q_dev = video["query_points"].to(dev)
    sam = factory.build_sam("vit_h")
    sam_sd = synth.condition_sam(synth.make_state_dict({k: tuple(v.shape) for k, v in sam.state_dict().items()}, bench.SAM_SEED))
    del sam
    model = factory.build_sam_pt("vit_h", sam_sd, None, positive_points_per_mask=P, sam_iou_threshold=-1e9, device=dev,
                                 pips_plus_plus_state_dict=synth.make_pips_plus_plus_state_dict())
    trk = model.point_tracker
    q_flat = q_dev.reshape(1, -1, 3)
    for _ in range(max(args.warmup, 1)):
        model._forward(frames_dev, q_dev)
        trk(frames_dev[None], q_flat.clone())
    torch.cuda.synchronize()
    ms = timed(lambda: model._forward(frames_dev, q_dev), args.steps)
    tms = timed(lambda: trk(frames_dev[None], q_flat.clone()), args.steps)
    print(json.dumps({"model": "vit_h+pips_plus_plus", "frames": T, "shape": [H, W], "points": P, "fps": round(T / (ms / 1e3), 3),
                      "tracker_ms_per_clip": round(tms, 2), "steps": args.steps, "gpu": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
