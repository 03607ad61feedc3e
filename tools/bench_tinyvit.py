"""MobileSAM / Light HQ-SAM throughput on the C2 clip (50 frames 480x854, PIPS, 8 positive points).

  python tools/bench_tinyvit.py [--steps K] [--warmup W] [--refine 3 12] [--dump-outputs DIR]

For each model (MobileSAM, Light HQ-SAM) and each refinement count it prints one JSON line with
  - fps: frames/s of SamPt with the clip resident on the GPU (CUDA events over K steps after W warm-up steps),
  - encoder_ms_per_frame: the TinyViT encoder alone (frames resized beforehand) over a warmed 8-frame batch (CUDA events,
    20 repetitions),
  - the card's name and power limit, read in the same run.
`--dump-outputs DIR` writes the last step's arrays as bench.py does, under DIR/<model>_r<refine>/.
Weights are seeded synthetic checkpoints (sampt_b200.synth); nothing is written into the tree."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "sam-pt_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import torch  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                          str(torch.cuda.current_device())], capture_output=True, text=True)
    name, power = (s.strip() for s in out.stdout.strip().split(",")) if out.returncode == 0 else (torch.cuda.get_device_name(), "?")
    return name, power


def encoder_ms(model, frames_dev, B=8, reps=20):
    """TinyViT alone: the frames are resized once beforehand, the timed calls are image_encoder.encode_resized_u8."""
    pred = model.sam_predictor
    resized = pred.resize_frames_u8(frames_dev[:B])
    mean, std = pred._pixel_stats()
    enc = pred.model.image_encoder
    want = pred._uses_interm()
    for _ in range(3):
        enc.encode_resized_u8(resized, mean, std, want_interm=want)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        enc.encode_resized_u8(resized, mean, std, want_interm=want)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / (reps * B)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--refine", type=int, nargs="+", default=[3, 12])
    ap.add_argument("--dump-outputs", default=None, metavar="DIR")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tinyvit needs a CUDA device")
    import bench
    from sam_pt.point_tracker.pips.pips import _pips_shapes
    from sampt_b200 import synth

    name, power = card()
    pips_sd = synth.condition_pips(synth.make_state_dict(_pips_shapes(8), bench.PIPS_SEED))
    with tempfile.TemporaryDirectory(prefix="sampt_bench_tinyvit_") as tmp:
        ckpt = synth.write_pips_checkpoint_dir(pips_sd, os.path.join(tmp, "pips"))
        run(args, ckpt, name, power)


def run(args, ckpt, name, power):
    import bench
    from sampt_b200 import factory, synth

    T, H, W, P = 50, 480, 854, 8
    dev = torch.device("cuda", 0)
    video = synth.make_video_dict(T, H, W, P, seed=72)
    frames_dev = torch.stack(video["image"]).to(dev)
    q_dev = video["query_points"].to(dev)
    for label, hq in (("mobile_sam", False), ("light_hq_sam", True)):
        sam = factory.build_sam(factory.TINY_VIT, hq=hq)
        shapes = {k: tuple(v.shape) for k, v in sam.state_dict().items() if not k.startswith("image_encoder.")}
        sam_sd = synth.condition_sam(synth.make_state_dict(shapes, bench.SAM_SEED))
        for k, v in synth.make_tinyvit_state_dict(bench.SAM_SEED).items():
            sam_sd["image_encoder." + k] = v
        for n_ref in args.refine:
            model = factory.build_sam_pt(factory.TINY_VIT, sam_sd, ckpt, positive_points_per_mask=P, sam_iou_threshold=-1e9,
                                         device=dev, hq=hq, iterative_refinement_iterations=n_ref)
            for _ in range(max(args.warmup, 1)):
                model._forward(frames_dev, q_dev)
            torch.cuda.synchronize()
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
            for i in range(args.steps):
                ev[i][0].record()
                traj, vis, logits, scores, spf = model._forward(frames_dev, q_dev)
                ev[i][1].record()
            torch.cuda.synchronize()
            ms = sum(a.elapsed_time(b) for a, b in ev)
            if args.dump_outputs:
                bench.dump_outputs(os.path.join(args.dump_outputs, f"{label}_r{n_ref}"), (logits, spf, traj, vis))
            line = {"model": label, "refinements": n_ref, "frames": T, "shape": [H, W], "points": P,
                    "fps": round(T * args.steps / (ms / 1e3), 3), "encoder_ms_per_frame": round(encoder_ms(model, frames_dev), 4),
                    "steps": args.steps, "gpu": name, "power_limit": power}
            print(json.dumps(line), flush=True)
            del model
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
