"""Interactive point correction on the H100: J&F counts per frame at 480x854 and 1080x1920, DBSCAN at n = 18 000, full-pass
time with and without the per-frame decode cache, and seconds per interaction of `SamPtInteractive.forward` (online, PIPS).
SAM ViT-B and PIPS carry seeded synthetic weights (timing does not depend on the values).  Prints one JSON line with the card
name and power limit.

    python tools/bench_interactive.py [--frames 16] [--interactions 12] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "sam-pt_b200")]


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def _time(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def _ellipses(T, h, w, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[:h, :w]
    out = np.zeros((T, h, w), bool)
    for t in range(T):
        out[t] = ((yy - rng.uniform(0.3, 0.7) * h) / (0.3 * h)) ** 2 + ((xx - rng.uniform(0.3, 0.7) * w) / (0.3 * w)) ** 2 <= 1
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--interactions", type=int, default=12)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    from oracle import pips_ref, sam_ref
    from sam_pt.modeling import sam_pt_interactive as I
    from sampt_b200 import factory, synth

    res = {"card": _card()}
    for h, w in ((480, 854), (1080, 1920)):
        T = 16
        P = torch.from_numpy(np.where(_ellipses(T, h, w, 1), 1.0, -1.0).astype(np.float32)).cuda()
        G = torch.from_numpy(_ellipses(T, h, w, 2).astype(np.uint8)).cuda()
        res[f"jf_us_per_frame_{h}x{w}"] = round(_time(lambda: I.jf_counts(P, G), 20) * 1e3 / T, 2)
    m = torch.from_numpy(_ellipses(1, 480, 854, 3)[0]).cuda()
    px = m.nonzero().float()
    px = px[torch.randperm(len(px), generator=torch.Generator().manual_seed(0))[:18000].cuda()]
    res["dbscan_ms_n18000_480x854"] = round(_time(lambda: I.dbscan_labels(px, 2.4 * 480 * 854 / 18000, 10), 5), 3)

    T, H, W = args.frames, 480, 854
    sam_sd = synth.condition_sam(synth.make_state_dict(sam_ref.sam_state_dict_shapes(sam_ref.VIT_B), 31))
    pips_sd = synth.condition_pips(synth.make_state_dict(pips_ref.pips_state_dict_shapes(), 7201))
    with tempfile.TemporaryDirectory() as d:
        ckpt = synth.write_pips_checkpoint_dir(pips_sd, os.path.join(d, "pips"))
        base = factory.build_sam_pt("vit_b", sam_sd, ckpt, positive_points_per_mask=8)
        kw = {k: getattr(base, k) for k in (
            "point_tracker", "sam_predictor", "sam_iou_threshold", "positive_point_selection_method",
            "negative_point_selection_method", "positive_points_per_mask", "negative_points_per_mask",
            "add_other_objects_positive_points_as_negative_points", "max_other_objects_positive_points",
            "point_tracker_mask_batch_size", "iterative_refinement_iterations", "use_patch_matching_filtering", "patch_size",
            "patch_similarity_threshold", "use_point_reinit", "reinit_point_tracker_horizon", "reinit_horizon", "reinit_variant")}
        video = synth.make_video_dict(T, H, W, 8, seed=5)
        video["video_id"] = "bench"
        video["gt_masks"] = [torch.from_numpy(g)[None] for g in _ellipses(T, H, W, 4)]
        for reuse in (True, False):
            model = I.SamPtInteractive(online=True, online_interactive_iou_threshold=0.99, interactions_max=8 + args.interactions,
                                       **kw).cuda().eval()
            model._reuse_decodes = reuse
            cwd = os.getcwd()
            os.chdir(d)
            try:
                orig = model._refresh
                spent = []

                def timed(frame_ids, *a, _orig=orig, _spent=spent):
                    ids = list(frame_ids)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    _orig(ids, *a)
                    torch.cuda.synchronize()
                    if len(ids) == T:
                        _spent.append(time.perf_counter() - t0)

                model._refresh = timed
                torch.manual_seed(0)
                model(video)          # warm-up: CUDA graphs, kernels
                spent.clear()
                torch.manual_seed(0)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                model(video)
                torch.cuda.synchronize()
                total = time.perf_counter() - t0
            finally:
                os.chdir(cwd)
            with open(os.path.join(d, "interactions", "bench", "history.json")) as f:
                n_int = len(json.load(f))
            tag = "cached" if reuse else "uncached"
            res[f"full_pass_decode_ms_{tag}"] = round(1e3 * float(np.mean(spent)), 2) if spent else None
            res[f"s_per_interaction_{tag}"] = round(total / max(n_int, 1), 4)
            res["interactions"] = n_int
    res["clip"] = f"{T}x{H}x{W}, SAM ViT-B + PIPS, synthetic weights, online threshold 0.99"
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
