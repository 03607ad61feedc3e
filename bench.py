#!/usr/bin/env python
"""bench.py -- SAM-PT hot path throughput on one H100 (DESIGN.md §measurement).

  python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--config C2|C1|...] [--dump-outputs DIR]

A "step" = one pass of the hot path (PIPS track -> SAM ViT encode -> prompt+mask decode with 12 refinements) over one
synthetic clip.  Headline workload = BASELINE config C2: 50 frames 480x854, SAM ViT-H + PIPS, 1 mask x 8 positive points.
`value`  : frames/s with the uint8 clip already resident in HBM (CUDA events, max over ranks).
`e2e`    : frames/s through the public API `SamPt.forward(video)` with the clip in pinned HOST memory (H2D inside the timed
           region) and the result summary (scores + trajectories + visibilities) read back D2H.
`--impl reference`: the reference's own CPU path (oracle port: reference PIPS restated + SAM restated, torch CPU, all host
           threads) on a bounded sample of the same workload.
`--dump-outputs DIR`: after the timed steps, the arrays the last resident step returned (trajectories, visibilities, per-frame
           scores, and a fixed seeded sample of the mask logits) are written as DIR/<name>.npy so that two builds can be
           compared output for output; inputs and weights are seeded, so they are identical from run to run.  The -inf of
           an empty mask is written as a finite stand-in and flagged in DIR/<name>_empty.npy (see dump_outputs).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
for _p in (ROOT, os.path.join(ROOT, "sam-pt_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import torch  # noqa: E402

CONFIGS = {
    # name: (T, H, W, vit, P)
    "C1": (2, 240, 320, "vit_b", 4),
    "C2": (50, 480, 854, "vit_h", 8),
    "C2b": (50, 480, 854, "vit_b", 8),
    "C2p": (4, 480, 854, "vit_h", 8),   # profiling-sized slice of C2 (ncu launch lists)
    "C3": (50, 480, 854, "vit_h", 64),  # BASELINE configs[2]: CoTracker (window 8), 64 query points
    "C5": (100, 1080, 1920, "vit_h", 256),  # BASELINE configs[4]: HQ-SAM ViT-H + CoTracker, 256 points (HBM-pressure stress)
}
TRACKER = {"C3": "cotracker", "C5": "cotracker"}   # every other config tracks with PIPS
HQ_SAM = {"C5"}                                    # configs that use segment_anything_hq (MaskDecoderHQ + early ViT features)
SAM_SEED, PIPS_SEED = 7202, 7201
PRECISION_NAMES = {1: "f16 (fp32 accumulate)", 2: "f16 x (f16 hi+lo weights), 2 passes (fp32 accumulate)",
                   3: "f16 hi+lo split (3 passes MLP, 2 passes qkv/proj)", 4: "f16 hi+lo split x3 (~fp32)",
                   5: "f16 hi+lo split (3 passes MLP + proj, 2 passes qkv)",
                   6: "f16 hi.hi + two e4m3 correction passes (~fp32 products) qkv/MLP, f16 hi+lo x3 elsewhere"}
COT_COORD_SCALE = 0.001   # synth.condition_cotracker: contractive over the 12 chained windows of a 50-frame clip
COT_VIS_BIAS = 0.6   # synth.condition_cotracker: ~90 % of the C3 / C5 query points visible (see its docstring)


def _peaks():
    """Peaks the roofline fractions divide by: MEASURED_PEAKS.json when present, else NVIDIA's H100 SXM data sheet (dense, for
    a card allowed 700 W; a power-limited card reaches less).  A data-sheet figure is a ceiling, never a measured rate."""
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return {"hbm_gbs": d.get("hbm_gbs", 3350.0), "bf16_tflops": d.get("bf16_tflops", 989.0),
                "bf16_tflops_sustained": d.get("bf16_tflops_sustained"), "src": "measured (MEASURED_PEAKS.json)"}
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "bf16_tflops_sustained": None, "src": "H100 SXM data sheet (dense, 700 W)"}


def _frac(a, b):
    return a / b if b else None


class ClockSampler:
    """nvidia-smi clocks + throttle reasons sampled DURING the timed region."""

    def __init__(self, index=0):
        self.index = index
        self.rows = []
        self._stop = threading.Event()
        self._t = None

    def _run(self):
        q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
             "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")
        while not self._stop.is_set():
            try:
                out = subprocess.run(["nvidia-smi", f"--id={self.index}", f"--query-gpu={q}", "--format=csv,noheader,nounits"],
                                     capture_output=True, text=True, timeout=5).stdout.strip()
                if out:
                    self.rows.append([c.strip() for c in out.split(",")])
            except Exception:
                pass
            self._stop.wait(0.2)

    def __enter__(self):
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()
        return self

    def __exit__(self, *a):
        self._stop.set()
        self._t.join(timeout=3)

    def summary(self):
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in self.rows:
            try:
                sm.append(float(r[0])); mx.append(float(r[1]))
            except Exception:
                continue
            for n, v in zip(names, r[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(n)
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None, "reasons": sorted(reasons),
                "samples": len(sm)}


def make_weights(vit, hq=False):
    """Seeded synthetic checkpoints, shapes taken from the product modules themselves (same tables as the oracle's)."""
    from sampt_b200 import factory, synth
    from sam_pt.point_tracker.pips.pips import _pips_shapes
    sam = factory.build_sam(vit, hq=hq)
    shapes = {k: tuple(v.shape) for k, v in sam.state_dict().items()}
    sam_sd = synth.condition_sam(synth.make_state_dict(shapes, SAM_SEED))
    pips_sd = synth.condition_pips(synth.make_state_dict(_pips_shapes(8), PIPS_SEED))
    return sam_sd, pips_sd


def run_ours(args):
    import torch.distributed as dist
    from sampt_b200 import factory, synth, native

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    T, H, W, vit, P = CONFIGS[args.config]
    hq = args.config in HQ_SAM
    sam_sd, pips_sd = make_weights(vit, hq=hq)
    tmp = tempfile.mkdtemp(prefix="sampt_bench_")
    ckpt = synth.write_pips_checkpoint_dir(pips_sd, os.path.join(tmp, "pips"))
    tracker = TRACKER.get(args.config, "pips")
    cot_sd = None
    if tracker == "cotracker":
        from sam_pt.point_tracker.cotracker.cotracker import cotracker_shapes
        cot_sd = synth.condition_cotracker(synth.make_state_dict(cotracker_shapes(), PIPS_SEED + 1), vis_bias=COT_VIS_BIAS, coord_scale=COT_COORD_SCALE)
        if not os.path.exists(os.path.join(ROOT, "tests", "golden", f"{args.config}_full_cpu.json")):
            args.no_cpu_baseline = True   # no measured full-clip CPU run committed for this configuration
    model = factory.build_sam_pt(vit, sam_sd, ckpt, positive_points_per_mask=P, sam_iou_threshold=-1e9, device=dev, hq=hq,
                                 cotracker_state_dict=cot_sd)
    model.sam_predictor.model.image_encoder.precision = args.precision
    model.encoder_batch = args.encoder_batch
    if world > 1 and args.mgpu_mode == "frame_shard":
        return run_ours_frame_sharded(args, model, dev, rank, world, local)
    # clip-per-GPU: every rank processes its own clip (seed 72 + rank), no data-path collective
    video = synth.make_video_dict(T, H, W, P, seed=72 + rank)
    frames_host = torch.stack(video["image"]).pin_memory()
    q_host = video["query_points"].pin_memory()
    ctx = native.get_context(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)  # > L2 (50 MB): flushed between timed iterations

    def step_resident(frames_dev, q_dev):
        traj, vis, logits, scores, spf = model._forward(frames_dev, q_dev)
        return logits, spf, traj, vis

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    # ---------------- warm-up
    frames_dev = frames_host.to(dev)
    q_dev = q_host.to(dev)
    for _ in range(max(args.warmup, 1)):
        step_resident(frames_dev, q_dev)
    torch.cuda.synchronize()

    # ---------------- timed: resident inputs
    launches0 = ctx.launch_count()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
    with ClockSampler(local) as clk:
        barrier()
        for i in range(args.steps):
            flush.fill_(i & 0xFF)
            ev[i][0].record()
            last = step_resident(frames_dev, q_dev)
            ev[i][1].record()
        barrier()
    ms = sum(a.elapsed_time(b) for a, b in ev)
    launches = ctx.launch_count() - launches0
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, last)
    # ---------------- timed: end to end through SamPt.forward with HOST inputs + D2H result summary
    video_host = dict(video)
    video_host["image"] = [f for f in frames_host]
    video_host["query_points"] = q_host
    model(video_host)  # warm
    torch.cuda.synchronize()
    ev2 = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
    barrier()
    d2h = 0
    for i in range(args.steps):
        flush.fill_(i & 0xFF)
        ev2[i][0].record()
        out = model(video_host)   # reference contract: logits / trajectories / visibilities come back as HOST tensors (sam_pt.py:863-864)
        ev2[i][1].record()
        assert all(not l.is_cuda for l in out["logits"]) and not out["trajectories"].is_cuda
        d2h = sum(l.numel() * l.element_size() for l in out["logits"]) + out["trajectories"].numel() * 4 + out["visibilities"].numel() * 4 \
            + 8 * (len(out["scores"]) + T)
    barrier()
    ms_e2e = sum(a.elapsed_time(b) for a, b in ev2)
    t = torch.tensor([ms, ms_e2e], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms, ms_e2e = t.tolist()

    breakdown = stage_breakdown(model, frames_dev, q_dev) if args.breakdown else None
    if args.kernel_table and rank == 0:
        kernel_table(lambda: step_resident(frames_dev, q_dev), args.kernel_table)
    # ---------------- roofline of the dominant kernel (ViT tensor-core GEMM), measured live with CUDA events
    roof = gemm_roofline(model, dev, args)
    if rank == 0 and world == 1:
        roof["in_step"] = in_step_share(lambda: step_resident(frames_dev, q_dev), T, vit)
    cpu_base = None
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        cpu_base = cpu_baseline(args.config, sample_frames=args.cpu_sample_frames)
    if rank == 0:
        frames_total = T * world * args.steps
        line = {
            "metric": "frames/sec, SAM-PT hot path (PIPS track + SAM ViT encode + prompt/mask decode w/ 12 refinements)",
            "value": frames_total / (ms / 1e3), "unit": "frames/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": PRECISION_NAMES[args.precision] + " ViT; f32 PIPS + decoder",
            "data": "synthetic",
            "config": {"workload": f"{args.config}: {T} frames {H}x{W}, {'HQ-' if hq else ''}SAM {vit} + {'CoTracker (S=8, stride 4, interp 384x512)' if tracker == 'cotracker' else 'PIPS (S=8, stride 4)'}, 1 mask x {P} points, "
                                   f"12 refinement iterations, random-init conditioned weights",
                       "clips_per_step": world, "parallelism": f"clip-per-GPU x{world}" if world > 1 else "single GPU",
                       "l2": "flushed between timed iterations (256 MiB write)", "vit_precision_passes": args.precision,
                       "encoder_batch": args.encoder_batch},
            "e2e": {"value": frames_total / (ms_e2e / 1e3), "unit": "frames/s",
                    "h2d_bytes_per_step": int(frames_host.numel() + q_host.numel() * 4), "d2h_bytes_per_step": int(d2h)},
            "gpu_launches": int(launches),
            "clocks": clk.summary(),
            "roofline": roof,
            "roofline_attention": attn_roofline(dev) if vit == "vit_h" else None,
            "roofline_corr_gather": corr_roofline(dev),
            "cpu_baseline": cpu_base,
        }
        if breakdown:
            line["breakdown_ms"] = breakdown
        print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()


def run_ours_frame_sharded(args, model, dev, rank, world, local):
    """N > 1, BASELINE config C4 shape: `world` clips per step, frames of every clip sharded round-robin over the ranks,
    one NCCL all-gather of the PIPS feature maps (SamPt.forward_clips_sharded).  Weak scaling: clips/step == ranks."""
    import torch.distributed as dist
    from sampt_b200 import native, synth
    from sampt_b200 import sharding
    T, H, W, vit, P = CONFIGS[args.config]
    tracker = TRACKER.get(args.config, "pips")
    # clips per step: one per rank (weak scaling, BASELINE configs[3]) unless the configuration is ONE clip spread over the GPUs
    # (BASELINE configs[4]: a single 100-frame 1080p clip on 8 GPUs -> strong scaling)
    n_clips = args.clips_per_step if args.clips_per_step > 0 else (1 if args.config == "C5" else world)
    videos = [synth.make_video_dict(T, H, W, P, seed=72 + c) for c in range(n_clips)]
    host = [dict(v, image=[f.pin_memory() for f in v["image"]]) for v in videos]
    resident = [dict(v, image=[f.to(dev) for f in v["image"]], query_points=v["query_points"].to(dev)) for v in videos]
    ctx = native.get_context(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def barrier():
        dist.barrier()
        torch.cuda.synchronize()

    for _ in range(max(args.warmup, 1)):
        model.forward_clips_sharded(resident)
    torch.cuda.synchronize()

    def timed(inputs, readback):
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
        nbytes = 0
        barrier()
        for i in range(args.steps):
            flush.fill_(i & 0xFF)
            ev[i][0].record()
            res = model.forward_clips_sharded(inputs)
            if readback:
                summ = [(r["trajectories"].cpu(), r["visibilities"].cpu(), r["scores_per_frame"].cpu(),
                         r["logits"].cpu()) for r in res]   # the masks of the frames this rank owns come back to the host
                nbytes = sum(t.numel() * t.element_size() for tup in summ for t in tup)
            ev[i][1].record()
        barrier()
        return sum(a.elapsed_time(b) for a, b in ev), nbytes

    l0 = ctx.launch_count()
    with ClockSampler(local) as clk:
        ms, _ = timed(resident, False)
    launches = ctx.launch_count() - l0
    model.forward_clips_sharded(host)
    ms_e2e, d2h = timed(host, True)
    t = torch.tensor([ms, ms_e2e], device=dev, dtype=torch.float64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms, ms_e2e = t.tolist()
    roof = gemm_roofline(model, dev, args)
    if rank == 0:
        frames_total = T * n_clips * args.steps
        own = sum(len(sharding.owned_frames(T, rank, world, c)) for c in range(n_clips))
        line = {
            "metric": "frames/sec, SAM-PT hot path (PIPS track + SAM ViT encode + prompt/mask decode w/ 12 refinements)",
            "value": frames_total / (ms / 1e3), "unit": "frames/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak" if n_clips == world else "strong", "vs_baseline": None,
            "dtype": PRECISION_NAMES[args.precision] + " ViT; f32 tracker + decoder",
            "data": "synthetic",
            "config": {"workload": f"{n_clips} x {args.config}: {T} frames {H}x{W}, {'HQ-' if args.config in HQ_SAM else ''}SAM {vit} + {tracker}, 1 mask x {P} points, 12 refinements; "
                                   f"frame f of clip c on rank (f + c) mod {world}, one NCCL all-gather of the fp32 tracker feature maps",
                       "clips_per_step": n_clips, "parallelism": f"frame-shard x{world} + all-gather",
                       "l2": "flushed between timed iterations (256 MiB write)", "vit_precision_passes": args.precision,
                       "encoder_batch": args.encoder_batch},
            "e2e": {"value": frames_total / (ms_e2e / 1e3), "unit": "frames/s",
                    "h2d_bytes_per_step": int(own * 3 * H * W + n_clips * P * 12), "d2h_bytes_per_step": int(d2h)},
            "gpu_launches": int(launches), "clocks": clk.summary(), "roofline": roof, "cpu_baseline": None,
        }
        print(json.dumps(line))
    dist.destroy_process_group()


DUMP_LOGITS_SAMPLE = 1 << 22   # logits elements kept by --dump-outputs (16 MB of float32; a C2 clip has 20.5 M)


DUMP_EMPTY_FILL = -1.0e4   # finite stand-in for the -inf of an empty mask in the dumped arrays (flagged in <name>_empty.npy)


def dump_outputs(path, result):
    """result = (logits, scores_per_frame, trajectories, visibilities) of one step -> path/<name>.npy (float32).  The logits
    are sampled at fixed, seeded positions (the same for every run of the same configuration).  A frame whose query points are
    all invisible has an empty mask: its logits and score are -inf, as in the reference (sam_pt.py:766).  The dump stays
    finite and lossless: such entries are written as DUMP_EMPTY_FILL and marked 1 in <name>_empty.npy.  Any other non-finite
    output (NaN, +inf) is an error."""
    import numpy as np
    logits, spf, traj, vis = result
    os.makedirs(path, exist_ok=True)
    flat = logits.detach().float().reshape(-1)
    if flat.numel() > DUMP_LOGITS_SAMPLE:
        g = torch.Generator(device="cpu").manual_seed(0)
        idx = torch.randperm(flat.numel(), generator=g)[:DUMP_LOGITS_SAMPLE].sort().values
        flat = flat[idx.to(flat.device)]
    arrays = {"logits_sample": flat, "scores_per_frame": spf, "trajectories": traj, "visibilities": vis}
    for name, t in arrays.items():
        a = t.detach().float().cpu().numpy().astype(np.float32)
        empty = np.isneginf(a)
        bad = ~np.isfinite(a) & ~empty
        if bad.any():
            raise RuntimeError(f"--dump-outputs: {name} has {int(bad.sum())} NaN / +inf values")
        if name in ("logits_sample", "scores_per_frame"):
            np.save(os.path.join(path, name + "_empty.npy"), empty.astype(np.float32))
            a = np.where(empty, np.float32(DUMP_EMPTY_FILL), a)
        elif empty.any():
            raise RuntimeError(f"--dump-outputs: {name} has {int(empty.sum())} -inf values")
        np.save(os.path.join(path, name + ".npy"), a)


def kernel_table(step_fn, path):
    """Per-kernel device time of one step via CUPTI (torch.profiler sees every kernel of the process, including the ones
    launched through the C ABI).  Not a bench value; written for profiles/."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step_fn()
        torch.cuda.synchronize()
    rows = []
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = getattr(e, "cuda_time_total", 0.0)
        if t > 0:
            rows.append((e.key, e.count, t))
    rows.sort(key=lambda r: -r[2])
    tot = sum(r[2] for r in rows)
    with open(path, "w") as f:
        f.write(f"# per-kernel device time of one step (CUPTI via torch.profiler); total {tot / 1e3:.2f} ms\n\n")
        f.write("| kernel | launches | total ms | mean us | share |\n|---|---:|---:|---:|---:|\n")
        for k, c, t in rows[:60]:
            f.write(f"| `{k[:110]}` | {c} | {t / 1e3:.2f} | {t / c:.1f} | {100 * t / tot:.1f}% |\n")


def in_step_share(step_fn, frames_per_step, vit, pattern="gemm_tc_kernel"):
    """Cross-check of the isolated roofline timing against the real step (VERDICT r1 #4): one extra, untimed step under CUPTI
    (torch.profiler); all launches of the dominant kernel are summed.  `achieved_algorithmic` uses SURVEY §8d's 5.48 TFLOP of
    linear-layer work per ViT-H frame (what the reference computes; the padding-window skip removes ~8 % of it from the launches)."""
    try:
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step_fn()
            torch.cuda.synchronize()
        tot = ker = 0.0
        n = 0
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = getattr(e, "cuda_time_total", 0.0)
            if t <= 0:
                continue
            tot += t
            if pattern in e.key:
                ker += t
                n += e.count
        out = {"kernel": pattern, "launches_per_step": int(n), "ms_per_step": ker / 1e3, "share_of_device_time": (ker / tot) if tot else None,
               "device_ms_per_step_all_kernels": tot / 1e3, "how": "one extra untimed step under CUPTI (torch.profiler)"}
        if vit == "vit_h" and ker > 0:
            pk = _peaks()
            ach = frames_per_step * 5.48 / (ker / 1e6)   # TFLOP / s
            out.update({"achieved_algorithmic": ach, "unit": "TFLOP/s", "frac_of_sustained_peak": _frac(ach, pk["bf16_tflops_sustained"]),
                        "frac_of_burst_peak": ach / pk["bf16_tflops"]})
        return out
    except Exception as e:   # a profiler problem must never cost the bench line
        return {"error": f"{type(e).__name__}: {e}"}


def stage_breakdown(model, frames_dev, q_dev):
    """Per-stage device time of one step (CUDA events; separate untimed pass, for DESIGN/PROFILE notes only)."""
    pred = model.sam_predictor
    trk = model.point_tracker
    T = frames_dev.shape[0]

    def timed(fn):
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        r = fn()
        b.record()
        torch.cuda.synchronize()
        return r, a.elapsed_time(b)

    out = {}
    pyr, out["pips_fnet_pyramid"] = timed(lambda: trk.model.encode_frames(frames_dev))
    q = q_dev.reshape(-1, 3).float().to(frames_dev.device)
    _, out["pips_chain"] = timed(lambda: trk.model.track(pyr, q, 0.9, iters=6, flip=False))
    B = model.encoder_batch
    t_res = t_vit = 0.0
    feats = None
    for f0 in range(0, T, B):
        r, ms = timed(lambda: pred.resize_frames_u8(frames_dev[f0:f0 + B]))
        t_res += ms
        m = pred.model
        feats, ms = timed(lambda: m.image_encoder.encode_resized_u8(r, m.pixel_mean.flatten().tolist(), m.pixel_std.flatten().tolist()))
        t_vit += ms
    out["sam_resize"], out["sam_vit_encode"] = t_res, t_vit
    pred.set_frames_features(tuple(frames_dev.shape[-2:]), feats[:1])
    c = torch.rand((q.shape[0], 2), device=frames_dev.device) * 500
    lab = torch.ones((q.shape[0],), dtype=torch.int32, device=frames_dev.device)
    lg = torch.empty(tuple(frames_dev.shape[-2:]), device=frames_dev.device)
    pred.predict_refine(c, lab, 0, 12, lg)
    _, ms = timed(lambda: [pred.predict_refine(c, lab, 0, 12, lg) for _ in range(5)])
    out["sam_decode_13calls_per_frame"] = ms / 5
    out["sam_decode_clip_estimate"] = ms / 5 * T
    return {k: round(v, 3) for k, v in out.items()}


ROOFLINE_WARM, ROOFLINE_REPS = 3, 10


def corr_roofline(dev, n_points=292):
    """Secondary roofline entry: the fused PIPS correlation gather (pips_corr lookup) at a large point count
    (C5-like: 256 queries + 36 support points), where it is bandwidth- rather than latency-bound.  Algorithmic bytes =
    N * S * L * 64 px * 128 ch * 4 B = N x 1 MiB per launch (SURVEY §8d, minimal formulation)."""
    from ctypes import c_int
    from sampt_b200 import native
    S, H4, W4 = 8, 120, 213
    g = torch.Generator(device="cpu").manual_seed(0)
    lv = [torch.randn((S, H4 >> l, W4 >> l, 128), generator=g).to(dev) for l in range(4)]
    ff = torch.randn((n_points, S, 128), generator=g).to(dev)
    cc = (torch.rand((n_points, S, 2), generator=g) * torch.tensor([W4 - 1.0, H4 - 1.0])).to(dev)
    out = torch.empty((n_points, S, 196), device=dev)
    ctx = native.get_context(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def run():
        native.check(native.lib().sampt_pips_corr_lookup(ctx.handle, native.ptr(lv[0]), native.ptr(lv[1]), native.ptr(lv[2]),
                                                         native.ptr(lv[3]), c_int(S), c_int(H4), c_int(W4), native.ptr(ff),
                                                         native.ptr(cc), c_int(n_points), native.ptr(out), native.stream_ptr()))
    for _ in range(ROOFLINE_WARM):
        run()
    torch.cuda.synchronize()
    times = []
    for i in range(ROOFLINE_REPS):
        flush.fill_(i)  # evict the pyramid from L2 so the gather is served by HBM
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    ms = sorted(times)[len(times) // 2]
    nbytes = n_points * S * 4 * 64 * 128 * 4 + n_points * S * 196 * 4
    pk = _peaks()
    gbs = nbytes / (ms * 1e-3) / 1e9
    return {"bound": "hbm", "kernel": "pips_corr_kernel (the tracker's fused correlation gather + mixer-row assembly, N=%d points; the "
                                     "timed call adds a 1.8 MB strided copy-out of the 196 correlation columns)" % n_points,
            # the 8x8 patches of neighbouring levels / slots overlap: part of the N x 1 MiB "minimal formulation" is served by L2
            "achieved": gbs, "peak": pk["hbm_gbs"], "unit": "GB/s", "frac": gbs / pk["hbm_gbs"], "ms": ms,
            "peak_source": pk["src"], "algorithmic_bytes": nbytes, "l2": "flushed before every launch"}


def attn_roofline(dev, frames=10, nheads=16, hd=80):
    """The north-star kernel: the ViT-H attention launches of one 10-frame encoder batch, timed in isolation with CUDA events.
    windowed: 25 windows x 16 heads per frame, 14x14 = 196 tokens (operands pre-extended: DK = 80 + 2*14 -> 128);
    global  : 16 heads per frame, 64x64 = 4096 tokens (DK = 80 + 2*64 -> 256).
    Algorithmic FLOPs (SURVEY §8d) = 4 * L^2 * hd per (window, head): the QK^T and P.V contractions at the true head dim, without
    the rel-pos extension columns or tile padding; `issued` counts what the tensor pipe executes (DK-wide QK^T, 128-row query tiles,
    64-key tiles)."""
    from ctypes import c_int
    from sampt_b200 import native
    ctx = native.get_context(dev)
    L_ = native.lib()
    pk = _peaks()
    out = {}
    g = torch.Generator(device="cpu").manual_seed(1)
    for name, BH, L, DK, NT in (("windowed", frames * 25 * nheads, 196, 128, 208), ("global", frames * nheads, 4096, 256, 128)):
        Lkp = ((L + 63) // 64) * 64
        Q = (torch.randn((min(BH, 64), L, DK), generator=g) * 0.3).half().to(dev)
        reps = (BH + Q.shape[0] - 1) // Q.shape[0]
        Q = Q.repeat(reps, 1, 1)[:BH].contiguous()
        K = Q.flip(0).contiguous()
        V = torch.randn((BH, hd, Lkp), device=dev).half()
        V[:, :, L:] = 0
        o = torch.empty((BH // nheads * L, nheads * hd), device=dev, dtype=torch.float16)

        def run():
            native.check(L_.sampt_attention_f16(ctx.handle, native.ptr(Q), native.ptr(K), native.ptr(V), c_int(BH), c_int(L), c_int(L), c_int(Lkp),
                                                c_int(DK), c_int(hd), c_int(NT), c_int(nheads), native.ptr(o), c_int(nheads * hd), c_int(0),
                                                native.stream_ptr()), "attention")
        for _ in range(ROOFLINE_WARM):
            run()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = max(1, ROOFLINE_REPS // 2)
        e0.record()
        for _ in range(n):
            run()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / n
        alg = 4.0 * L * L * hd * BH
        mt = ((L + 127) // 128) * 128
        issued = 2.0 * mt * (((L + 63) // 64) * 64) * (DK + hd) * BH
        ach = alg / (ms * 1e-3) / 1e12
        out[name] = {"bound": "tensor", "kernel": "attention (ViT-H %s, %d (window, head) units of %d tokens)" % (name, BH, L), "achieved": ach,
                     "peak": pk["bf16_tflops"], "unit": "TFLOP/s", "frac": ach / pk["bf16_tflops"],
                     "achieved_issued": issued / (ms * 1e-3) / 1e12, "frac_issued": issued / (ms * 1e-3) / 1e12 / pk["bf16_tflops"], "ms": ms,
                     "algorithmic_flops": alg, "operands_bytes": int(Q.numel() * 2 * 2 + V.numel() * 2 + o.numel() * 2),
                     "peak_source": pk["src"]}
        del Q, K, V, o
    return out


def gemm_roofline(model, dev, args):
    """Times the ViT's largest GEMM shape (mlp.lin1: M=B*4096, N=4D, K=D) in isolation with CUDA events."""
    from ctypes import c_int
    from sampt_b200 import native
    enc = model.sam_predictor.model.image_encoder
    D, B = enc.embed_dim, args.encoder_batch
    M, N, K = B * 4096, 4 * D, D
    f8c = args.precision == 6                  # fp16 hi.hi pass + two e4m3 correction passes at twice the rate
    p = min(args.precision, 3)
    asp, bsp = (2 if p >= 3 else 1), (2 if p >= 2 else 1)
    out = torch.empty((M, N), device=dev, dtype=torch.float16)
    ctx = native.get_context(dev)
    L = native.lib()
    if f8c:
        x = torch.randn((M, K), device=dev)
        A = torch.empty((M, 2 * K), device=dev, dtype=torch.float16)
        native.check(L.sampt_split_f8c(ctx.handle, native.ptr(x), c_int(M), c_int(K), native.ptr(A), native.stream_ptr()))
        from segment_anything.modeling.image_encoder import ImageEncoderViT
        Wt, w_scale = ImageEncoderViT._w8(torch.randn((N, K), device=dev) * 0.02)

        def run():
            native.check(L.sampt_gemm_f8c(ctx.handle, native.ptr(A), native.ptr(Wt), c_int(M), c_int(N), c_int(K), native.ptr(w_scale),
                                          native.ptr(None), c_int(0), native.ptr(out), native.ptr(None), native.ptr(None), c_int(N),
                                          c_int(0), c_int(0), native.stream_ptr()))
    else:
        A = torch.randn((M, K * asp), device=dev).half()
        Wt = torch.randn((N, K * bsp), device=dev).half()

        def run():
            native.check(L.sampt_gemm_f16(ctx.handle, native.ptr(A), c_int(K * asp), native.ptr(Wt), c_int(K * bsp), c_int(M), c_int(N),
                                          c_int(K), c_int(p), c_int(0), native.ptr(None), c_int(0), native.ptr(out), native.ptr(None),
                                          native.ptr(None), c_int(N), c_int(0), native.stream_ptr()))
    for _ in range(ROOFLINE_WARM):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = ROOFLINE_REPS
    e0.record()
    for _ in range(n):
        run()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / n
    flops_alg = 2.0 * M * N * K           # algorithmic (what the layer needs)
    # tensor-core work actually issued, in fp16-pass equivalents: an e4m3 pass moves the same flops through the pipe in half
    # the cycles, so the fp8-corrected form costs 1 + 2 * 0.5 = 2 passes of fp16 pipe time
    passes_eq = 2.0 if f8c else float(p)
    flops_exec = flops_alg * passes_eq
    pk = _peaks()
    ach = flops_alg / (ms * 1e-3) / 1e12
    return {"bound": "tensor", "kernel": "gemm_tc_kernel (ViT mlp.lin1 shape)", "achieved": ach, "peak": pk["bf16_tflops"], "unit": "TFLOP/s",
            "frac": ach / pk["bf16_tflops"],                                    # ALGORITHMIC flops (2*M*N*K) / time / measured peak
            "achieved_issued": flops_exec / (ms * 1e-3) / 1e12,                 # tensor-core work issued incl. the split-precision passes
            "frac_issued": flops_exec / (ms * 1e-3) / 1e12 / pk["bf16_tflops"],
            # the same two against a SUSTAINED peak (measured back to back under the power cap) when MEASURED_PEAKS.json gives one
            "peak_sustained": pk["bf16_tflops_sustained"], "frac_of_sustained": _frac(ach, pk["bf16_tflops_sustained"]),
            "frac_issued_of_sustained": _frac(flops_exec / (ms * 1e-3) / 1e12, pk["bf16_tflops_sustained"]),
            "algorithmic_bytes": 2.0 * (M * K * asp + N * K * bsp + M * N),
            "peak_source": pk["src"], "shape": [M, N, K], "passes": ("1 fp16 + 2 e4m3 (= 2 fp16-pass equivalents)" if f8c else p), "ms": ms}


def usable_cores(cap=16):
    """CPU threads this process may really use: scheduler affinity, cgroup quota, capped (a 128-thread torch pool on a
    quota-limited container is ~50x slower than 8 threads: measured on the GPU box)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        q = open("/sys/fs/cgroup/cpu.max").read().split()
        if q[0] != "max":
            n = min(n, max(1, int(int(q[0]) / int(q[1]))))
    except Exception:
        pass
    try:  # cgroup v1
        quota = int(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
        period = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
        if quota > 0 and period > 0:
            n = min(n, max(1, quota // period))
    except Exception:
        pass
    return max(1, min(n, cap))


def cpu_baseline(config, sample_frames=2):
    """Reference CPU path on the host cores: the MEASURED full-clip run of the whole path recorded by
    tests/golden/make_golden_full.py (tests/golden/<config>_full_cpu.json: every frame of the clip, unmodified reference PIPS
    tracker + restated SAM, per-stage wall seconds on the build container's cores) -- no composition model, no subset.
    A full clip is ~10 min of CPU, so it is cached; on this host a bounded calibration sample (oracle/cpu_sample.py: one ViT
    frame, one frame's 13-call decode chain, the tracker encoder on 2 frames + one window; ~20-30 s) is re-timed and each cached
    stage is rescaled by (unit seconds here / unit seconds in the build container).  `value` = frames / rescaled total."""
    from oracle import cpu_sample
    T, H, W, vit, P = CONFIGS[config]
    tracker = TRACKER.get(config, "pips")
    cores = usable_cores()
    torch.set_num_threads(cores)
    cached_path = os.path.join(ROOT, "tests", "golden", f"{config}_full_cpu.json")
    live = cpu_sample.bounded_sample(H, W, P, tracker=tracker, hq=config in HQ_SAM, threads=cores, vit=vit)
    if not os.path.exists(cached_path):
        # configs without a committed full run (C1, profiling slices): the calibration sample alone, labelled as such
        per_frame = live["vit"] + live["decode"] + live["tracker"] / 2.0
        return {"value": 1.0 / per_frame, "unit": "frames/s", "cores": cores, "kind": "port",
                "sample": f"{config}: NO cached full-clip run; bounded sample only (ViT 1 frame {live['vit']:.1f}s + decode chain of 1 frame "
                          f"{live['decode']:.1f}s + tracker unit {live['tracker']:.1f}s / 2 frames)", "full_clip_measured": None}
    cached = json.load(open(cached_path))
    res = cpu_sample.rescale_full_run(cached, live)
    there = cached["calibration_sample"]
    return {"value": res["frames_per_s"], "unit": "frames/s", "cores": cores, "kind": "port" if tracker != "pips" else "reference+port",
            "sample": f"full {config}, cached: all {cached['frames_run']} frames measured once on {cached['threads']} threads of "
                      f"'{cached['cpu']}' = {cached['seconds']['total']:.0f} s ({cached['frames_per_s']:.4f} frames/s; tracker "
                      f"{cached['seconds']['tracker']:.0f} s [unmodified reference PipsPointTracker], ViT {cached['seconds']['sam_set_image']:.0f} s, "
                      f"decode {cached['seconds']['sam_decode']:.0f} s), rescaled per stage to this host's {cores} threads by a live "
                      f"calibration sample (ViT frame {live['vit']:.1f}s vs {there['vit']:.1f}s, decode chain {live['decode']:.1f}s vs "
                      f"{there['decode']:.1f}s, tracker unit {live['tracker']:.1f}s vs {there['tracker']:.1f}s)",
            "full_clip_measured": {"seconds": cached["seconds"], "frames_per_s": cached["frames_per_s"], "threads": cached["threads"],
                                   "cpu": cached["cpu"], "where": "build container (tests/golden/make_golden_full.py)"},
            "rescaled_seconds": res["seconds"], "live_sample_seconds": live}


def run_reference(args):
    """--impl reference: the reference's CPU path for the same config.  One live calibration sample per run (about 30 s of CPU);
    every `step` is the same deterministic clip, so the cached full-clip measurement (rescaled to this host) is the per-step
    time -- `fits_in_driver_run` is explained by that cache: a real full clip is ~10 min of CPU per step."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    T, H, W, vit, P = CONFIGS[args.config]
    base = cpu_baseline(args.config, sample_frames=args.cpu_sample_frames)
    v = base["value"]
    world = int(os.environ.get("WORLD_SIZE", "1"))
    tracker = TRACKER.get(args.config, "pips")
    line = {"impl": "reference", "metric": "frames/sec, SAM-PT hot path (PIPS track + SAM ViT encode + prompt/mask decode w/ 12 refinements)",
            "value": v, "unit": "frames/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": 1e3 * T / v, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": (f"{world} x " if world > 1 else "") +
                                   f"{args.config}: {T} frames {H}x{W}, SAM {vit} + {tracker}, 1 mask x {P} points, 12 refinement iterations "
                                   f"(CPU: one clip at a time on the host cores; {base['sample']})",
                       "cached_full_clip": base.get("full_clip_measured") is not None},
            "cpu_baseline": base, "e2e": {"value": v, "unit": "frames/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--config", default="C2", choices=sorted(CONFIGS))
    ap.add_argument("--precision", type=int, default=int(os.environ.get("SAMPT_VIT_PRECISION", "6")))
    ap.add_argument("--encoder-batch", type=int, default=10)
    ap.add_argument("--cpu-sample-frames", type=int, default=2)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--breakdown", action="store_true")
    ap.add_argument("--kernel-table", default=None, help="write a per-kernel time table of one step (CUPTI) to this path")
    ap.add_argument("--mgpu-mode", default="frame_shard", choices=["frame_shard", "clip_per_gpu"])
    ap.add_argument("--clips-per-step", type=int, default=0, help="N > 1: clips per step (default: one per rank; C5: a single clip)")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="write what the last timed step computed to DIR/<name>.npy (single-GPU clip path)")
    args = ap.parse_args()
    if args.impl == "reference":
        run_reference(args)
    else:
        run_ours(args)


if __name__ == "__main__":
    main()
