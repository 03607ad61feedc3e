#!/usr/bin/env python
"""Times the ViT-H tensor-core GEMM launches of one 10-frame encoder batch at the default precision 6, each in isolation with
CUDA events over many back-to-back launches, at the row counts the pipeline really runs (csrc/vit_pipeline.cu):

  qkv / proj   49000 rows (all 25 windows of 14 x 14 per frame), 29400 (the 15 live windows of a 480 x 854 frame when the
               padding windows are skipped), 40960 (global blocks)
  lin1 / lin2  40960 rows (every token), 26880 (the 42 x 64 live tokens per frame)
  neck, patch embedding: 40960 rows, three fp16 passes (these shapes keep the fp16 split form)

Each launch gets the epilogue the pipeline gives it (bias, GELU + the chained e4m3 operand of lin2, in-place residual through
the window row map, pos_embed broadcast).  Reports us per launch, algorithmic TFLOP/s (2 M N K / time) and fp16-pass-equivalent
TFLOP/s (an e4m3 pass costs half an fp16 pass: precision 6 = 2 passes, three fp16 passes = 3), with the card name, power limit and
SM clock of the run.

usage: python tools/gemm_sweep.py --out DIR [--launches 20] [--repeats 5]
"""
import argparse
import json
import os
import subprocess
import sys
from ctypes import c_int

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "sam-pt_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)
import torch  # noqa: E402

D, B, G, WS = 1280, 10, 64, 14


def _e4m3(t):
    return t.clamp(-448.0, 448.0).to(torch.float8_e4m3fn).view(torch.uint8)


def _f8c_rows(x):
    hi = x.half()
    return torch.cat([hi.view(torch.uint8), _e4m3((x - hi.float()) * 4096.0), _e4m3(x * 0.125)], dim=1).contiguous().view(torch.float16)


def _window_map(ny, nx):
    """window-partitioned row -> token row of the frame batch (-1 = padding), ny x nx windows of WS x WS per frame"""
    L = WS * WS
    r = torch.arange(B * ny * nx * L)
    t, wb = r % L, r // L
    w, b = wb % (ny * nx), wb // (ny * nx)
    y, x = (w // nx) * WS + t // WS, (w % nx) * WS + t % WS
    return torch.where((y < G) & (x < G), b * G * G + y * G + x, torch.full_like(r, -1)).int()


def _live_token_map(rows_live):
    r = torch.arange(B * rows_live * G)
    return ((r // (rows_live * G)) * G * G + r % (rows_live * G)).int()


def launches():
    """(name, M, N, K, kind, epilogue) for one batch; kind "f8" = precision 6's fp8-corrected form, "p3" = three fp16 passes"""
    tok = B * G * G
    rows = []
    for name, M, rmap in (("all windows", B * 25 * WS * WS, _window_map(5, 5)), ("live windows", B * 15 * WS * WS, _window_map(3, 5)),
                          ("global", tok, None)):
        rows.append((f"qkv {name}", M, 3 * D, D, "f8", {"out": "16", "bias": True}))
        rows.append((f"proj {name}", M, D, D, "f8", {"out": "32", "bias": True, "resid": "inplace", "rowmap": rmap}))
    for name, M, rmap in (("all tokens", tok, None), ("live tokens", B * 42 * G, _live_token_map(42))):
        rows.append((f"lin1 {name}", M, 4 * D, D, "f8", {"out": "16", "bias": True, "act": 1, "chain_f8": True}))
        rows.append((f"lin2 {name}", M, D, 4 * D, "f8", {"out": "32", "bias": True, "resid": "inplace", "rowmap": rmap}))
    rows.append(("neck 1x1", tok, 256, D, "p3", {"out": "32"}))
    rows.append(("neck 3x3", tok, 256, 9 * 256, "p3", {"out": "32"}))
    rows.append(("patch embed", tok, D, 768, "p3", {"out": "32", "bias": True, "resid": "pos"}))
    return rows


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["sm_clock"], info["sm_clock_max"] = [s.strip() for s in q.split(",")]
    except Exception as e:   # the timings stand without it
        info["error"] = f"{type(e).__name__}: {e}"
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    from sampt_b200 import native
    from segment_anything.modeling.image_encoder import ImageEncoderViT
    dev = torch.device("cuda", 0)
    ctx = native.get_context(dev)
    L = native.lib()
    g =torch.Generator(device="cuda").manual_seed(0)
    x_tok = torch.randn((B * G * G, D), generator=g, device="cuda")
    results = []
    for name, M, N, K, kind, epi in launches():
        x = torch.randn((M, K), generator=g, device="cuda")
        w = torch.randn((N, K), generator=g, device="cuda") / K ** 0.5
        if kind == "f8":
            A = _f8c_rows(x)
            Bm, scale = ImageEncoderViT._w8(w)
            segs = [(0, 0, 0), (K, K, 1), (K + K // 2, K + K // 2, 1)]
        else:
            A = torch.cat([x.half(), (x - x.half().float()).half()], dim=1).contiguous()
            Bm = torch.cat([w.half(), (w - w.half().float()).half()], dim=1).contiguous()
            scale = None
            segs = [(0, 0, 0), (K, 0, 0), (0, K, 0)]
        del x, w
        bias = torch.randn((N,), generator=g, device="cuda") if epi.get("bias") else None
        o16 = o32 = resid = rowmap = None
        ldc, split_off, out_f8, resid_mod = N, 0, 0, 0
        if epi["out"] == "16":
            ldc = 2 * N if epi.get("chain_f8") else N
            split_off, out_f8 = (N, 1) if epi.get("chain_f8") else (0, 0)
            o16 = torch.empty((M, ldc), device="cuda", dtype=torch.float16)
        elif epi.get("resid") == "inplace":
            o32 = x_tok.clone() if N == D else torch.zeros((M, N), device="cuda")
            resid = o32
            rowmap = epi["rowmap"].cuda() if epi.get("rowmap") is not None else None
        else:
            o32 = torch.empty((M, N), device="cuda")
            if epi.get("resid") == "pos":
                resid, resid_mod = torch.randn((G * G, N), generator=g, device="cuda"), G * G
        arr = lambda i: (c_int * 3)(*[s[i] for s in segs])

        fn = lambda: native.check(L.sampt_test_gemm_tc(
            ctx.handle, native.ptr(A), c_int(A.shape[1]), native.ptr(Bm), c_int(Bm.shape[1]), c_int(M), c_int(N), c_int(K),
            c_int(len(segs)), arr(0), arr(1), arr(2), native.ptr(bias), c_int(epi.get("act", 0)), c_int(0), native.ptr(o16),
            native.ptr(o32), native.ptr(resid), c_int(resid_mod), native.ptr(rowmap), native.ptr(None), native.ptr(scale), c_int(ldc),
            c_int(split_off), c_int(out_f8), native.stream_ptr()), name)
        row = {"launch": name, "M": M, "N": N, "K": K, "kind": kind}
        flops = 2.0 * M * N * K
        passes = 2.0 if kind == "f8" else 3.0
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        per = []
        for _ in range(args.repeats):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.launches):
                fn()
            e1.record()
            torch.cuda.synchronize()
            per.append(e0.elapsed_time(e1) * 1e3 / args.launches)
        us = sorted(per)[len(per) // 2]
        row.update({"us": round(us, 1), "us_min": round(min(per), 1), "us_max": round(max(per), 1),
                    "tflops_algorithmic": round(flops / us / 1e6, 1), "tflops_fp16_pass_eq": round(flops * passes / us / 1e6, 1)})
        results.append(row)
        print(json.dumps(row), flush=True)
        del A, Bm, o16, o32, resid
        torch.cuda.empty_cache()
    out = {"card": card(), "batch_frames": B, "launches_per_timing": args.launches, "repeats": args.repeats, "timing": "median of repeats",
           "shapes": results}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "gemm_sweep.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out["card"]))


if __name__ == "__main__":
    main()
