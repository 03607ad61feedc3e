#!/usr/bin/env python
"""Isolated kernel timings through the C ABI (CUDA events, median of 20, L2 not flushed): optimisation guidance only."""
import json
import os
import sys
from ctypes import c_int

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "sam-pt_b200")):
    sys.path.insert(0, p)
import torch  # noqa: E402
from sampt_b200 import native  # noqa: E402

dev = torch.device("cuda", 0)
ctx = native.get_context(dev)
L = native.lib()


def timeit(fn, n=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


out = {}
# ---- fp32 linear shapes
for (M, N, K) in [(64, 2048, 512), (64, 512, 2048), (64, 512, 520), (8, 1040, 512), (15, 256, 256), (15, 2048, 256), (15, 256, 2048),
                  (4096, 128, 256), (4096, 256, 128), (4096, 256, 256), (2336, 2048, 512), (2336, 512, 2048)]:
    x = torch.randn((M, K), device=dev); w = torch.randn((N, K), device=dev); b = torch.randn((N,), device=dev)
    y = torch.empty((M, N), device=dev)
    f = lambda: native.check(L.sampt_linear_f32(ctx.handle, native.ptr(x), c_int(K), native.ptr(w), c_int(K), native.ptr(b), native.ptr(None),
                                                c_int(0), native.ptr(y), c_int(N), c_int(M), c_int(N), c_int(K), c_int(0), native.stream_ptr()))
    us = timeit(f)
    out[f"linear_f32 M{M} N{N} K{K}"] = {"us": round(us, 1), "tflops": round(2 * M * N * K / us / 1e6, 2)}

# ---- tensor-core GEMM shapes (ViT-H, batch 10), precision 1 and 3
for (M, N, K) in [(49000, 3840, 1280), (49000, 1280, 1280), (40960, 5120, 1280), (40960, 1280, 5120), (40960, 256, 1280), (40960, 1280, 768)]:
    for p in (1, 3):
        asp, bsp = (2 if p >= 3 else 1), (2 if p >= 2 else 1)
        A = torch.randn((M, K * asp), device=dev).half(); W = torch.randn((N, K * bsp), device=dev).half()
        o = torch.empty((M, N), device=dev, dtype=torch.float16)
        f = lambda: native.check(L.sampt_gemm_f16(ctx.handle, native.ptr(A), c_int(K * asp), native.ptr(W), c_int(K * bsp), c_int(M), c_int(N),
                                                  c_int(K), c_int(p), c_int(0), native.ptr(None), c_int(0), native.ptr(o), native.ptr(None),
                                                  native.ptr(None), c_int(N), c_int(0), native.stream_ptr()))
        us = timeit(f, 10)
        out[f"gemm_tc p{p} M{M} N{N} K{K}"] = {"us": round(us, 1), "tflops_issued": round(2 * M * N * K * p / us / 1e6, 1)}
        del A, W, o

# ---- attention (ViT-H, 10 frames): windowed and global
for name, (BH, Lq, Lk, Lkp, DK, HD, NT, nh) in {"attn windowed": (10 * 25 * 16, 196, 196, 256, 128, 80, 208, 16),
                                                "attn global": (10 * 16, 4096, 4096, 4096, 256, 80, 128, 16)}.items():
    Q = torch.randn((BH, Lq, DK), device=dev).half() * 0.3; Kx = torch.randn((BH, Lk, DK), device=dev).half() * 0.3
    Vt = torch.randn((BH, HD, Lkp), device=dev).half()
    o = torch.empty(((BH // nh) * Lq, nh * HD), device=dev, dtype=torch.float16)
    f = lambda: native.check(L.sampt_attention_f16(ctx.handle, native.ptr(Q), native.ptr(Kx), native.ptr(Vt), c_int(BH), c_int(Lq), c_int(Lk),
                                                   c_int(Lkp), c_int(DK), c_int(HD), c_int(NT), c_int(nh), native.ptr(o), c_int(nh * HD), c_int(0),
                                                   native.stream_ptr()))
    us = timeit(f, 10)
    flops = 4.0 * BH * Lq * Lk * HD  # algorithmic (QK^T + PV at head_dim)
    out[name] = {"us": round(us, 1), "tflops_algorithmic": round(flops / us / 1e6, 1)}
    del Q, Kx, Vt, o

print(json.dumps(out, indent=1))
json.dump(out, open(os.path.join(ROOT, "gpurun_out", "microbench.json"), "w"), indent=1)
