"""GPU: the wgmma/TMA GEMM against a float64 torch reference of the same op (tolerances stated per mode)."""
from ctypes import c_int

import pytest
import torch

pytestmark = pytest.mark.gpu


def _run(A, B, M, N, K, precision=1, bf16=False, bias=None, act=0, out32=False, resid=None, split_off=0, ldc=None):
    from sampt_b200 import native
    ctx = native.get_context("cuda")
    ldc = ldc or N
    o16 = None if out32 else torch.zeros((M, ldc), device="cuda", dtype=torch.bfloat16 if bf16 else torch.float16)
    o32 = torch.zeros((M, ldc), device="cuda", dtype=torch.float32) if out32 else None
    native.check(native.lib().sampt_gemm_f16(
        ctx.handle, native.ptr(A), c_int(A.shape[1]), native.ptr(B), c_int(B.shape[1]), c_int(M), c_int(N), c_int(K),
        c_int(precision), c_int(1 if bf16 else 0), native.ptr(bias), c_int(act), native.ptr(o16), native.ptr(o32),
        native.ptr(resid), c_int(ldc), c_int(split_off), native.stream_ptr()), "gemm_f16")
    torch.cuda.synchronize()
    return o32 if out32 else o16


@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (128, 256, 256), (256, 512, 128), (4900, 3840, 1280), (300, 384, 128),
                                    (4096, 1280, 5120), (77, 96, 64)])
def test_gemm_fp16_single_pass(M, N, K):
    g = torch.Generator().manual_seed(M + N + K)
    A = (torch.randn((M, K), generator=g)).half().cuda()
    B = (torch.randn((N, K), generator=g) / K ** 0.5).half().cuda()
    bias = torch.randn((N,), generator=g).cuda()
    out = _run(A, B, M, N, K, bias=bias, out32=True)
    ref = A.double().cpu() @ B.double().cpu().T + bias.double().cpu()
    err = (out.cpu().double() - ref).abs().max().item()
    assert err < 2e-3 * max(1.0, ref.abs().max().item()) * 1e-1 + 1e-4, err  # fp32 accumulation of exact fp16 products


def test_gemm_bf16_and_gelu_fp16_out():
    M, N, K = 512, 512, 256
    g = torch.Generator().manual_seed(1)
    A = torch.randn((M, K), generator=g).bfloat16().cuda()
    B = (torch.randn((N, K), generator=g) / K ** 0.5).bfloat16().cuda()
    out = _run(A, B, M, N, K, bf16=True, act=1)
    ref = torch.nn.functional.gelu(A.double().cpu() @ B.double().cpu().T)
    assert (out.cpu().double() - ref).abs().max() < 3e-2  # bf16 output rounding


def test_gemm_residual_and_split_output():
    M, N, K = 384, 256, 128
    g = torch.Generator().manual_seed(2)
    A = torch.randn((M, K), generator=g).half().cuda()
    B = (torch.randn((N, K), generator=g) / K ** 0.5).half().cuda()
    resid = torch.randn((M, N), generator=g).cuda()
    out = _run(A, B, M, N, K, out32=True, resid=resid)
    ref = A.double().cpu() @ B.double().cpu().T + resid.double().cpu()
    assert (out.cpu().double() - ref).abs().max() < 1e-4
    # split fp16 output: hi|lo at column offset N reconstructs the fp32 value to ~2^-22
    o = _run(A, B, M, N, K, split_off=N, ldc=2 * N)
    rec = o[:, :N].double().cpu() + o[:, N:].double().cpu()
    ref = A.double().cpu() @ B.double().cpu().T
    assert (rec - ref).abs().max() < 2e-5


@pytest.mark.parametrize("precision", [2, 3])
def test_gemm_split_precision(precision):
    """operands carried as fp16 hi|lo: 3 passes reach ~fp32 accuracy for fp32 A and B; 2 passes are exact in B (weights)
    for fp16-representable A."""
    M, N, K = 640, 768, 512
    g = torch.Generator().manual_seed(3)
    A32 = torch.randn((M, K), generator=g)
    B32 = torch.randn((N, K), generator=g) / K ** 0.5
    if precision == 2:
        A32 = A32.half().float()  # activations are fp16 in this mode

    def split(x):
        hi = x.half()
        lo = (x - hi.float()).half()
        return torch.cat([hi, lo], dim=1).cuda()

    A = split(A32) if precision == 3 else A32.half().cuda()
    B = split(B32)
    out = _run(A, B, M, N, K, precision=precision, out32=True)
    ref = A32.double() @ B32.double().T
    err = (out.cpu().double() - ref).abs().max().item()
    assert err < 5e-5, err
    # and it must be far better than the single-pass result
    single = _run(A32.half().cuda(), B32.half().cuda(), M, N, K, out32=True)
    err1 = (single.cpu().double() - (A32.double() @ B32.double().T)).abs().max().item()
    assert err < err1 / 20


# ---------------------------------------------------------------------------------------------------------------------
# fp8-corrected split GEMM (include/sampt_b200.h: sampt_gemm_f8c): hi.hi in fp16 + the two 2^-12 correction terms in e4m3
def _pack_w8(w):
    from segment_anything.modeling.image_encoder import ImageEncoderViT
    return ImageEncoderViT._w8(w)


def _split_f8c(x):
    from sampt_b200 import native
    ctx = native.get_context("cuda")
    M, K = x.shape
    if K > 1536:   # the device entry is the ViT's LayerNorm kernel (rows <= 1536 wide): build wider operands with torch
        hi = x.half()
        e4 = lambda t: t.clamp(-448.0, 448.0).to(torch.float8_e4m3fn).view(torch.uint8)
        return torch.cat([hi.view(torch.uint8), e4((x - hi.float()) * 4096.0), e4(x * 0.125)], dim=1).contiguous().view(torch.float16)
    out = torch.empty((M, 2 * K), device="cuda", dtype=torch.float16)
    native.check(native.lib().sampt_split_f8c(ctx.handle, native.ptr(x), c_int(M), c_int(K), native.ptr(out), native.stream_ptr()), "split_f8c")
    return out


def _gemm_f8c(A, W8, scale, M, N, K, bias=None, act=0, out32=True, split_off=0, out_f8=0, ldc=None):
    from sampt_b200 import native
    ctx = native.get_context("cuda")
    ldc = ldc or N
    o16 = None if out32 else torch.zeros((M, ldc), device="cuda", dtype=torch.float16)
    o32 = torch.zeros((M, ldc), device="cuda", dtype=torch.float32) if out32 else None
    native.check(native.lib().sampt_gemm_f8c(
        ctx.handle, native.ptr(A), native.ptr(W8), c_int(M), c_int(N), c_int(K), native.ptr(scale), native.ptr(bias), c_int(act),
        native.ptr(o16), native.ptr(o32), native.ptr(None), c_int(ldc), c_int(split_off), c_int(out_f8), native.stream_ptr()), "gemm_f8c")
    torch.cuda.synchronize()
    return o32 if out32 else o16


def test_split_f8c_layout():
    """[fp16(x) | e4m3((x - fp16(x)) 2^12) | e4m3(x 2^-3)] byte for byte against torch's own e4m3 conversion."""
    g = torch.Generator().manual_seed(5)
    x = torch.randn((300, 256), generator=g) * torch.logspace(-3, 2, 256)[None, :]
    out = _split_f8c(x.cuda()).cpu()
    K = 256
    hi = x.half()
    assert torch.equal(out[:, :K], hi)
    raw = out[:, K:].contiguous().view(torch.uint8)
    lo8 = ((x - hi.float()) * 4096.0).clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8)
    hi8 = (x * 0.125).clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8)

    def same(a, b):   # +0 / -0 are both zero
        return bool(((a == b) | (((a & 0x7F) == 0) & ((b & 0x7F) == 0))).all())
    assert same(raw[:, :K], lo8) and same(raw[:, K:], hi8)


@pytest.mark.parametrize("M,N,K", [(512, 512, 256), (4900, 3840, 1280), (4096, 1280, 5120), (300, 256, 128)])
def test_gemm_f8c_accuracy(M, N, K):
    """relative rms error vs float64: ~1e-5 (emulated on the CPU: 1.0e-5), i.e. 20x below the two-pass form (2e-4) that the
    full-clip IoU bar rejects, at two fp16-pass equivalents of tensor work instead of three."""
    g = torch.Generator().manual_seed(M + N + K)
    x = torch.randn((M, K), generator=g)
    x[:, : K // 16] *= 8.0
    w = torch.randn((N, K), generator=g) * 0.02
    bias = torch.randn((N,), generator=g)
    W8, s = _pack_w8(w.cuda())
    out = _gemm_f8c(_split_f8c(x.cuda()), W8, s, M, N, K, bias=bias.cuda()).cpu().double()
    ref = x.double() @ w.double().T + bias.double()
    core = x.double() @ w.double().T
    rel = ((out - ref).pow(2).mean().sqrt() / core.pow(2).mean().sqrt()).item()
    assert rel < 3e-5, rel
    two_pass = x.half().double() @ w.double().T       # what dropping the A_lo term would give
    rel2 = ((two_pass - core).pow(2).mean().sqrt() / core.pow(2).mean().sqrt()).item()
    assert rel < rel2 / 8, (rel, rel2)


def test_gemm_f8c_chained_output_layout():
    """GELU epilogue writing the NEXT fp8-corrected GEMM's A operand (lin1 -> lin2 of the ViT MLP)."""
    M, K, Hn, N = 512, 256, 1024, 256
    g = torch.Generator().manual_seed(11)
    x = torch.randn((M, K), generator=g)
    w1 = torch.randn((Hn, K), generator=g) * 0.05
    w2 = torch.randn((N, Hn), generator=g) * 0.03
    W1, s1 = _pack_w8(w1.cuda())
    W2, s2 = _pack_w8(w2.cuda())
    h = _gemm_f8c(_split_f8c(x.cuda()), W1, s1, M, Hn, K, act=1, out32=False, split_off=Hn, out_f8=1, ldc=2 * Hn)
    href = torch.nn.functional.gelu(x.double() @ w1.double().T)
    assert (h[:, :Hn].cpu().double() - href).abs().max() < 2e-3          # the fp16 hi block
    exp = _split_f8c(href.float().cuda()).cpu()                            # layout of the byte blocks (values may differ by 1 ulp)
    raw, raw_exp = h.cpu()[:, Hn:].contiguous().view(torch.uint8).int(), exp[:, Hn:].contiguous().view(torch.uint8).int()
    hi8, hi8_exp = raw[:, Hn:], raw_exp[:, Hn:]
    assert ((hi8 - hi8_exp).abs() <= 1).float().mean() > 0.999          # e4m3(x/8) codes agree up to rounding ties
    out = _gemm_f8c(h, W2, s2, M, N, Hn).cpu().double()
    ref = href @ w2.double().T
    rel = ((out - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()
    assert rel < 5e-5, rel


# ---------------------------------------------------------------------------------------------------------------------
# gemm_tc with every GemmSeg / GemmEpi option (include/sampt_b200.h: sampt_test_gemm_tc).  The reference is float64 computed
# from exactly the operand values the kernel reads (fp16 / bf16 as stored, e4m3 bytes decoded), and each error is bounded per
# element by the magnitudes that enter it rather than by the largest output:
_U16 = 2.0 ** -21    # x sqrt(k16 steps) x sum_k |a_ik b_jk| over fp16 / bf16 segments: exact products; each k16 step of wgmma
                     # adds into the fp32 accumulator with up to ~2^-23 relative error (on H100 it truncates), a random walk
_U8 = 2.0 ** -8      # x the same sum over e4m3 segments (they carry 2^-12 of the result; their wgmma accumulates in < fp32)
_UEPI = 2.0 ** -20   # x the magnitudes the fp32 epilogue combines (scaled product, bias, GELU, residual)
_GELU_SLOPE = 1.13   # max |GELU'(x)| (erf and tanh forms)


def _e4m3(t):
    return t.clamp(-448.0, 448.0).to(torch.float8_e4m3fn).view(torch.uint8)


def _hilo(x):
    """fp32 -> [fp16 hi | fp16 lo] (vit_pipeline.cu make_seg operands)"""
    hi = x.half()
    return torch.cat([hi, (x - hi.float()).half()], dim=1).contiguous()


def _f8c_rows(x):
    """fp32 -> [fp16(x) | e4m3((x - fp16(x)) 2^12) | e4m3(x 2^-3)] (tc_api.cuh), built with torch"""
    hi = x.half()
    return torch.cat([hi.view(torch.uint8), _e4m3((x - hi.float()) * 4096.0), _e4m3(x * 0.125)], dim=1).contiguous().view(torch.float16)


# the pipelines' segment layouts (vit_pipeline.cu make_seg, tc_api.cuh make_seg_f8): (a_off, b_off, f8) per segment
def _segs(kind, K):
    return {"p1": [(0, 0, 0)], "p2": [(0, 0, 0), (0, K, 0)], "p3": [(0, 0, 0), (K, 0, 0), (0, K, 0)],
            "f8": [(0, 0, 0), (K, K, 1), (K + K // 2, K + K // 2, 1)]}[kind]


def _operands(x, w, kind):
    """fp32 activations x [M,K] and weights w [N,K] -> (A, B, segments, acc_scale) as the pipelines lay them out"""
    K = x.shape[1]
    if kind == "f8":
        W8, s = _pack_w8(w)
        return _f8c_rows(x), W8, _segs(kind, K), s
    A = _hilo(x) if kind == "p3" else x.half().contiguous()
    B = _hilo(w) if kind in ("p2", "p3") else w.half().contiguous()
    return A, B, _segs(kind, K), None


def _seg_values(X, off, K, f8):
    if f8:
        return X.view(torch.uint8)[:, 2 * off: 2 * off + K].contiguous().view(torch.float8_e4m3fn).double()
    return X[:, off: off + K].double()


def _product(A, B, segs, K):
    """float64 sum over segments of A_seg B_seg^T, and the error bound of its fp32 accumulation"""
    P = torch.zeros((A.shape[0], B.shape[0]), dtype=torch.float64, device=A.device)
    tol = torch.zeros_like(P)
    u16 = _U16 * (sum(K // 16 for _, _, f8 in segs if not f8)) ** 0.5
    for a_off, b_off, f8 in segs:
        a, b = _seg_values(A, a_off, K, f8), _seg_values(B, b_off, K, f8)
        P += a @ b.T
        tol += (_U8 if f8 else u16) * (a.abs() @ b.abs().T)
    return P, tol


def _epilogue_ref(P, tol, acc_scale=None, bias=None, act=0):
    """float64 value before the residual and its bound: (P * acc_scale + bias) -> GELU"""
    s = float(acc_scale.item()) if acc_scale is not None else 1.0
    v = P * s
    tol = tol * s + _UEPI * v.abs()
    if bias is not None:
        v = v + bias.double()
        tol = tol + _UEPI * bias.double().abs()
    if act == 1:
        v = 0.5 * v * (1.0 + torch.erf(v / 2.0 ** 0.5))
    elif act == 3:
        v = 0.5 * v * (1.0 + torch.tanh((2.0 / torch.pi) ** 0.5 * (v + 0.044715 * v ** 3)))
    if act:
        tol = _GELU_SLOPE * tol + _UEPI * v.abs()
    return v, tol


def _tc(A, B, M, N, K, segs, bias=None, act=0, bf16=False, out16=None, out32=None, resid=None, resid_mod=0, rowmap=None, skip=None,
        acc_scale=None, ldc=None, split_off=0, out_f8=0):
    """sampt_test_gemm_tc; returns the C return code (0 = ok) after synchronising"""
    from sampt_b200 import native
    ctx = native.get_context("cuda")
    arr = lambda i: (c_int * 3)(*[s[i] for s in segs], *[0] * (3 - len(segs)))
    rc = native.lib().sampt_test_gemm_tc(
        ctx.handle, native.ptr(A), c_int(A.shape[1]), native.ptr(B), c_int(B.shape[1]), c_int(M), c_int(N), c_int(K), c_int(len(segs)),
        arr(0), arr(1), arr(2), native.ptr(bias), c_int(act), c_int(1 if bf16 else 0), native.ptr(out16), native.ptr(out32),
        native.ptr(resid), c_int(resid_mod), native.ptr(rowmap), native.ptr(skip), native.ptr(acc_scale), c_int(ldc or N),
        c_int(split_off), c_int(out_f8), native.stream_ptr())
    torch.cuda.synchronize()
    return rc


def _assert_within(out, ref, tol, what):
    err = (out.double() - ref).abs()
    worst = (err / tol).max().item()
    print(f"{what}: max err {err.max().item():.3g}, worst err / bound {worst:.3g}")
    assert worst <= 1.0, (what, worst)


def _fp16_tol(ref):   # rounding of the fp16 output (+ the subnormal floor)
    return 2.0 ** -11 * ref.abs() + 2.0 ** -24


def _inputs(M, N, K, seed, xscale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((M, K), generator=g, device="cuda") * xscale
    x[:, : max(1, K // 16)] *= 8.0          # a few large channels, as LayerNorm outputs have
    w = torch.randn((N, K), generator=g, device="cuda") / K ** 0.5
    bias = torch.randn((N,), generator=g, device="cuda")
    return x, w, bias


def _vit_launches(model, D, B):
    """vit_pipeline.cu's gemm_tc launches for one frame batch: (site, M, N, K, segments), segments at the default precision 6
    ("f8" where gemm_f8c_applicable) and at precision 3 (qkv / proj weights split "p2", the rest "p3")"""
    tok, win = B * 4096, B * 4900          # 64 x 64 tokens per frame; 25 windows of 14 x 14 (zero-padded) per frame
    rows = [
        ("patch_embed", tok, D, 768, "p3"),            # patch embedding, K = 3 * 16 * 16
        ("qkv windowed", win, 3 * D, D, "f8"), ("qkv windowed", win, 3 * D, D, "p2"),
        ("qkv global", tok, 3 * D, D, "f8"), ("qkv global", tok, 3 * D, D, "p2"),
        ("proj windowed", win, D, D, "f8"), ("proj windowed", win, D, D, "p2"),
        ("proj global", tok, D, D, "f8"), ("proj global", tok, D, D, "p2"),
        ("lin1", tok, 4 * D, D, "f8"), ("lin1", tok, 4 * D, D, "p3"),
        ("lin2", tok, D, 4 * D, "f8"), ("lin2", tok, D, 4 * D, "p3"),
        ("neck 1x1", tok, 256, D, "p3"), ("neck 3x3", tok, 256, 9 * 256, "p3"),
    ]
    return [(f"vit_pipeline {model} B{B} {site}", M, N, K, kind) for site, M, N, K, kind in rows]


_LAUNCHES = (
    _vit_launches("ViT-B", 768, 1) + _vit_launches("ViT-B", 768, 2) + _vit_launches("ViT-H", 1280, 1) + _vit_launches("ViT-H", 1280, 2) + [
        # vit_pipeline.cu, padding-window skip of a 480x854 frame (15 live windows, 42 x 64 live tokens)
        ("vit_pipeline ViT-H live windows qkv", 15 * 196, 3840, 1280, "f8"),
        ("vit_pipeline ViT-H live tokens lin1", 42 * 64, 5120, 1280, "f8"),
        # pips_pipeline.cu:108 fnet conv1 (7x7 s2 on 3 channels, K padded to 192) and :46 conv_by_name (K = pad64(9 C_in))
        ("pips fnet conv1", 128 * 128, 64, 192, "p3"),
        ("pips fnet layer1 3x3 64->64", 128 * 128, 64, 576, "p3"),
        ("pips fnet layer2 3x3 64->96", 64 * 64, 96, 576, "p3"),
        ("pips fnet layer2 3x3 96->96", 64 * 64, 96, 896, "p3"),
        ("pips fnet layer2 1x1 downsample", 64 * 64, 96, 64, "p3"),
        ("pips fnet layer3 3x3 96->128", 32 * 32, 128, 896, "p3"),
        ("pips fnet layer3 1x1 downsample", 32 * 32, 128, 128, "p3"),
        ("pips fnet layer4 3x3 128->128", 16 * 16, 128, 1152, "p3"),
        ("pips fnet conv2 3x3 416->128", 64 * 64, 128, 3776, "p3"),
        # decoder.cu tcg: image-token projections, and token rows (M < 16)
        ("decoder tcg keys Wk", 4096, 128, 256, "p3"),
        ("decoder tcg i2t out", 4096, 256, 128, "p3"),
        ("decoder tcg upscale", 4096, 256, 256, "p3"),
        ("decoder tcg 7 token rows", 7, 256, 256, "p3"),
        ("decoder tcg 5 token rows", 5, 128, 256, "p3"),
        # cotracker.cu cot_tcg: UpdateFormer qkv / proj / fc1 / fc2 at 64 points x 8 slots
        ("cotracker qkv", 512, 1152, 384, "p3"), ("cotracker proj", 512, 384, 384, "p3"),
        ("cotracker fc1", 512, 1536, 384, "p3"), ("cotracker fc2", 512, 384, 1536, "p3"),
        # tails: M = 1 and around one 128-row tile, N = 32 and 160
        ("tail M=1", 1, 256, 128, "p1"), ("tail M=127", 127, 256, 128, "p3"), ("tail M=129", 129, 256, 128, "f8"),
        ("tail N=32", 300, 32, 64, "p1"), ("tail N=160", 300, 160, 128, "p3"),
    ])


def _distinct(rows):
    seen, out = set(), []
    for r in rows:
        if r[1:] not in seen:
            seen.add(r[1:])
            out.append(r)
    return out


@pytest.mark.parametrize("site,M,N,K,kind", _distinct(_LAUNCHES), ids=lambda v: str(v).replace(" ", "_"))
def test_gemm_tc_launch_shapes(site, M, N, K, kind):
    x, w, bias = _inputs(M, N, K, seed=M * 7 + N * 3 + K)
    A, B, segs, s = _operands(x, w, kind)
    out = torch.full((M, N), float("nan"), device="cuda")
    assert _tc(A, B, M, N, K, segs, bias=bias, out32=out, acc_scale=s) == 0
    P, tol = _product(A, B, segs, K)
    ref, tol = _epilogue_ref(P, tol, s, bias)
    _assert_within(out, ref, tol, f"{site} {kind}")
    # semantic: the split forms reach the fp32 product of x and w (p2: of fp16(x) and w)
    if kind != "p1":
        xs = x.half().double() if kind == "p2" else x.double()
        sem = xs @ w.double().T + bias.double()
        bound = (2.0 ** -14 if kind == "f8" else 2.0 ** -18) * (xs.abs() @ w.double().abs().T) + tol
        _assert_within(out, sem, bound, f"{site} {kind} vs fp32 x.w")


def _random_segments(M, N, K, f8s, seed):
    """A [M, lda], B [N, ldb] with one region of random operand values per segment (fp16 or e4m3 bytes), laid out in
    opposite orders in A and B"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    widths = [K // 2 if f8 else K for f8 in f8s]

    def region(rows, f8):
        v = torch.randn((rows, K), generator=g, device="cuda")
        return _e4m3(v * 4.0).view(torch.float16) if f8 else (v / K ** 0.5).half()
    a_parts = [region(M, f8) for f8 in f8s]
    b_parts = [region(N, f8) for f8 in f8s]
    a_off = [sum(widths[:i]) for i in range(len(f8s))]
    b_off = [sum(widths[i + 1:]) for i in range(len(f8s))]
    A = torch.cat(a_parts, dim=1).contiguous()
    B = torch.cat(b_parts[::-1], dim=1).contiguous()
    return A, B, [(a_off[i], b_off[i], f8s[i]) for i in range(len(f8s))]


# k-blocks per segment: K / 64 for fp16, K / 128 for e4m3; the producer / consumer ring has 3 stages.  gemm_tc issues the e4m3
# segments first, whatever order the caller lists them in.
@pytest.mark.parametrize("f8s,K", [
    ((0,), 64),            # 1 k-block
    ((1,), 128),           # 1
    ((0,), 128),           # 2 (below the ring depth)
    ((0,), 192),           # 3 (equal)
    ((0,), 256),           # 4 (one above)
    ((1, 1), 128),         # 1 + 1 = 2
    ((0, 1), 128),         # 2 + 1 = 3, e4m3 listed last
    ((0, 0, 1), 128),      # 2 + 2 + 1 = 5, e4m3 listed last
    ((1, 0, 1), 256),      # 2 + 4 + 2 = 8
    ((1, 1, 0), 640),      # 5 + 5 + 10 = 20
    ((0, 0, 0), 320),      # 15
    ((0, 1, 1), 5120),     # 80 + 40 + 40 = 160 (far above)
])
def test_gemm_tc_ring_phases(f8s, K):
    M, N = 300, 256
    A, B, segs = _random_segments(M, N, K, f8s, seed=K + 10 * sum(f8s))
    out = torch.full((M, N), float("nan"), device="cuda")
    assert _tc(A, B, M, N, K, segs, out32=out) == 0
    P, tol = _product(A, B, segs, K)
    ref, tol = _epilogue_ref(P, tol)
    _assert_within(out, ref, tol, f"segments {f8s} K={K}")


def _window_map(B, G, ws, ny, nx):
    """window_map_kernel / live_window_map_kernel (vit_pipeline.cu): row r of the window-partitioned operand -> token row of
    the frame batch, -1 for padding; ny x nx windows per frame, row-major"""
    L = ws * ws
    r = torch.arange(B * ny * nx * L)
    t, wb = r % L, r // L
    w, b = wb % (ny * nx), wb // (ny * nx)
    y, x = (w // nx) * ws + t // ws, (w % nx) * ws + t % ws
    return torch.where((y < G) & (x < G), b * G * G + y * G + x, torch.full_like(r, -1)).int()


# proj of a windowed block: x = x + proj(attn) with the window un-partition; all 25 windows, or the 15 live windows of a
# 480x854 frame (padding-window skip: token rows outside them must stay untouched)
@pytest.mark.parametrize("windows,kind", [((5, 5), "f8"), ((5, 5), "p2"), ((3, 5), "f8")])
def test_gemm_tc_rowmap_residual_in_place(windows, kind):
    Bf, G, ws, D = 2, 64, 14, 768
    rmap = _window_map(Bf, G, ws, *windows)
    M = rmap.numel()
    x, w, bias = _inputs(M, D, D, seed=M + len(kind))
    A, Bm, segs, s = _operands(x, w, kind)
    g = torch.Generator(device="cuda").manual_seed(9)
    old = torch.randn((Bf * G * G, D), generator=g, device="cuda") * 4.0
    out = old.clone()
    dev_map = rmap.cuda()
    assert _tc(A, Bm, M, D, D, segs, bias=bias, out32=out, resid=out, rowmap=dev_map, acc_scale=s) == 0
    P, tol = _product(A, Bm, segs, D)
    val, tol = _epilogue_ref(P, tol, s, bias)
    keep = dev_map >= 0
    dst = dev_map[keep].long()
    assert dst.unique().numel() == dst.numel()
    ref = old.double().clone()
    ref[dst] += val[keep]
    bound = torch.full_like(ref, 1.0)
    bound[dst] = tol[keep] + _UEPI * old.double()[dst].abs()
    touched = torch.zeros(Bf * G * G, dtype=torch.bool, device="cuda")
    touched[dst] = True
    assert torch.equal(out[~touched], old[~touched])       # rows no source row maps to: bit-identical
    _assert_within(out[touched], ref[touched], bound[touched], f"rowmap {windows} {kind}")


def test_gemm_tc_resid_mod_broadcast():
    """patch embedding: out = A.W^T + bias + pos_embed[row % (G*G)] over a batch of 3 frames"""
    Bf, GG, D, K = 3, 256, 256, 768
    M = Bf * GG
    x, w, bias = _inputs(M, D, K, seed=31)
    A, Bm, segs, _ = _operands(x, w, "p3")
    pos = torch.randn((GG, D), generator=torch.Generator(device="cuda").manual_seed(32), device="cuda")
    out = torch.full((M, D), float("nan"), device="cuda")
    assert _tc(A, Bm, M, D, K, segs, bias=bias, out32=out, resid=pos, resid_mod=GG) == 0
    P, tol = _product(A, Bm, segs, K)
    val, tol = _epilogue_ref(P, tol, None, bias)
    prow = pos.double().repeat(Bf, 1)
    _assert_within(out, val + prow, tol + _UEPI * prow.abs(), "resid_mod")


@pytest.mark.parametrize("out_kind", ["out32", "out16"])
def test_gemm_tc_skip_flag(out_kind):
    """the mask decoder's on-device break: skip != 0 writes nothing at all, skip == 0 computes"""
    M, N, K = 4096, 128, 256
    x, w, bias = _inputs(M, N, K, seed=41)
    A, Bm, segs, _ = _operands(x, w, "p3")
    resid = torch.randn((M, N), generator=torch.Generator(device="cuda").manual_seed(42), device="cuda")
    for flag in (1, 0):
        skip = torch.tensor([flag], dtype=torch.int32, device="cuda")
        if out_kind == "out32":
            out = torch.full((M, N), 1234.5, device="cuda")
            sentinel = out.clone()
            assert _tc(A, Bm, M, N, K, segs, bias=bias, out32=out, resid=resid, skip=skip) == 0
        else:
            out = torch.full((M, 2 * N), 77.0, device="cuda", dtype=torch.float16)
            sentinel = out.clone()
            assert _tc(A, Bm, M, N, K, segs, bias=bias, out16=out, ldc=2 * N, split_off=N, skip=skip) == 0
        if flag:
            assert torch.equal(out.view(torch.int16 if out_kind == "out16" else torch.int32),
                               sentinel.view(torch.int16 if out_kind == "out16" else torch.int32))
        else:
            P, tol = _product(A, Bm, segs, K)
            val, tol = _epilogue_ref(P, tol, None, bias)
            if out_kind == "out32":
                _assert_within(out, val + resid.double(), tol + _UEPI * resid.double().abs(), "skip=0 out32")
            else:
                _assert_within(out[:, :N].double() + out[:, N:].double(), val, tol + 2.0 ** -21 * val.abs() + 2.0 ** -24, "skip=0 hi+lo")


@pytest.mark.parametrize("kind", ["p3", "f8"])
def test_gemm_tc_acc_scale(kind):
    """acc_scale multiplies the accumulator before the bias is added (with fp16 segments too)"""
    M, N, K = 512, 256, 256
    x, w, bias = _inputs(M, N, K, seed=51)
    A, Bm, segs, s = _operands(x, w, kind)
    if s is None:
        s = torch.tensor([2.0 ** -5], device="cuda")
    out = torch.full((M, N), float("nan"), device="cuda")
    assert _tc(A, Bm, M, N, K, segs, bias=bias * 64.0, out32=out, acc_scale=s) == 0
    P, tol = _product(A, Bm, segs, K)
    val, tol = _epilogue_ref(P, tol, s, bias * 64.0)
    _assert_within(out, val, tol, f"acc_scale {kind}")


# GELU epilogues: lin1 of the ViT MLP (erf; out32 and the fp16 hi|lo operand of lin2) and CoTracker's fc1 (tanh, hi|lo)
@pytest.mark.parametrize("act,M,N,K,split", [(1, 512, 1024, 256, False), (1, 512, 1024, 256, True), (3, 512, 1536, 384, True),
                                             (3, 300, 160, 384, False)])
def test_gemm_tc_gelu(act, M, N, K, split):
    x, w, bias = _inputs(M, N, K, seed=60 + act, xscale=0.5)
    A, Bm, segs, _ = _operands(x, w, "p3")
    P, tol = _product(A, Bm, segs, K)
    val, tol = _epilogue_ref(P, tol, None, bias, act=act)
    if split:
        out = torch.full((M, 2 * N), float("nan"), device="cuda", dtype=torch.float16)
        assert _tc(A, Bm, M, N, K, segs, bias=bias, act=act, out16=out, ldc=2 * N, split_off=N) == 0
        hi, lo = out[:, :N].double(), out[:, N:].double()
        _assert_within(hi, val, tol + _fp16_tol(val), f"act {act} hi")
        _assert_within(hi + lo, val, tol + 2.0 ** -21 * val.abs() + 2.0 ** -24, f"act {act} hi+lo")
    else:
        out = torch.full((M, N), float("nan"), device="cuda")
        assert _tc(A, Bm, M, N, K, segs, bias=bias, act=act, out32=out) == 0
        _assert_within(out, val, tol, f"act {act} out32")


def test_gemm_tc_bf16_out16():
    M, N, K = 384, 512, 320
    g = torch.Generator(device="cuda").manual_seed(71)
    A = torch.randn((M, K), generator=g, device="cuda").bfloat16()
    Bm = (torch.randn((N, K), generator=g, device="cuda") / K ** 0.5).bfloat16()
    bias = torch.randn((N,), generator=g, device="cuda")
    out = torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16)
    assert _tc(A, Bm, M, N, K, [(0, 0, 0)], bias=bias, bf16=True, out16=out) == 0
    P, tol = _product(A, Bm, [(0, 0, 0)], K)
    val, tol = _epilogue_ref(P, tol, None, bias)
    _assert_within(out, val, tol + 2.0 ** -8 * val.abs(), "bf16 out16")


def _e4m3_ulp(t):
    """spacing of e4m3 values around |t| (subnormal spacing 2^-9 below 2^-6)"""
    e = torch.floor(torch.log2(t.abs().clamp(min=2.0 ** -6)))
    return torch.pow(2.0, e - 3)


def _check_f8_blocks(raw, hi, ref, tol, n0, split_off, what):
    """raw: uint8 rows; the e4m3 bytes of (v - hi) 2^12 at 2 split_off + n and of v 2^-3 at 3 split_off + n must be within
    one e4m3 code of the float64 value (plus what the bound on v allows)"""
    ncols = hi.shape[1]
    lo8 = raw[:, 2 * split_off + n0: 2 * split_off + n0 + ncols].contiguous().view(torch.float8_e4m3fn).double()
    hi8 = raw[:, 3 * split_off + n0: 3 * split_off + n0 + ncols].contiguous().view(torch.float8_e4m3fn).double()
    t_lo = ((ref - hi.double()) * 4096.0).clamp(-448, 448)
    t_hi = (ref * 0.125).clamp(-448, 448)
    _assert_within(lo8, t_lo, _e4m3_ulp(t_lo) + 4096.0 * tol, f"{what} e4m3 lo block")
    _assert_within(hi8, t_hi, _e4m3_ulp(t_hi) + 0.125 * tol, f"{what} e4m3 hi block")


@pytest.mark.parametrize("kind,act", [("f8", 1), ("f8", 0), ("p3", 0)])
def test_gemm_tc_out_f8(kind, act):
    """out_f8: the output row is the next fp8-corrected GEMM's A operand [fp16(v) | e4m3((v - hi) 2^12) | e4m3(v 2^-3)]"""
    M, N, K = 512, 768, 256
    x, w, bias = _inputs(M, N, K, seed=80 + act + len(kind))
    A, Bm, segs, s = _operands(x, w, kind)
    out = torch.full((M, 2 * N), float("nan"), device="cuda", dtype=torch.float16)
    assert _tc(A, Bm, M, N, K, segs, bias=bias, act=act, out16=out, ldc=2 * N, split_off=N, out_f8=1, acc_scale=s) == 0
    P, tol = _product(A, Bm, segs, K)
    val, tol = _epilogue_ref(P, tol, s, bias, act=act)
    hi = out[:, :N]
    _assert_within(hi, val, tol + _fp16_tol(val), f"out_f8 {kind} hi")
    _check_f8_blocks(out.view(torch.uint8), hi, val, tol, 0, N, f"out_f8 {kind}")


@pytest.mark.parametrize("act", [2, 4, -1])
def test_gemm_tc_rejects_unknown_act(act):
    """act 2 is ReLU in the CUDA-core GEMM's convention; gemm_tc has no ReLU and must refuse it, not run without activation"""
    from sampt_b200 import native
    ctx = native.get_context("cuda")
    A = torch.zeros((128, 64), device="cuda", dtype=torch.float16)
    out = torch.zeros((128, 128), device="cuda")
    n0 = native.lib().sampt_launch_count(ctx.handle)
    assert _tc(A, torch.zeros((128, 64), device="cuda", dtype=torch.float16), 128, 128, 64, [(0, 0, 0)], act=act, out32=out) != 0
    assert native.lib().sampt_launch_count(ctx.handle) == n0
