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
