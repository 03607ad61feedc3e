"""GPU: the PIPS tracker (csrc/pips_kernels.cu, csrc/pips_pipeline.cu) kernel by kernel against float64, through the unit-test
entries of include/sampt_b200.h (sampt_test_pips_conv / _inorm / _resize / _corr / _window_op) and sampt_linear_f32.

Bounds are derived from fp32 rounding, u = 2^-24, and the summation length n of the kernel under test (gamma_n = n u / (1 - n u));
the float64 reference is computed from exactly the fp32 operands the kernel reads.  Each group prints its worst error / bound.
Outputs start as NaN with a guard row: rows the kernel must not write stay NaN.  Inputs carry a guard row of 1e30, so an over-read
turns an output into garbage."""
import math
from ctypes import c_char_p, c_float, c_int

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import pips_ref
from sampt_b200 import native, synth

pytestmark = pytest.mark.gpu

_U = 2.0 ** -24
_S = 8
_C2 = (120, 213)           # level-0 feature map of the 480x854 C2 frames; pooled levels 60x106, 30x53, 15x26


def _gamma(n):
    return n * _U / (1 - n * _U)


def _report(what, err, bound):
    worst = (err / bound).max().item()
    print(f"{what}: max err {err.max().item():.3g}, worst err / bound {worst:.3g}")
    assert worst <= 1.0, (what, worst)


@pytest.fixture(scope="module")
def model():
    from sam_pt.point_tracker.pips import Pips
    sd = synth.condition_pips(synth.make_state_dict(pips_ref.pips_state_dict_shapes(), 7201))
    m = Pips(S=8, stride=4)
    m.load_state_dict(sd, strict=True)      # tensor-core path: registers both the fp32 "_rsck" and the fp16 hi|lo ".w16" weights
    m = m.cuda().eval()
    return m, {k: v.cuda().double() for k, v in sd.items()}


def _ctx(m):
    return m.native_context()


def _guarded(t, fill=1e30):
    """flat device buffer holding t, followed by one guard row of `fill`; returns (buffer, view of t)"""
    row = t.shape[-1] if t.dim() else 1
    buf = torch.cat([t.reshape(-1).float().cuda(), torch.full((row,), fill, device="cuda")])
    return buf, buf[: t.numel()].view(t.shape)


def _nan_out(shape, guard_row):
    buf = torch.full((math.prod(shape) + guard_row,), float("nan"), device="cuda")
    return buf, buf[: math.prod(shape)].view(shape)


def _guard_ok(buf, n):
    torch.cuda.synchronize()
    assert torch.isnan(buf[n:]).all(), "a value past the output was written"


# ======================================================================================================= encoder convolutions
# (name, Cin, Cout, R, stride, pad, H, W): every layer shape of the BasicEncoder, at the C2 geometry, CoTracker's 384x512 and an
# odd 61x107 frame
_CONVS = [
    ("fnet.layer1.0.conv1", 64, 64, 3, 1, 1, 240, 427),
    ("fnet.layer2.0.conv1", 64, 96, 3, 2, 1, 240, 427),
    ("fnet.layer2.0.downsample.0", 64, 96, 1, 2, 0, 240, 427),
    ("fnet.layer2.1.conv1", 96, 96, 3, 1, 1, 120, 214),
    ("fnet.layer3.0.conv1", 96, 128, 3, 2, 1, 120, 214),
    ("fnet.layer3.0.downsample.0", 96, 128, 1, 2, 0, 120, 214),
    ("fnet.layer4.0.conv1", 128, 128, 3, 2, 1, 60, 107),
    ("fnet.layer4.1.conv2", 128, 128, 3, 1, 1, 30, 54),
    ("fnet.conv2", 416, 256, 3, 1, 1, 120, 213),
    ("fnet.conv3", 256, 128, 1, 1, 0, 120, 213),
    ("fnet.layer2.0.conv1", 64, 96, 3, 2, 1, 96, 128),      # CoTracker 384x512
    ("fnet.layer3.0.conv1", 96, 128, 3, 2, 1, 16, 27),      # odd 61x107 frame
    ("fnet.conv2", 416, 256, 3, 1, 1, 15, 26),
]


def _conv_bound(tc, K, A, Wabs, Xabs, v, bias):
    """fp32 path: one fma chain of K terms then + bias.  Tensor-core path: 3-pass fp16 hi|lo (tests/test_gpu_gemm.py: 2^-21
    sqrt(k16 steps) per product sum), the dropped lo.lo and the two split roundings (2^-20 of the products), fp16 subnormals of
    the lo halves (2^-25 absolute per operand), the fp32 epilogue"""
    if not tc:
        return _gamma(K + 1) * (A + bias.abs()) + 1e-30
    Kp = -(-K // 64) * 64
    return ((2.0 ** -21 * (3 * Kp / 16) ** 0.5 + 2.0 ** -20) * A + 2.0 ** -25 * (Wabs + Xabs)
            + 2.0 ** -20 * (v.abs() + bias.abs()) + 1e-30)


def _run_conv(m, name, tc, x_buf, is_f32, n, H, W, Cin, Cout, R, stride, pad):
    Ho, Wo = (H + 2 * pad - R) // stride + 1, (W + 2 * pad - R) // stride + 1
    obuf, out = _nan_out((n, Ho, Wo, Cout), Cout)
    native.check(native.lib().sampt_test_pips_conv(
        _ctx(m).handle, c_char_p(name.encode()), c_int(tc), native.ptr(x_buf), c_int(is_f32), c_int(n), c_int(H), c_int(W), c_int(Cin),
        c_int(Cout), c_int(R), c_int(stride), c_int(pad), native.ptr(obuf), native.stream_ptr()), "test_pips_conv")
    _guard_ok(obuf, out.numel())
    return out


def _conv_expected(sd64, name, x64, stride, pad, tc):
    w, b = sd64[name + ".weight"], sd64[name + ".bias"]
    v = F.conv2d(x64, w, b, stride=stride, padding=pad)
    A = F.conv2d(x64.abs(), w.abs(), None, stride=stride, padding=pad)
    R = w.shape[-1]
    Wabs = F.conv2d(torch.ones_like(x64[:, :1]), w.abs().sum(1, keepdim=True), None, stride=stride, padding=pad) if tc else 0
    Xabs = F.conv2d(x64.abs().sum(1, keepdim=True), torch.ones((1, 1, R, R), dtype=x64.dtype, device=x64.device), None,
                    stride=stride, padding=pad) if tc else 0
    K = w.shape[1] * w.shape[2] * w.shape[3]
    return v, _conv_bound(tc, K, A, Wabs, Xabs, v, b.view(1, -1, 1, 1))


@pytest.mark.parametrize("tc", [0, 1])
@pytest.mark.parametrize("case", range(len(_CONVS)))
def test_encoder_conv(model, case, tc):
    """one encoder convolution by weight name on both paths; a random input, then a saturated border around a zero interior"""
    m, sd64 = model
    name, Cin, Cout, R, stride, pad, H, W = _CONVS[case]
    g = torch.Generator().manual_seed(case)
    for kind in ("random", "border"):
        if kind == "random":
            x = torch.randn((1, H, W, Cin), generator=g) * torch.rand((1, 1, 1, Cin), generator=g) * 3
        else:
            x = torch.zeros((1, H, W, Cin))
            x[:, :2], x[:, -2:], x[:, :, :2], x[:, :, -2:] = 4.0, -4.0, 4.0, -4.0
        xb, xg = _guarded(x)
        out = _run_conv(m, name, tc, xb, 1, 1, H, W, Cin, Cout, R, stride, pad)
        v, tol = _conv_expected(sd64, name, xg.double().permute(0, 3, 1, 2), stride, pad, tc)
        _report(f"conv {name} {H}x{W} tc={tc} {kind}", (out.double().permute(0, 3, 1, 2) - v).abs(), tol)


@pytest.mark.parametrize("tc", [0, 1])
@pytest.mark.parametrize("H,W", [(480, 854), (384, 512), (61, 107)])
def test_encoder_conv1(model, H, W, tc):
    """conv1 on uint8 frames and on float frames holding 0..255, random and with a saturated border around a black interior.
    The operand is the kernel's own fp32 2*(x/255)-1 (torch's fp32 tensor division and subtraction round the same way)."""
    m, sd64 = model
    g = torch.Generator().manual_seed(H)
    rnd = torch.randint(0, 256, (1, 3, H, W), generator=g, dtype=torch.uint8)
    border = torch.zeros((1, 3, H, W), dtype=torch.uint8)
    border[..., :3, :], border[..., -3:, :], border[..., :, :3], border[..., :, -3:] = 255, 255, 255, 255
    for kind, fr in (("random", rnd), ("border", border)):
        for is_f32 in (0, 1):
            if is_f32:
                buf, frames = _guarded(fr.float())
            else:
                frames = fr.cuda().contiguous()
                buf = torch.cat([frames.reshape(-1), torch.full((W,), 255, dtype=torch.uint8, device="cuda")])
            out = _run_conv(m, "fnet.conv1", tc, buf, is_f32, 1, H, W, 3, 64, 7, 2, 3)
            x = 2.0 * (frames.float() / torch.full_like(frames, 255.0, dtype=torch.float32)) - 1.0
            v, tol = _conv_expected(sd64, "fnet.conv1", x.double(), 2, 3, tc)
            _report(f"conv1 {H}x{W} tc={tc} f32={is_f32} {kind}", (out.double().permute(0, 3, 1, 2) - v).abs(), tol)


# ======================================================================================================= instance norm
def _inorm_input(n, HW, C, seed):
    """channels with |mean| / std from 0 to 1e4, exactly constant channels and variances below eps"""
    g = torch.Generator().manual_seed(seed)
    ratio = torch.cat([torch.zeros(1), torch.logspace(-1, 4, C - 1)])
    std = torch.exp(torch.randn((C,), generator=g)).clamp(0.05, 5)
    mean = ratio * std * torch.where(torch.rand((C,), generator=g) < 0.5, -1.0, 1.0)
    x = mean + std * torch.randn((n, HW, C), generator=g)
    x[:, :, C - 4] = 0.7                                           # exactly constant
    x[:, :, C - 3] = -2.5
    x[:, :, C - 2] = 1e-4 * torch.randn((n, HW), generator=g)     # variance below eps
    x[:, :, C - 1] = 1.0 + 1e-4 * torch.randn((n, HW), generator=g)
    return x


def _inorm_ref(x64):
    """float64 mean, biased variance and rstd per (image, channel) of exactly the fp32 values the kernel reads"""
    m = x64.mean(dim=1, keepdim=True)
    var = ((x64 - m) ** 2).mean(dim=1, keepdim=True)
    return m, var, 1.0 / torch.sqrt(var + 1e-5)


def _inorm_stats_bound(x64, m, var, rstd):
    """What a correctly rounded two-pass fp32 instance norm reaches, plus the summation of the kernel.  Both passes sum fp32
    partials of <= 64 pixels promoted to fp64 (gamma_64).  Pass 1 sums d = x - xc (xc the centre pixel): the mean of d^2 is
    var + (m - xc)^2, and its statistics are kept where (m - xc)^2 <= 8 (var + eps) (covered up to 9).  Elsewhere pass 2 sums
    d = x - m1, m1 the fp32 mean of pass 1, off by dm1 <= u |m| + 2 gamma_64 sqrt(var + (m - xc)^2).  The mean is stored in fp32
    (u |m|), rstd goes through a float division and sqrt (2 u).  No term grows with (mean / std)^2."""
    dc = m - x64[:, x64.shape[1] // 2:x64.shape[1] // 2 + 1]
    dm1 = _U * m.abs() + 2 * _gamma(64) * (var + dc ** 2).sqrt()
    shift = torch.maximum(torch.minimum(dc.abs(), (9 * (var + 1e-5)).sqrt()), dm1)
    msq = var + shift ** 2                                # mean of d^2 on the branch taken
    var_err = 3 * _gamma(64) * (msq + shift * msq.sqrt())
    rel_rstd = 0.5 * var_err / (var + 1e-5) + 2 * _U
    return _U * m.abs() + 2 * _gamma(64) * msq.sqrt() + 1e-45, rel_rstd


def _norm_bound(x64, m, rstd, m_err, rel_rstd):
    """(x - mean) * rstd in fp32 from the stored stats"""
    d = x64 - m
    return rstd * (m_err + _U * d.abs()) * (1 + rel_rstd) + d.abs() * rstd * rel_rstd + 2 * _U * d.abs() * rstd


def _run_inorm(m, x, res, mode, n, HW, C):
    xb, xg = _guarded(x)
    rb, rg = _guarded(res) if res is not None else (None, None)
    ybuf, y = _nan_out((n, HW, C), C)
    sbuf, stats = _nan_out((n, C, 2), 2)
    rsbuf, rstats = _nan_out((n, C, 2), 2)
    native.check(native.lib().sampt_test_pips_inorm(
        _ctx(m).handle, native.ptr(xb), native.ptr(rb), c_int(mode), c_int(n), c_int(HW), c_int(C), native.ptr(ybuf), native.ptr(sbuf),
        native.ptr(rsbuf), native.stream_ptr()), "test_pips_inorm")
    for b, t in ((ybuf, y), (sbuf, stats), (rsbuf, rstats)):
        _guard_ok(b, t.numel())
    return xg, rg, y, stats, rstats


@pytest.mark.parametrize("C", [64, 96, 128, 256])
@pytest.mark.parametrize("HW", [1, 511, 512, 513, 240 * 427])
def test_instance_norm(model, C, HW):
    m = model[0]
    n = 2
    x = _inorm_input(n, HW, C, seed=C + HW)
    res = torch.randn((n, HW, C), generator=torch.Generator().manual_seed(1)) * 2 + 0.5
    res_in = _inorm_input(n, HW, C, seed=C + HW + 1)
    for mode, r in ((0, None), (1, res), (2, res_in)):
        xg, rg, y, stats, rstats = _run_inorm(m, x, r, mode, n, HW, C)
        x64 = xg.double()
        mu, var, rstd = _inorm_ref(x64)
        m_err, rel_rstd = _inorm_stats_bound(x64, mu, var, rstd)
        _report(f"inorm mean C={C} HW={HW} mode {mode}", (stats[..., 0].double() - mu[:, 0]).abs(), m_err[:, 0])
        _report(f"inorm rstd C={C} HW={HW} mode {mode}", (stats[..., 1].double() - rstd[:, 0]).abs(), rel_rstd[:, 0] * rstd[:, 0])
        yn = (x64 - mu) * rstd
        tol = _norm_bound(x64, mu, rstd, m_err, rel_rstd)
        ref = torch.relu(yn)
        if mode == 1:
            ref = torch.relu(ref + rg.double())
            tol = tol + _U * (ref.abs() + rg.double().abs())
        elif mode == 2:
            r64 = rg.double()
            rm, rv, rr = _inorm_ref(r64)
            rme, rre = _inorm_stats_bound(r64, rm, rv, rr)
            _report(f"inorm res rstd C={C} HW={HW}", (rstats[..., 1].double() - rr[:, 0]).abs(), rre[:, 0] * rr[:, 0])
            rn = (r64 - rm) * rr
            ref = torch.relu(ref + rn)
            tol = tol + _norm_bound(r64, rm, rr, rme, rre) + _U * (ref.abs() + rn.abs())
        _report(f"inorm y C={C} HW={HW} mode {mode}", (y.double() - ref).abs(), tol + 1e-45)


# ======================================================================================================= pyramid and resize
@pytest.mark.parametrize("H,W", [(120, 213), (61, 107), (17, 23), (9, 11)])
def test_avgpool_pyramid(model, H, W):
    """avg_pool2d(2, 2) (floor) on odd sizes: (a + b + c + d) * 0.25 in fp32 is the same add order as F.avg_pool2d's CPU kernel,
    so float32 results must be bit-exact"""
    m = model[0]
    g = torch.Generator().manual_seed(H * W)
    T = 2
    fm = torch.randn((T, H, W, 128), generator=g).cuda()
    lv = [torch.full((T * (H >> l) * (W >> l) * 128 + 128,), float("nan"), device="cuda") for l in (1, 2, 3)]
    native.check(native.lib().sampt_pips_pyramid(_ctx(m).handle, native.ptr(fm), c_int(T), c_int(H), c_int(W), native.ptr(lv[0]),
                                                 native.ptr(lv[1]), native.ptr(lv[2]), native.stream_ptr()), "pips_pyramid")
    ref = pips_ref.build_pyramid(fm.permute(0, 3, 1, 2).cpu()[None])
    for l in (1, 2, 3):
        h, w = H >> l, W >> l
        _guard_ok(lv[l - 1], T * h * w * 128)
        got = lv[l - 1][: T * h * w * 128].view(T, h, w, 128).permute(0, 3, 1, 2).cpu()
        assert torch.equal(got, ref[l][0]), (H, W, l)
    print(f"avgpool {H}x{W}: bit-exact")


@pytest.mark.parametrize("Hi,Wi,C,Ho,Wo,coff", [(240, 427, 64, 120, 213, 0), (120, 214, 96, 120, 213, 64), (60, 107, 128, 120, 213, 160),
                                                (30, 54, 128, 120, 213, 288), (5, 7, 64, 1, 1, 0), (13, 17, 128, 40, 60, 160)])
def test_resize_concat(model, Hi, Wi, C, Ho, Wo, coff):
    """bilinear, align_corners=True, into a channel slice of the 416-channel concat buffer: the other channels stay NaN.  The
    source position is the kernel's own fp32 scale * dst (torch float32 rounds the same way); the blend of 4 corners in fp32
    costs <= 4 u sum |w v| and each weight product 2 u."""
    m = model[0]
    g = torch.Generator().manual_seed(Hi + C)
    x = torch.randn((1, Hi, Wi, C), generator=g)
    xb, xg = _guarded(x)
    Ctot = 416
    obuf, out = _nan_out((1, Ho, Wo, Ctot), Ctot)
    native.check(native.lib().sampt_test_pips_resize(_ctx(m).handle, native.ptr(xb), c_int(1), c_int(Hi), c_int(Wi), c_int(C),
                                                     native.ptr(obuf), c_int(Ho), c_int(Wo), c_int(Ctot), c_int(coff),
                                                     native.stream_ptr()), "test_pips_resize")
    _guard_ok(obuf, out.numel())
    other = torch.ones(Ctot, dtype=torch.bool)
    other[coff: coff + C] = False
    assert torch.isnan(out[..., other]).all(), "channels outside the slice were written"

    def src(n_in, n_out):
        sc = torch.tensor(float(n_in - 1)) / torch.tensor(float(n_out - 1)) if n_out > 1 else torch.tensor(0.0)
        f = sc * torch.arange(n_out, dtype=torch.float32)
        i0 = f.long()
        i1 = torch.where(i0 < n_in - 1, i0 + 1, i0)
        return i0, i1, (f - i0.float()).double()
    y0, y1, ly = src(Hi, Ho)
    x0, x1, lx = src(Wi, Wo)
    v = xg[0].double().cpu()
    ly, lx = ly[:, None, None], lx[None, :, None]
    hy, hx = 1 - ly, 1 - lx
    c00, c01, c10, c11 = v[y0][:, x0], v[y0][:, x1], v[y1][:, x0], v[y1][:, x1]
    ref = hy * (hx * c00 + lx * c01) + ly * (hx * c10 + lx * c11)
    mag = hy * (hx * c00.abs() + lx * c01.abs()) + ly * (hx * c10.abs() + lx * c11.abs())
    _report(f"resize {Hi}x{Wi}->{Ho}x{Wo} C={C}", (out[0, ..., coff: coff + C].double().cpu() - ref).abs(), 6 * _U * mag + 1e-45)


# ======================================================================================================= correlation rows
def _c2_pyramid(T, seed):
    g = torch.Generator().manual_seed(seed)
    fm = (torch.randn((T, 128, *_C2), generator=g) * 0.5).cuda()
    return [p[0] for p in pips_ref.build_pyramid(fm[None])]          # (T, 128, H_l, W_l) fp32


def _corr_points(N, H4, W4, g):
    """(N, S, 2) level-0 coordinates: interior points, integral and half-integral at every level (multiples of 8 and 4),
    points on every border of every level and one pixel outside, far outside"""
    c = torch.rand((N, _S, 2), generator=g) * torch.tensor([W4 - 1.0, H4 - 1.0])
    special = []
    for l in range(4):
        s = 2.0 ** l
        Wl, Hl = W4 // 2 ** l, H4 // 2 ** l
        for fx, fy in ((0, 0), (Wl - 1, 0), (0, Hl - 1), (Wl - 1, Hl - 1), (-1, 3), (Wl, 3), (3, -1), (3, Hl), (5, 7), (5.5, 7.5)):
            special.append((fx * s, fy * s))
    special += [(-1e4, 20.0), (1e4, 20.0), (30.0, -1e4), (30.0, 1e4), (0.5, 0.5), (W4 - 1.5, H4 - 1.5)]
    sp = torch.tensor(special)
    k = 0
    for n in range(N):
        for s in range(_S):
            if (n * _S + s) % 3 == 0 or N == 1:
                c[n, s] = sp[k % len(sp)]
                k += 1
    return c


def _roundtrip_taps(cx, cy, level, H, W):
    """the kernel's fp32 sample positions of the 7x7 window (grid_sample align_corners round trip), in the reference's
    transposed order: out[a*7 + b] samples x = cx + a - 3, y = cy + b - 3"""
    sc = 1.0 / 2 ** level
    cxl, cyl = cx * sc, cy * sc
    a = torch.arange(7, device=cx.device, dtype=torch.float32) - 3
    sx = (cxl[:, None, None] + a[:, None]).expand(-1, 7, 7)
    sy = (cyl[:, None, None] + a[None, :]).expand(-1, 7, 7)
    # divisions by a tensor: torch turns a division by a Python scalar into a multiplication by its reciprocal
    gx = 2.0 * sx / torch.full_like(sx, W - 1) - 1.0
    gy = 2.0 * sy / torch.full_like(sy, H - 1) - 1.0
    ux = ((gx + 1.0) * 0.5) * float(W - 1)
    uy = ((gy + 1.0) * 0.5) * float(H - 1)
    return ux.reshape(-1, 49), uy.reshape(-1, 49), sx.reshape(-1, 49)


def _corr_expected(lv, ff, co, slots):
    """float64 correlation rows from the kernel's fp32 sample positions, and the bound.  Dot products: per lane 4 fp32 terms,
    a 5-level warp tree (n = 9), times fl(1/sqrt(128)) (2 u).  Blend: weight products and the 4-term sum (6 u of sum |w D|).
    A corner the 8x8 patch does not hold (index -1 or 8 after the round trip) is read as 0: its weight must be below
    8 u (|x| + W) (asserted) and its term is added to the bound."""
    NS = co.shape[0] * co.shape[1]
    f64 = ff.reshape(NS, 128).double()
    out = torch.zeros((NS, 196), dtype=torch.float64, device="cuda")
    tol = torch.zeros_like(out)
    fr = torch.tensor(slots, device="cuda").repeat(co.shape[0])       # frame of each (n, s) row
    cx, cy = co.reshape(NS, 2)[:, 0], co.reshape(NS, 2)[:, 1]
    for l, fm in enumerate(lv):
        T, H, W, _ = fm.shape
        ux, uy, sx = _roundtrip_taps(cx, cy, l, H, W)
        x0, y0 = torch.floor(ux), torch.floor(uy)
        fx, fy = (ux - x0).double(), (uy - y0).double()
        bx = torch.floor(cx / 2 ** l) - 3
        by = torch.floor(cy / 2 ** l) - 3
        fmd = fm.double()
        val = torch.zeros((NS, 49), dtype=torch.float64, device="cuda")
        mag = torch.zeros_like(val)
        dropped = torch.zeros_like(val)
        for dy, dx, w in ((0, 0, (1 - fx) * (1 - fy)), (0, 1, fx * (1 - fy)), (1, 0, (1 - fx) * fy), (1, 1, fx * fy)):
            px, py = (x0 + dx).long(), (y0 + dy).long()
            inside = (px >= 0) & (px < W) & (py >= 0) & (py < H)
            ix, iy = px - bx.long()[:, None], py - by.long()[:, None]
            in_patch = (ix >= 0) & (ix < 8) & (iy >= 0) & (iy < 8)
            vec = fmd[fr[:, None].expand(-1, 49), py.clamp(0, H - 1), px.clamp(0, W - 1)]          # (NS, 49, 128)
            d = (vec * f64[:, None]).sum(-1) / math.sqrt(128)
            a = (vec.abs() * f64.abs()[:, None]).sum(-1) / math.sqrt(128)
            d = torch.where(inside, d, torch.zeros_like(d))
            a = torch.where(inside, a, torch.zeros_like(a))
            miss = inside & ~in_patch
            if miss.any():
                lim = 8 * _U * (sx.abs().double() + W)
                assert (w[miss] <= lim[miss]).all(), f"level {l}: a corner outside the 8x8 patch carries weight {w[miss].max().item():.3g}"
            val += torch.where(in_patch, w * d, torch.zeros_like(d))
            dropped += torch.where(miss, w * d.abs(), torch.zeros_like(d))
            mag += w * a
        out[:, l * 49:(l + 1) * 49] = val
        tol[:, l * 49:(l + 1) * 49] = (_gamma(9) + 2 * _U) * mag + 6 * _U * mag + dropped + 1e-45
    return out, tol


@pytest.mark.parametrize("N", [1, 8, 292])
def test_corr_rows_c2(model, N):
    m = model[0]
    H4, W4 = _C2
    T = 10
    lv_nchw = _c2_pyramid(T, seed=N)
    lv = [p.permute(0, 2, 3, 1).contiguous() for p in lv_nchw]
    bufs = [torch.cat([p.reshape(-1), torch.full((128,), 1e30, device="cuda")]) for p in lv]
    g = torch.Generator().manual_seed(N + 1)
    co = _corr_points(N, H4, W4, g).cuda()
    ff = (torch.randn((N, _S, 128), generator=g) * 0.5).cuda()
    ffb, ffg = _guarded(ff)
    cob, cog = _guarded(co)
    active = np.ones(N, dtype=np.uint8)
    if N > 1:
        active[1::3] = 0
    slots = [2, 3, 4, 5, 6, 7, 9, 9]                                   # tail padding repeats the last frame
    f, n_missing = 2, 1
    obuf, xin = _nan_out((N * _S, 520), 520)
    native.check(native.lib().sampt_test_pips_corr(
        _ctx(m).handle, native.ptr(bufs[0]), native.ptr(bufs[1]), native.ptr(bufs[2]), native.ptr(bufs[3]), c_int(H4), c_int(W4),
        native.ptr(ffb), native.ptr(cob), c_int(N), c_int(_S), np.ctypeslib.as_ctypes(active), c_int(f), c_int(n_missing), (c_int * 8)(*slots), native.ptr(obuf), native.stream_ptr()),
        "test_pips_corr")
    _guard_ok(obuf, xin.numel())
    rows = xin.view(N, _S, 520)
    act = torch.from_numpy(active).bool().cuda()
    assert torch.isnan(rows[~act]).all(), "rows of inactive points were written"
    r = rows[act].reshape(-1, 520)
    ffa, coa = ffg[act], cog[act]
    # ffeat copy, flow columns and pad: exact
    assert torch.equal(r[:, :128], ffa.reshape(-1, 128))
    flow = coa - coa[:, :1]
    t = torch.linspace(0, _S, _S, dtype=torch.float32).cuda()         # times_ of pips.py:527, as the reference builds it
    assert torch.equal(r[:, 516:518], flow.reshape(-1, 2)), "flow columns"
    assert torch.equal(r[:, 518].view(-1, _S), t[None].expand(coa.shape[0], -1)), "time column"
    assert (r[:, 519] == 0).all()
    # correlation
    exp, tol = _corr_expected(lv, ffa, coa, slots)
    _report(f"corr rows N={N}", (r[:, 128:324].double() - exp).abs(), tol)
    # sin/cos embedding: fp32 argument arg = flow * div (u |arg|), sinf/cosf within 2 ulps (|.| <= 1: 2^-23)
    xyz = r[:, 516:519].double()
    div = torch.arange(0, 64, 2, device="cuda", dtype=torch.float64) * (1000.0 / 64)
    arg = xyz[:, :, None] * div
    emb = torch.stack([torch.sin(arg), torch.cos(arg)], dim=-1).reshape(-1, 192)
    tol = (_U * arg.abs()).repeat_interleave(2, dim=-1).reshape(-1, 192) + 2.0 ** -22
    _report(f"sincos N={N} (|arg| up to {arg.abs().max().item():.3g})", (r[:, 324:516].double() - emb).abs(), tol)


# ======================================================================================================= window ops
def _window_op(m, op, N, T, f, n_missing, active=None, slots=None, fmaps=None, H4=0, W4=0, coords=None, ffeats=None, feat_init=None,
               traj=None, vis=None, cur=None, x=None, xln=None, layer=0, delta=None, thr0=0.9, stride=4):
    act = np.ascontiguousarray(active if active is not None else np.ones(N, dtype=np.uint8))
    sl = (c_int * 8)(*(slots if slots is not None else range(8)))
    native.check(native.lib().sampt_test_pips_window_op(
        _ctx(m).handle, c_int(op), c_int(N), c_int(_S), c_int(T), c_int(stride), c_int(f), c_int(n_missing), sl,
        np.ctypeslib.as_ctypes(act), native.ptr(fmaps), c_int(H4), c_int(W4), native.ptr(coords), native.ptr(ffeats),
        native.ptr(feat_init), native.ptr(traj), native.ptr(vis), native.ptr(cur), native.ptr(x), native.ptr(xln), c_int(layer),
        native.ptr(delta), c_float(thr0), native.stream_ptr()), f"test_pips_window_op {op}")
    torch.cuda.synchronize()


def test_window_init(model):
    """coords = traj[f] / stride exactly for every slot; feat_init = bilinear_sample2d of slot 0's frame (clamped indices,
    unclamped weights) for points left of, right of, on and beyond the map edge: 3 u per weight product, 4-term sum 3 u"""
    m = model[0]
    H4, W4 = _C2
    T, N, f = 12, 12, 4
    g = torch.Generator().manual_seed(11)
    fm = (torch.randn((T, H4, W4, 128), generator=g) * 0.5).cuda()
    fmb = torch.cat([fm.reshape(-1), torch.full((128,), 1e30, device="cuda")])
    xy = torch.tensor([[-0.75, 3.0], [0.0, 0.0], [-1.0, 5.5], [W4 - 1.0, 7.25], [W4 - 0.5, 8.0], [W4 + 2.25, 60.0],
                       [10.5, -0.5], [20.0, H4 - 1.0], [30.25, H4 - 0.25], [40.0, H4 + 3.5], [1e4, -1e4], [57.3, 44.9]]) * 4.0
    traj = torch.full((T, N, 2), float("nan"), device="cuda")
    traj[f] = xy.cuda()
    active = np.ones(N, dtype=np.uint8)
    active[5] = 0
    slots = [7, 8, 9, 10, 11, 11, 11, 11]
    coords = torch.full((N, _S, 2), float("nan"), device="cuda")
    ffeats = torch.full((N, _S, 128), float("nan"), device="cuda")
    feat_init = torch.full((N, 128), float("nan"), device="cuda")
    _window_op(m, 1, N, T, f, 0, active=active, slots=slots, fmaps=fmb, H4=H4, W4=W4, coords=coords, ffeats=ffeats,
               feat_init=feat_init, traj=traj)
    a = torch.from_numpy(active).bool().cuda()
    assert torch.isnan(coords[~a]).all() and torch.isnan(ffeats[~a]).all() and torch.isnan(feat_init[~a]).all()
    assert torch.equal(coords[a], (traj[f][a] / 4.0)[:, None].expand(-1, _S, -1))
    c = traj[f] / 4.0
    ref = pips_ref.bilinear_sample2d(fm[slots[0]].permute(2, 0, 1)[None].double(), c[None, :, 0].double(), c[None, :, 1].double())[0].T
    mag = pips_ref.bilinear_sample2d(fm[slots[0]].permute(2, 0, 1)[None].double().abs(), c[None, :, 0].double(),
                                     c[None, :, 1].double())[0].T.abs()
    _report("window init feat", (feat_init[a].double() - ref[a]).abs(), 6 * _U * mag[a] + 1e-45)
    assert torch.equal(ffeats[a], feat_init[a][:, None].expand(-1, _S, -1))
    # sample_feat = 0: the stored feat_init is broadcast
    ffeats.fill_(float("nan"))
    _window_op(m, 0, N, T, f, 0, active=active, slots=slots, coords=coords, ffeats=ffeats, feat_init=feat_init, traj=traj)
    assert torch.equal(ffeats[a], feat_init[a][:, None].expand(-1, _S, -1)) and torch.isnan(ffeats[~a]).all()


@pytest.mark.parametrize("N", [1, 8, 292])
def test_update(model, N):
    """GroupNorm(1,128) (block sums of 128: n = 7) + Linear 128x128 (fma chain, n = 129) + GELU (erff: slope <= 1.13, 2 u),
    added to ffeats; coords += dxy except slot 0, which stays bitwise; inactive points untouched"""
    m, sd64 = model
    g = torch.Generator().manual_seed(N)
    delta = torch.randn((N, _S * 130), generator=g).cuda()
    delta.view(N, _S, 130)[:, :, 2:] += torch.randn((N, _S, 1), generator=g).cuda() * 30     # large common offsets
    ffeats = torch.randn((N, _S, 128), generator=g).cuda()
    coords = (torch.rand((N, _S, 2), generator=g) * 200).cuda()
    active = np.ones(N, dtype=np.uint8)
    if N > 1:
        active[::4] = 0
    f0, c0 = ffeats.clone(), coords.clone()
    _window_op(m, 5, N, 10, 0, 0, active=active, coords=coords, ffeats=ffeats, delta=delta)
    a = torch.from_numpy(active).bool().cuda()
    assert torch.equal(ffeats[~a], f0[~a]) and torch.equal(coords[~a], c0[~a])
    assert torch.equal(coords[:, 0], c0[:, 0]), "slot 0 coordinates moved"
    d = delta.view(N, _S, 130).double()
    assert torch.equal(coords[a][:, 1:], (c0[a][:, 1:] + delta.view(N, _S, 130)[a][:, 1:, :2]))
    v = d[..., 2:]
    mu = v.mean(-1, keepdim=True)
    dv = v - mu
    var = (dv ** 2).mean(-1, keepdim=True)
    rstd = 1 / torch.sqrt(var + 1e-5)
    gw, gb = sd64["norm.weight"], sd64["norm.bias"]
    gn = dv * rstd * gw + gb
    m_err = _gamma(8) * v.abs().mean(-1, keepdim=True) + _U * mu.abs()
    rel = 0.5 * (_gamma(9) * var + 2 * m_err * dv.abs().mean(-1, keepdim=True)) / (var + 1e-5) + 3 * _U
    e_gn = (rstd * (m_err + _U * dv.abs()) + dv.abs() * rstd * rel) * gw.abs() + 3 * _U * (dv.abs() * rstd * gw.abs() + gb.abs())
    W, b = sd64["ffeat_updater.0.weight"], sd64["ffeat_updater.0.bias"]
    acc = gn @ W.T + b
    e_acc = _gamma(129) * (gn.abs() @ W.abs().T + b.abs()) + e_gn @ W.abs().T
    up = F.gelu(acc)
    ref = f0.double() + up
    tol = 1.13 * e_acc + 2 * _U * up.abs() + _U * ref.abs() + 1e-45
    _report(f"update ffeats N={N}", (ffeats.double() - ref).abs()[a], tol[a])


@pytest.mark.parametrize("N", [1, 2, 4, 8, 33, 64, 292])
def test_mixer_sgemm(model, N):
    """the five sgemm_nt calls of one iteration at M = 8 N rows (every dispatch branch), incl. 2048->512 with the residual
    aliased to the output, as pips_iteration runs it: any summation order of K terms is within gamma_K sum |x w|"""
    m, sd64 = model
    ctx = _ctx(m)
    M = N * _S
    g = torch.Generator().manual_seed(M)
    p = "delta_block.to_delta."
    w0 = torch.zeros((512, 520), device="cuda")
    w0[:, :519] = sd64[p + "0.weight"].float()
    for what, K, Nout, W, b, act, alias in (("520->512", 520, 512, w0, sd64[p + "0.bias"], 0, False),
                                            ("512->2048 GELU", 512, 2048, sd64[p + "1.1.fn.0.weight"].float(), sd64[p + "1.1.fn.0.bias"], 1, False),
                                            ("2048->512 +x in place", 2048, 512, sd64[p + "1.1.fn.3.weight"].float(), sd64[p + "1.1.fn.3.bias"], 0, True),
                                            ("512->1040", 512, _S * 130, sd64[p + "15.weight"].float(), sd64[p + "15.bias"], 0, False)):
        rows = N if Nout == _S * 130 else M
        X = torch.randn((rows + 1, K), generator=g).cuda()
        X[rows] = 1e30
        W = W.contiguous()
        bf = b.float().contiguous()
        ybuf = torch.randn((rows + 1, Nout), generator=g).cuda() if alias else torch.full((rows + 1, Nout), float("nan"), device="cuda")
        if alias:
            ybuf[rows] = float("nan")
        y0 = ybuf[:rows].clone()
        native.check(native.lib().sampt_linear_f32(ctx.handle, native.ptr(X), c_int(K), native.ptr(W), c_int(K), native.ptr(bf),
                                                   native.ptr(ybuf) if alias else native.ptr(None), c_int(Nout), native.ptr(ybuf),
                                                   c_int(Nout), c_int(rows), c_int(Nout), c_int(K), c_int(act), native.stream_ptr()))
        torch.cuda.synchronize()
        assert torch.isnan(ybuf[rows]).all(), "guard row written"
        x64, w64 = X[:rows].double(), W.double()
        v = x64 @ w64.T + b
        tol = _gamma(K + 1) * (x64.abs() @ w64.abs().T + b.abs())
        if act == 1:
            tol = 1.13 * tol + 2 * _U * F.gelu(v).abs()
            v = F.gelu(v)
        if alias:
            v = v + y0.double()
            tol = tol + _U * v.abs()
        _report(f"sgemm {what} N={N} (M={rows})", (ybuf[:rows].double() - v).abs(), tol + 1e-45)


def _ln64(x, g, b):
    """float64 LayerNorm over the last axis and the bound of the kernel's fp32 row LayerNorm (mixer_token_kernel: 256 threads x 2
    values, block sums n = 9 for the mean and the centred variance, rstd by sqrtf and a division, (x - m) rstd g + b)"""
    m = x.mean(-1, keepdim=True)
    d = x - m
    var = (d ** 2).mean(-1, keepdim=True)
    r = 1 / torch.sqrt(var + 1e-5)
    y = d * r * g + b
    dm = _gamma(9) * x.abs().mean(-1, keepdim=True) + _U * m.abs()
    eps_r = 0.5 * (_gamma(11) * var + dm ** 2 + 2 * dm * d.abs().mean(-1, keepdim=True)) / (var + 1e-5) + 2 * _U
    tol = g.abs() * r * (dm + _U * d.abs()) * (1 + eps_r) + d.abs() * r * g.abs() * (eps_r + 2 * _U) + _U * y.abs()
    return y, r, tol


def _ln_propagate(x, g, r, dx):
    """first-order effect on LayerNorm(x) of an input error |dx| <= dx"""
    d = x - x.mean(-1, keepdim=True)
    return g.abs() * r * (dx + dx.mean(-1, keepdim=True) + d.abs() * r ** 2 * (d.abs() * dx).mean(-1, keepdim=True))


@pytest.mark.parametrize("layer", [0, 11])
def test_mixer_token(model, layer):
    """token mixing of one mixer layer, then the channel-mixing LayerNorm; and the final LayerNorm alone.  Rows include a large
    common offset (LayerNorm conditioning); inactive points stay untouched.  Token MLP: S -> 4S fma chain from the bias
    (n = 9), GELU (slope <= 1.13, 4 u), 4S -> S (n = 33), then x + out (u)."""
    m, sd64 = model
    N = 37
    g = torch.Generator().manual_seed(layer)
    x = torch.randn((N, _S, 512), generator=g)
    x[::3] += torch.randn((len(range(0, N, 3)), _S, 1), generator=g) * 300      # large common offsets per row
    x = x.cuda()
    active = np.ones(N, dtype=np.uint8)
    active[1::5] = 0
    a = torch.from_numpy(active).bool().cuda()
    p = f"delta_block.to_delta.{layer + 1}."
    for mix in (1, 0):
        xk = x.clone()
        xln = torch.full((N, _S, 512), float("nan"), device="cuda")
        _window_op(m, 2 if mix else 3, N, 10, 0, 0, active=active, x=xk, xln=xln, layer=layer)
        assert torch.equal(xk[~a], x[~a]) and torch.isnan(xln[~a]).all(), "inactive points were written"
        x64 = x.double()
        if mix:
            xn, _, e_xn = _ln64(x64, sd64[p + "0.norm.weight"], sd64[p + "0.norm.bias"])
            w1, b1 = sd64[p + "0.fn.0.weight"][:, :, 0], sd64[p + "0.fn.0.bias"]
            w2, b2 = sd64[p + "0.fn.3.weight"][:, :, 0], sd64[p + "0.fn.3.bias"]
            h = torch.einsum("js,nsc->njc", w1, xn) + b1[:, None]
            e_h = _gamma(9) * (torch.einsum("js,nsc->njc", w1.abs(), xn.abs()) + b1.abs()[:, None]) + torch.einsum("js,nsc->njc", w1.abs(), e_xn)
            gl = F.gelu(h)
            e_gl = 1.13 * e_h + 4 * _U * h.abs()
            out = torch.einsum("sj,njc->nsc", w2, gl) + b2[:, None]
            e_out = _gamma(33) * (torch.einsum("sj,njc->nsc", w2.abs(), gl.abs()) + b2.abs()[:, None]) + torch.einsum("sj,njc->nsc", w2.abs(), e_gl)
            x_new = x64 + out
            e_x = e_out + _U * x_new.abs()
            _report(f"mixer token layer {layer} x", (xk.double() - x_new).abs()[a], e_x[a] + 1e-45)
            g2, b2n = sd64[p + "1.norm.weight"], sd64[p + "1.norm.bias"]
        else:
            assert torch.equal(xk, x), "the final LayerNorm wrote x"
            x_new, e_x = x64, torch.zeros_like(x64)
            g2, b2n = sd64["delta_block.to_delta.13.weight"], sd64["delta_block.to_delta.13.bias"]
        y, r2, e_y = _ln64(x_new, g2, b2n)
        tol = e_y + _ln_propagate(x_new, g2, r2, e_x) + 1e-45
        _report(f"mixer {'token' if mix else 'final'} LN layer {layer}", (xln.double() - y).abs()[a], tol[a])


def test_mixer_mean(model):
    m = model[0]
    N = 33
    g = torch.Generator().manual_seed(5)
    xln = torch.randn((N, _S, 512), generator=g).cuda() + 100.0
    xm = torch.full((N * 512 + 512,), float("nan"), device="cuda")
    _window_op(m, 4, N, 10, 0, 0, x=xm, xln=xln)
    _guard_ok(xm, N * 512)
    ref = xln.double().mean(1)
    _report("mixer mean", (xm[: N * 512].view(N, 512).double() - ref).abs(), _gamma(9) * xln.double().abs().mean(1) + 1e-45)


# ======================================================================================================= linking
def _link_restated(vis_col, f, n_missing, S, thr0):
    """pips/tracker.py:138-145 for one point, in fp32 arithmetic like the kernel"""
    thr = np.float32(thr0)
    earliest, last = f + 1, f + S - n_missing - 1
    nxt = last
    for _ in range(100000):
        if not (np.float32(vis_col[nxt]) <= thr):
            break
        nxt -= 1
        if nxt < earliest:
            thr = np.float32(thr - np.float32(0.02))
            nxt = last
    return nxt


@pytest.mark.parametrize("n_missing", range(7))
def test_link(model, n_missing):
    """vis head logits are controlled through one ffeat column, so the sigmoids land on both sides of thr0 - k 0.02, exactly on
    1.0 (a tie at thr0 = 1), and on exactly 0 (logit -200: every wrap until the threshold is negative)"""
    m, sd64 = model
    vw, vb = sd64["vis_predictor.0.weight"][0], sd64["vis_predictor.0.bias"][0]
    k0 = int(vw.abs().argmax())
    T, f = 20, 5
    rng = np.random.default_rng(n_missing)
    cases = []
    for thr0 in (0.9, 1.0, 0.5):
        for pattern in ("steps", "ones", "zeros", "random", "falling"):
            cases.append((thr0, pattern))
    N = len(cases)
    logits = np.zeros((N, _S))
    for n, (thr0, pattern) in enumerate(cases):
        if pattern == "steps":
            p = thr0 - 0.02 * rng.integers(0, 4, _S) + rng.choice([-1e-7, 1e-7, 0.0], _S)
            logits[n] = np.log(np.clip(p, 1e-6, 1 - 1e-7) / (1 - np.clip(p, 1e-6, 1 - 1e-7)))
        elif pattern == "ones":
            logits[n] = 30.0
        elif pattern == "zeros":
            logits[n] = -200.0
        elif pattern == "falling":
            logits[n] = np.linspace(4.0, -2.0, _S)                  # visibilities fall strictly along the window
        else:
            logits[n] = rng.normal(0, 3, _S)
    ffeats = torch.zeros((N, _S, 128), dtype=torch.float64)
    ffeats[:, :, k0] = (torch.from_numpy(logits) - vb.item()) / vw[k0].item()
    ffeats = ffeats.float().cuda()
    coords = (torch.rand((N, _S, 2), generator=torch.Generator().manual_seed(3)) * 100).cuda()
    results = {}
    for thr0 in (0.9, 1.0, 0.5):
        sel = [n for n, c in enumerate(cases) if c[0] == thr0]
        active = np.zeros(N, dtype=np.uint8)
        active[sel] = 1
        vis = torch.full((T + 1, N), float("nan"), device="cuda")
        traj = torch.full((T + 1, N, 2), float("nan"), device="cuda")
        cur = torch.full((N,), -7, dtype=torch.int32, device="cuda")
        _window_op(m, 6, N, T, f, n_missing, active=active, coords=coords, ffeats=ffeats, traj=traj, vis=vis, cur=cur, thr0=thr0)
        a = torch.from_numpy(active).bool().cuda()
        lo, hi = f + 1, f + _S - n_missing            # frames written: (f, f + S - 1 - n_missing]
        outside = torch.ones(T + 1, dtype=torch.bool)
        outside[lo:hi] = False
        assert torch.isnan(vis[outside]).all() and torch.isnan(traj[outside]).all(), "frames outside the window were written"
        assert torch.isnan(vis[:, ~a]).all() and (cur[~a] == -7).all(), "inactive points were written"
        assert torch.equal(traj[lo:hi][:, a], (coords[a][:, 1: _S - n_missing] * 4.0).transpose(0, 1)), "traj = coords * stride"
        lg = ffeats.double()[:, :, k0] * vw[k0] + vb
        sig = torch.sigmoid(lg)
        got = vis[lo:hi].T.double()
        ref = sig[:, 1: _S - n_missing]
        tol = ref * (1 - ref) * (2 * _U * (lg.abs()[:, 1: _S - n_missing] + vb.abs()) + 2 * _U) + 3 * _U * ref + 1e-45
        _report(f"link vis n_missing={n_missing} thr0={thr0}", (got - ref).abs()[a], tol[a])
        vis_h = vis.cpu().numpy()
        cur_h = cur.cpu().numpy()
        for n in sel:
            results[(thr0, cases[n][1])] = int(cur_h[n])
            assert cur_h[n] == _link_restated(vis_h[:, n], f, n_missing, _S, thr0), (n, cases[n], n_missing)
        if thr0 == 0.9:
            first_vis = vis_h
    print(f"link n_missing={n_missing}: cur = {results}")
    # ties by construction: thr0 is a visibility the kernel has just returned, at a frame k after which visibilities only fall.
    # `<=` walks past the tie and stops at k - 1 (or at k after a wrap when k is the earliest frame); `<` would stop at k.
    nd = cases.index((0.9, "falling"))
    only = np.zeros(N, dtype=np.uint8)
    only[nd] = 1
    for k in range(lo, hi):
        tie = float(np.float32(first_vis[k, nd]))
        vis = torch.full((T + 1, N), float("nan"), device="cuda")
        traj = torch.full((T + 1, N, 2), float("nan"), device="cuda")
        cur = torch.full((N,), -7, dtype=torch.int32, device="cuda")
        _window_op(m, 6, N, T, f, n_missing, active=only, coords=coords, ffeats=ffeats, traj=traj, vis=vis, cur=cur, thr0=tie)
        assert float(vis[k, nd]) == tie, "the visibility changed between two identical calls"
        got = int(cur[nd])
        assert got == _link_restated(vis.cpu().numpy()[:, nd], f, n_missing, _S, tie)
        assert got == (k - 1 if k > lo else k), (k, got)


# ======================================================================================================= encoder, window and clip
# End to end, each output's error against float64 must stay within 4x the float32 oracle's own error plus 2^-20 of its largest
# value.  The float32 oracle runs on the GPU with TF32 off, so its convolutions and matmuls are plain fp32.
@pytest.fixture()
def no_tf32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _within_oracle(what, got, ref64, ref32):
    e = (got.double() - ref64).abs().max().item()
    e32 = (ref32.double() - ref64).abs().max().item()
    bound = 4 * e32 + 2.0 ** -20 * ref64.abs().max().item()
    print(f"{what}: err {e:.3g}, float32 oracle err {e32:.3g}, err / bound {e / bound if bound else 0:.3g}")
    assert e <= bound, (what, e, e32)


def _sd32(sd64):
    return {k: v.float() for k, v in sd64.items()}


def test_fnet_end_to_end(model, no_tf32):
    """sampt_pips_fnet on C2 frames: all black (every channel of every stage is constant: the instance-norm edge), letterboxed
    (black bars above and below a textured picture) and a ramp rising one grey level every 3 columns"""
    m, sd64 = model
    H, W = 480, 854
    black = torch.zeros((3, H, W), dtype=torch.uint8)
    letterbox = synth.make_clip(1, H, W, seed=21)["frames"][0].clone()
    letterbox[:, :60], letterbox[:, -60:] = 0, 0
    ramp = ((torch.arange(W) // 3) % 256).to(torch.uint8).expand(3, H, W).contiguous()
    sd32 = _sd32(sd64)
    for name, fr in (("black", black), ("letterbox", letterbox), ("ramp", ramp)):
        got = m.fnet_frames(fr[None].cuda()).permute(0, 3, 1, 2)
        x64 = 2 * (fr[None].cuda().double() / 255.0) - 1.0
        ref64 = pips_ref.fnet(sd64, x64)
        ref32 = pips_ref.fnet(sd32, 2 * (fr[None].cuda().float() / 255.0) - 1.0)
        _within_oracle(f"fnet {name}", got, ref64, ref32)


def _c2_features(m, T, seed):
    """the GPU's own encoder output of a synthetic C2 clip: the same feature maps go to the kernel chain and to both oracles"""
    clip = synth.make_clip(T, 480, 854, seed=seed)
    fm = torch.cat([m.fnet_frames(clip["frames"][i:i + 8].cuda()) for i in range(0, T, 8)])
    return clip, fm


@pytest.mark.parametrize("N", [1, 8, 64, 292])
def test_window_end_to_end(model, no_tf32, N):
    """sampt_pips_window (Pips.forward on one 8-frame window) at the C2 geometry: per-iteration coordinates, visibility logits
    and the returned feature"""
    m, sd64 = model
    clip, fm = _c2_features(m, _S, seed=40 + N)
    pyr = m.build_pyramid(fm)
    xys = synth.make_query_points(clip, N, seed=N)[0, :, 1:].cuda().contiguous()
    coords_out = torch.empty((6, _S, N, 2), device="cuda")
    vis_e = torch.empty((_S, N), device="cuda")
    ffeat = torch.empty((N, 128), device="cuda")
    native.check(native.lib().sampt_pips_window(
        _ctx(m).handle, native.ptr(pyr[0]), native.ptr(pyr[1]), native.ptr(pyr[2]), native.ptr(pyr[3]), c_int(_C2[0]), c_int(_C2[1]),
        native.ptr(xys), native.ptr(None), native.ptr(None), c_int(N), c_int(_S), c_int(4), c_int(6), native.ptr(coords_out),
        native.ptr(vis_e), native.ptr(ffeat), native.stream_ptr()), "pips_window")
    torch.cuda.synchronize()
    fmn = fm.permute(0, 3, 1, 2)[None]
    p64, v64, f64 = pips_ref.pips_forward(sd64, xys.double()[None], None, None, 6, fmaps=fmn.double())
    p32, v32, f32 = pips_ref.pips_forward(_sd32(sd64), xys[None], None, None, 6, fmaps=fmn)
    for it in range(6):
        _within_oracle(f"window N={N} coords iteration {it}", coords_out[it], p64[it][0], p32[it][0])
    _within_oracle(f"window N={N} vis logits", vis_e, v64[0], v32[0])
    _within_oracle(f"window N={N} feature", ffeat, f64[0], f32[0])


@pytest.mark.parametrize("N", [8, 37])
def test_clip_end_to_end(model, no_tf32, N):
    """sampt_pips_track over 50 frames at 120x213, both directions; with N = 37 a third of the points are born mid-clip.
    Trajectories follow the 4x rule; boolean visibilities must equal the float64 oracle's except where the float32 oracle also
    disagrees with it"""
    m, sd64 = model
    T = 50
    clip, fm = _c2_features(m, T, seed=70 + N)
    pyr = m.build_pyramid(fm)
    q = synth.make_query_points(clip, N, seed=N)[0].clone()
    if N > 8:
        q[::3, 0] = torch.randint(1, T - 1, (len(range(0, N, 3)),), generator=torch.Generator().manual_seed(N)).float()
    rg = torch.zeros((1, T, 3, 1, 1), dtype=torch.uint8)
    fmn = fm.permute(0, 3, 1, 2)
    sd32 = _sd32(sd64)
    for flip in (False, True):
        traj, vis = m.track(pyr, q.cuda(), 0.9, flip=flip)
        qf = q.clone()
        fmo = fmn
        if flip:
            qf[:, 0] = T - 1 - qf[:, 0]
            fmo = fmn.flip(0)
        t64, b64 = pips_ref.track_one_direction(sd64, rg, qf.cuda().double()[None], fmaps_all=fmo.double())
        t32, b32 = pips_ref.track_one_direction(sd32, rg, qf.cuda()[None], fmaps_all=fmo)
        _within_oracle(f"clip N={N} flip={flip} trajectories", traj, t64[0], t32[0])
        ours, r64, r32 = vis > 0.5, b64[0], b32[0]
        excused = r32 != r64
        bad = (ours != r64) & ~excused
        print(f"clip N={N} flip={flip}: visibilities differing from float64: {int((ours != r64).sum())}, "
              f"float32 oracle differs at {int(excused.sum())}, unexplained {int(bad.sum())}")
        assert not bad.any()
