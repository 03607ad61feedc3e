"""GPU: the CoTracker window (csrc/cotracker.cu) kernel by kernel against float64, through the unit-test entries of
include/sampt_b200.h (sampt_test_cotracker_input / _ln / _attn / _block / _update), sampt_linear_f32, sampt_resize_bilinear_u8_f32
and sampt_cotracker_sample_features; then the whole window and the tracker at the C3 / C5 point counts against the float64 oracle.

Bounds are derived from fp32 rounding, u = 2^-24, and the summation length n of the kernel under test (gamma_n = n u / (1 - n u));
the float64 reference is computed from exactly the fp32 operands the kernel reads.  Each group prints its worst error / bound.
Outputs start as NaN with a guard row: rows the kernel must not write stay NaN.  Inputs carry a guard row of 1e30, so an over-read
turns an output into garbage.  Point counts N = 1 ... 292 (M = 8 N token rows) reach every sgemm_nt dispatch branch, both sides of
the window's M = 128 switch to tensor-core GEMMs, M not a multiple of 128, and the C3 (84) and C5 (292) counts."""
import math
from ctypes import c_int

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import cotracker_ref as R
from oracle import pips_ref
from sampt_b200 import native, synth
from tests.test_gpu_pips_kernels import _corr_expected

pytestmark = pytest.mark.gpu

_U = 2.0 ** -24
_S = 8
_HID = 384
_H4, _W4 = 96, 128                 # level-0 feature map of CoTracker's 384x512 interp_shape; levels 48x64, 24x32, 12x16
_NS = [1, 4, 9, 15, 16, 37, 84, 292]


def _gamma(n):
    return n * _U / (1 - n * _U)


def _report(what, err, bound):
    worst = (err / bound).max().item()
    print(f"{what}: max err {err.max().item():.3g}, worst err / bound {worst:.3g}")
    assert worst <= 1.0, (what, worst)


def _guarded(t, fill=1e30):
    row = t.shape[-1] if t.dim() else 1
    buf = torch.cat([t.reshape(-1).float().cuda(), torch.full((row,), fill, device="cuda")])
    return buf, buf[: t.numel()].view(t.shape)


def _nan_out(shape, guard_row, dtype=torch.float32):
    buf = torch.full((math.prod(shape) + guard_row,), float("nan"), device="cuda", dtype=dtype)
    return buf, buf[: math.prod(shape)].view(shape)


def _guard_ok(buf, n):
    torch.cuda.synchronize()
    assert torch.isnan(buf[n:]).all(), "a value past the output was written"


@pytest.fixture(scope="module")
def model():
    from sam_pt.point_tracker.cotracker.cotracker import CoTracker, cotracker_shapes
    sd = synth.condition_cotracker(synth.make_state_dict(cotracker_shapes(), 31))
    m = CoTracker()
    m.load_state_dict(sd)
    m = m.cuda().eval()
    m.native_context()                      # registers the fp32 weights and the UpdateFormer's fp16 hi | lo ".w16" copies
    return m, {k: v.cuda().double() for k, v in sd.items()}


def _h(m):
    return m.native_context().handle


# ======================================================================================================= resize and sampling
@pytest.mark.parametrize("H,W,Ho,Wo", [(480, 854, 384, 512), (1080, 1920, 384, 512), (80, 112, 96, 128), (384, 512, 384, 512),
                                       (61, 107, 384, 512), (3, 5, 384, 512)])
def test_resize(model, H, W, Ho, Wo):
    """against ATen's float32 F.interpolate (what the reference wrapper runs), and against a float64 evaluation of the same
    formula whose bound carries the fp32 source-coordinate rounding (a few ulps of the coordinate, times 255 per axis)"""
    m = model[0]
    g = torch.Generator().manual_seed(H + W)
    fr = torch.randint(0, 256, (2, 3, H, W), generator=g, dtype=torch.uint8)
    fr[0, :, : H // 2] = 255 * ((torch.arange(W) // 2) % 2).to(torch.uint8)        # one-pixel stripes: the largest neighbour steps
    inb = torch.cat([fr.reshape(-1), torch.full((W,), 255, dtype=torch.uint8)]).cuda()
    obuf, out = _nan_out((6, Ho, Wo), Wo)
    native.check(native.lib().sampt_resize_bilinear_u8_f32(_h(m), native.ptr(inb), c_int(6), c_int(H), c_int(W), c_int(Ho), c_int(Wo),
                                                           native.ptr(obuf), native.stream_ptr()), "resize")
    _guard_ok(obuf, out.numel())
    got = out.view(2, 3, Ho, Wo).cpu().double()
    aten = F.interpolate(fr.float(), (Ho, Wo), mode="bilinear", align_corners=False).double()

    def axis(n_in, n_out):
        src = ((np.arange(n_out) + 0.5) * (n_in / n_out) - 0.5).clip(0)
        i0 = np.minimum(np.floor(src).astype(np.int64), n_in - 1)
        i1 = np.minimum(i0 + 1, n_in - 1)
        err = 4 * _U * (src + 1) + 2.0 ** -23 * (n_in / n_out) * (np.arange(n_out) + 0.5)
        return torch.from_numpy(i0), torch.from_numpy(i1), torch.from_numpy(src - i0), torch.from_numpy(err)
    y0, y1, ly, ey = axis(H, Ho)
    x0, x1, lx, ex = axis(W, Wo)
    v = fr.double()
    ly, ey, lx, ex = ly[:, None], ey[:, None], lx[None, :], ex[None, :]
    c00, c01, c10, c11 = v[..., y0, :][..., x0], v[..., y0, :][..., x1], v[..., y1, :][..., x0], v[..., y1, :][..., x1]
    ref = (1 - ly) * ((1 - lx) * c00 + lx * c01) + ly * ((1 - lx) * c10 + lx * c11)      # values >= 0: also sum |w v|
    tol = 255.0 * (ey + ex) + 8 * _U * ref + 1e-45
    _report(f"resize {H}x{W}->{Ho}x{Wo} vs ATen float32", (got - aten).abs(), 2 * tol)
    _report(f"resize {H}x{W}->{Ho}x{Wo} vs float64", (got - ref).abs(), tol)


@pytest.mark.parametrize("S", [1, 8])
def test_sample_features(model, S):
    """bilinear_sample2d at integer and fractional positions, on the last row / column, up to 2 px outside (clamped indices,
    unclamped weights: the sample extrapolates) and at negative coordinates, each point on its own frame"""
    m = model[0]
    g = torch.Generator().manual_seed(S)
    T = 5
    fm = (torch.randn((T, _H4, _W4, 128), generator=g) * 0.5).cuda()
    fmb = torch.cat([fm.reshape(-1), torch.full((128,), 1e30, device="cuda")])
    xy = torch.tensor([[10.0, 20.0], [10.25, 20.75], [_W4 - 1.0, 7.5], [33.5, _H4 - 1.0], [_W4 - 1.0, _H4 - 1.0], [-2.0, 40.0],
                       [_W4 + 1.0, 30.5], [64.5, _H4 + 1.75], [-0.5, -1.25], [-1.75, 50.0], [5.0, -2.0], [0.0, 0.0],
                       [127.9, 95.1], [_W4 - 0.5, -0.5]])
    N = xy.shape[0]
    frame = (torch.arange(N) % T).to(torch.int32).cuda()
    xyb, xyg = _guarded(xy)
    obuf, out = _nan_out((N, S, 128), 128)
    native.check(native.lib().sampt_cotracker_sample_features(_h(m), native.ptr(fmb), c_int(_H4), c_int(_W4), native.ptr(frame),
                                                              native.ptr(xyb), c_int(N), c_int(S), native.ptr(obuf),
                                                              native.stream_ptr()), "sample_features")
    _guard_ok(obuf, out.numel())
    assert torch.equal(out, out[:, :1].expand(-1, S, -1)), "slots differ"
    x, y = xyg[:, 0].double(), xyg[:, 1].double()
    ref = torch.stack([pips_ref.bilinear_sample2d(fm[int(frame[n])].permute(2, 0, 1)[None].double(), x[n:n + 1][None],
                                                  y[n:n + 1][None])[0, :, 0] for n in range(N)])
    x0, y0 = torch.floor(x), torch.floor(y)
    mag = torch.zeros_like(ref)
    for dx, dy in ((0, 0), (1, 0), (0, 1), (1, 1)):
        w = ((x - x0) if dx else (x0 + 1 - x)).abs() * ((y - y0) if dy else (y0 + 1 - y)).abs()
        xi, yi = (x0 + dx).long().clamp(0, _W4 - 1), (y0 + dy).long().clamp(0, _H4 - 1)
        mag += w[:, None] * fm[frame.long(), yi, xi].double().abs()
    _report(f"sample features S={S}", (out[:, 0].double() - ref).abs(), 8 * _U * mag + 1e-45)


# ======================================================================================================= input rows
def _pyramid(T, seed):
    g = torch.Generator().manual_seed(seed)
    fm = (torch.randn((T, 128, _H4, _W4), generator=g) * 0.5).cuda()
    return [p[0].permute(0, 2, 3, 1).contiguous() for p in pips_ref.build_pyramid(fm[None])]     # (T, H_l, W_l, 128)


def _input_coords(N, g):
    """slot 0: interior, integers, the last row / column, a few px outside and negative; later slots add flows up to +-100 px"""
    c0 = torch.rand((N, 2), generator=g) * torch.tensor([_W4 - 1.0, _H4 - 1.0])
    special = torch.tensor([[20.0, 30.0], [_W4 - 1.0, 40.0], [50.0, _H4 - 1.0], [_W4 - 1.0, _H4 - 1.0], [-2.5, 10.0], [_W4 + 2.0, 33.0],
                            [64.0, -3.25], [-0.75, -0.5], [120.5, 90.5], [0.0, 0.0]])
    for n in range(0, N, 2):
        c0[n] = special[(n // 2) % len(special)]
    flow = (torch.rand((N, _S, 2), generator=g) * 2 - 1) * torch.linspace(0, 100, _S)[None, :, None]
    flow[1::3] = torch.round(flow[1::3])
    co = c0[:, None] + flow
    co[:, 0] = c0
    return co


@pytest.mark.parametrize("N", [1, 9, 84, 292])
def test_input_rows(model, N):
    m = model[0]
    T = 10
    lv = _pyramid(T, seed=N)
    bufs = [torch.cat([p.reshape(-1), torch.full((128,), 1e30, device="cuda")]) for p in lv]
    g = torch.Generator().manual_seed(100 + N)
    co = _input_coords(N, g)
    ff = torch.randn((N, _S, 128), generator=g)
    tm = (torch.rand((N, _S), generator=g) < 0.7).float()
    vi = torch.randn((N, _S), generator=g) * 5
    cob, cog = _guarded(co)
    ffb, ffg = _guarded(ff)
    tmb, tmg = _guarded(tm)
    vib, vig = _guarded(vi)
    tab = m._time_emb
    t64 = torch.from_numpy(R._sincos_1d(R.IN_DIM, np.arange(_S, dtype=np.float64))).cuda()
    _report("time table fp32 rounding", (tab.double() - t64).abs(), _U * t64.abs() + 1e-45)
    for name, slots in (("identity", list(range(8))), ("tail-repeated", [4, 5, 6, 7, 8, 9, 9, 9]), ("reversed", [9, 8, 7, 6, 5, 4, 3, 2])):
        pbuf, pos = _nan_out((N, R.IN_DIM), R.IN_DIM)
        xbuf, xin = _nan_out((N * _S, R.IN_DIM), R.IN_DIM)
        native.check(native.lib().sampt_test_cotracker_input(
            _h(m), native.ptr(bufs[0]), native.ptr(bufs[1]), native.ptr(bufs[2]), native.ptr(bufs[3]), c_int(_H4), c_int(_W4),
            (c_int * 8)(*slots), native.ptr(cob), native.ptr(ffb), native.ptr(tmb), native.ptr(vib), native.ptr(tab), c_int(N),
            native.ptr(pbuf), native.ptr(xbuf), native.stream_ptr()), "test_cotracker_input")
        _guard_ok(pbuf, pos.numel())
        _guard_ok(xbuf, xin.numel())
        # pos: the float64 table rounded to fp32 (u), then the 4-term fp32 bilinear with fp32 weights (8 u of sum |w t|)
        c0 = cog[:, 0].double()[None]
        pref = R.sample_pos_embed((_H4, _W4), R.IN_DIM, c0)[0]
        x0, y0 = torch.floor(c0[0, :, 0]), torch.floor(c0[0, :, 1])
        tab64 = torch.from_numpy(R.get_2d_sincos_pos_embed(R.IN_DIM, (_H4, _W4))).cuda().view(_H4, _W4, R.IN_DIM)
        pmag = torch.zeros_like(pref)
        for dx, dy in ((0, 0), (1, 0), (0, 1), (1, 1)):
            w = ((c0[0, :, 0] - x0) if dx else (x0 + 1 - c0[0, :, 0])).abs() * ((c0[0, :, 1] - y0) if dy else (y0 + 1 - c0[0, :, 1])).abs()
            pmag += w[:, None] * tab64[(y0 + dy).long().clamp(0, _H4 - 1), (x0 + dx).long().clamp(0, _W4 - 1)].abs()
        _report(f"pos N={N} {name}", (pos.double() - pref).abs(), 9 * _U * pmag + 1e-45)
        rows = xin.view(N, _S, R.IN_DIM)
        base = (pos.double()[:, None, :].abs() + tab.double()[None].abs())

        def exact(cols, v):     # the kernel adds (v + pos) + time
            assert torch.equal(rows[..., cols], (v + pos[:, None, cols]) + tab[None, :, cols]), (name, cols)

        def bounded(what, cols, v64, e64):
            ref = v64 + pos.double()[:, None, cols] + tab.double()[None, :, cols]
            tol = e64 * (1 + 4 * _U) + 2 * _U * (v64.abs() + base[..., cols]) + 1e-45
            _report(f"{what} N={N} {name}", (rows[..., cols].double() - ref).abs(), tol)
        flow = cog - cog[:, :1]
        exact(slice(0, 2), flow)
        exact(slice(326, 454), ffg)
        exact(slice(454, 455), tmg[..., None])
        exact(slice(455, 456), vig[..., None])
        # flow embedding: [sincos(x) | sincos(y)], sin at even, cos at odd columns; fp32 argument (u |arg|), sinf / cosf (2 ulp)
        div = torch.arange(0, 64, 2, device="cuda", dtype=torch.float64) * (1000.0 / 64)
        arg = flow.double()[..., :, None] * div                                         # (N, S, 2, 32)
        emb = torch.stack([torch.sin(arg), torch.cos(arg)], dim=-1).reshape(N, _S, 128)
        e_emb = (2.0 ** -23 * arg.abs()).repeat_interleave(2, dim=-1).reshape(N, _S, 128) + 2.0 ** -22
        bounded(f"flow embedding (|arg| up to {arg.abs().max().item():.3g})", slice(2, 130), emb, e_emb)
        # correlation: the same gather as PIPS (tests/test_gpu_pips_kernels.py), from the kernel's fp32 round-trip sample positions
        cexp, ctol = _corr_expected(lv, ffg, cog, slots)
        bounded("corr", slice(130, 326), cexp.view(N, _S, 196), ctol.view(N, _S, 196))


# ======================================================================================================= LayerNorm and split
def _ln64(x):
    """float64 LayerNorm (no affine, eps 1e-6) of the fp32 rows x and the bound of ln384_kernel: per lane 12 values in 3 float4
    groups, a 5-level warp tree (sums of n = 17), times fl(1/384) (2 u); the centred variance (n = 18, with the fp32 mean's
    error dm entering squared), rstd by sqrtf and a division; (x - m) rstd"""
    m = x.mean(-1, keepdim=True)
    d = x - m
    var = (d ** 2).mean(-1, keepdim=True)
    r = 1 / torch.sqrt(var + 1e-6)
    y = d * r
    dm = _gamma(17) * x.abs().mean(-1, keepdim=True) + 2 * _U * m.abs()
    eps_r = 0.5 * (_gamma(20) * (var + dm ** 2) + dm ** 2 + _U * 1e-6) / (var + 1e-6) + 3 * _U
    tol = r * (dm + _U * d.abs()) * (1 + eps_r) + d.abs() * r * (eps_r + _U)
    return y, r, tol


def _ln_propagate(x, r, dx):
    """first-order effect on LayerNorm(x) (no affine) of an input error |dx| <= dx"""
    d = x - x.mean(-1, keepdim=True)
    return r * (dx + dx.mean(-1, keepdim=True) + d.abs() * r ** 2 * (d.abs() * dx).mean(-1, keepdim=True))


def _ln_rows(M, g):
    x = torch.randn((M, _HID), generator=g) * (torch.rand((M, 1), generator=g) * 3 + 0.1)
    x[::3] = 1e3 + 0.05 * torch.randn((len(range(0, M, 3)), _HID), generator=g)     # large common offset, tiny variance
    x[1::7] += 40.0
    return x


@pytest.mark.parametrize("M", [8 * n for n in _NS] + [13, 2337])
def test_layernorm_and_split(model, M):
    m = model[0]
    g = torch.Generator().manual_seed(M)
    xb, xg = _guarded(_ln_rows(M, g))
    ybuf, y = _nan_out((M, _HID), _HID)
    native.check(native.lib().sampt_test_cotracker_ln(_h(m), c_int(0), native.ptr(xb), c_int(M), c_int(_HID), native.ptr(ybuf),
                                                      native.ptr(None), native.stream_ptr()), "test_cotracker_ln 0")
    _guard_ok(ybuf, y.numel())
    ref, _, tol = _ln64(xg.double())
    _report(f"layernorm M={M}", (y.double() - ref).abs(), tol + 1e-45)
    # the split LayerNorm: hi = fp16(v), lo = fp16(v - hi) of the same fp32 value v, row pitch 768
    hbuf, h = _nan_out((M, 2 * _HID), 2 * _HID, torch.float16)
    native.check(native.lib().sampt_test_cotracker_ln(_h(m), c_int(1), native.ptr(xb), c_int(M), c_int(_HID), native.ptr(None),
                                                      native.ptr(hbuf), native.stream_ptr()), "test_cotracker_ln 1")
    _guard_ok(hbuf, h.numel())
    _check_split(f"split layernorm M={M}", y, h)
    # the plain split of [M, K]
    for K in (384, 1536):
        x = torch.randn((M, K), generator=g) * torch.logspace(-6, 3, K)[torch.randperm(K, generator=g)]
        xb2, xg2 = _guarded(x)
        sbuf, s16 = _nan_out((M, 2 * K), 2 * K, torch.float16)
        native.check(native.lib().sampt_test_cotracker_ln(_h(m), c_int(2), native.ptr(xb2), c_int(M), c_int(K), native.ptr(None),
                                                          native.ptr(sbuf), native.stream_ptr()), "test_cotracker_ln 2")
        _guard_ok(sbuf, s16.numel())
        _check_split(f"split M={M} K={K}", xg2, s16)


def _check_split(what, v, h):
    K = v.shape[1]
    hi, lo = h[:, :K], h[:, K:]
    assert torch.equal(hi, v.half()), f"{what}: hi != fp16(v)"
    assert torch.equal(lo, (v - hi.float()).half()), f"{what}: lo != fp16(v - hi)"
    err = (hi.double() + lo.double() - v.double()).abs()
    _report(what, err, 2.0 ** -11 * (v.double() - hi.double()).abs() + 2.0 ** -25)


# ======================================================================================================= attention core
def _attn64(qkv, G, L, gstride, lstride):
    """float64 softmax(q k^T / sqrt(48)) v per (group, head), the gathered token rows and the kernel's bound: fma chains of 48
    (scores) and L (output), fl(1/sqrtf(48)) (2 u), expf (2 ulp) of an fp32 difference, the sum of L exponentials and 1 / sum"""
    rows = (torch.arange(G, device="cuda")[:, None] * gstride + torch.arange(L, device="cuda")[None] * lstride)     # (G, L)
    t = qkv.double()[rows].view(G, L, 3, 8, 48).permute(2, 0, 3, 1, 4)                                           # (3, G, H, L, 48)
    q, k, v = t[0], t[1], t[2]
    sc = 48 ** -0.5
    s = q @ k.transpose(-1, -2) * sc
    p = s.softmax(-1)
    o = p @ v
    e_s = _gamma(48) * (q.abs() @ k.abs().transpose(-1, -2)) * sc + 3 * _U * s.abs()
    spread = (s - s.max(-1, keepdim=True).values).abs()
    delta = (2 * e_s.max(-1, keepdim=True).values + _U * spread + 2 * _U)                      # per-weight relative error
    dmax = delta.max(-1, keepdim=True).values
    tol = (p * 2 * dmax) @ v.abs() + (_gamma(L + 40) + 2 * _U) * (p @ v.abs()) + _U * o.abs()
    return rows, o, tol, (q, k, v, p, s)


def _attn_qkv(G, L, gstride, lstride, M, pattern, g):
    qkv = torch.randn((M, 3 * _HID), generator=g)
    rows = (torch.arange(G)[:, None] * gstride + torch.arange(L)[None] * lstride).reshape(-1)
    if pattern == "dominant":
        qkv.view(M, 3, 8, 48)[rows.view(G, L)[:, L // 2], 1] *= 6.0              # one key far above the others in every group
    elif pattern == "equal":
        qkv.view(M, 3, 8, 48)[rows, 1] = qkv.view(M, 3, 8, 48)[rows[:1], 1]      # identical keys: uniform weights
    return qkv


def _run_attn(m, qkv, M, G, L, gstride, lstride, qsplit):
    qb, qg = _guarded(qkv)
    obuf, out = _nan_out((M, _HID), _HID)
    rc = native.lib().sampt_test_cotracker_attn(_h(m), native.ptr(qb), native.ptr(obuf), c_int(G), c_int(L), c_int(gstride),
                                                c_int(lstride), c_int(qsplit), native.stream_ptr())
    return rc, qg, obuf, out


@pytest.mark.parametrize("N", _NS)
@pytest.mark.parametrize("layout", ["time", "space"])
def test_attention_core(model, N, layout):
    m = model[0]
    M = N * _S
    G, L, gs, ls = (N, _S, _S, 1) if layout == "time" else (_S, N, 1, _S)
    g = torch.Generator().manual_seed(N * 3 + (layout == "space"))
    for pattern in ("random", "dominant", "equal"):
        qkv = _attn_qkv(G, L, gs, ls, M, pattern, g)
        prev = None
        for qsplit in (1, 2, 8, 0):
            rc, qg, obuf, out = _run_attn(m, qkv, M, G, L, gs, ls, qsplit)
            native.check(rc, "test_cotracker_attn")
            _guard_ok(obuf, out.numel())
            rows, o, tol, _ = _attn64(qg, G, L, gs, ls)
            got = out.double()[rows].view(G, L, 8, 48).permute(0, 2, 1, 3)
            _report(f"attention {layout} N={N} {pattern} qsplit={qsplit}", (got - o).abs(), tol + 1e-45)
            if prev is not None:
                assert torch.equal(out, prev), "the query split changed a result"
            prev = out.clone()


def test_attention_strided_rows_and_limits(model):
    """a layout with gaps (rows outside the groups stay NaN) and L = 9 split 8 ways (three CTAs per group get no query);
    L = 483 is the largest group that fits 200 KB of shared memory, L = 484 is refused before any launch"""
    m = model[0]
    g = torch.Generator().manual_seed(9)
    G, L, gs, ls = 2, 9, 20, 2
    M = 40
    qkv = _attn_qkv(G, L, gs, ls, M, "random", g)
    rc, qg, obuf, out = _run_attn(m, qkv, M, G, L, gs, ls, 8)
    native.check(rc, "test_cotracker_attn strided")
    _guard_ok(obuf, out.numel())
    rows, o, tol, _ = _attn64(qg, G, L, gs, ls)
    hit = torch.zeros(M, dtype=torch.bool, device="cuda")
    hit[rows.reshape(-1)] = True
    assert torch.isnan(out[~hit]).all(), "rows outside the groups were written"
    _report("attention strided L=9 qsplit=8", (out.double()[rows].view(G, L, 8, 48).permute(0, 2, 1, 3) - o).abs(), tol + 1e-45)
    for L, ok in ((483, True), (484, False)):
        M = 8 * L
        qkv = torch.randn((M, 3 * _HID), generator=g)
        rc, qg, obuf, out = _run_attn(m, qkv, M, _S, L, 1, _S, 0)
        torch.cuda.synchronize()
        if ok:
            native.check(rc, "test_cotracker_attn L=483")
            rows, o, tol, _ = _attn64(qg, _S, L, 1, _S)
            _report("attention space L=483", (out.double()[rows].view(_S, L, 8, 48).permute(0, 2, 1, 3) - o).abs(), tol + 1e-45)
        else:
            assert rc != 0 and b"do not fit shared memory" in native.lib().sampt_last_error()
            assert torch.isnan(obuf).all(), "a refused call wrote its output"


# ======================================================================================================= sgemm at CoTracker's shapes
def _gelu_tanh_bound(v, e):
    """GELU(tanh): slope <= 1.13 times the input error, tanhf (2 ulp, absolute near +-1) and the cubic's rounding: 2 u of
    |gelu| and 2 u of |x|"""
    return 1.13 * e + 2 * _U * F.gelu(v, approximate="tanh").abs() + 2 * _U * v.abs()


@pytest.mark.parametrize("N", _NS)
def test_sgemm_shapes(model, N):
    """the six sgemm_nt calls of one window iteration at M = 8 N rows: any summation order of K terms is within
    gamma_(K+1) sum |x w| + |b|"""
    m, sd64 = model
    M = N * _S
    g = torch.Generator().manual_seed(M + 1)
    p = "updateformer."
    b0 = p + "time_blocks.0."
    for what, K, Nout, wk, act, alias in (("456->384", R.IN_DIM, _HID, p + "input_transform", 0, False),
                                          ("384->1152", _HID, 3 * _HID, b0 + "attn.qkv", 0, False),
                                          ("384->384 +x in place", _HID, _HID, b0 + "attn.proj", 0, True),
                                          ("384->1536 GELU(tanh)", _HID, 4 * _HID, b0 + "mlp.fc1", 3, False),
                                          ("1536->384 +x in place", 4 * _HID, _HID, b0 + "mlp.fc2", 0, True),
                                          ("384->130", _HID, 130, p + "flow_head", 0, False)):
        W = sd64[wk + ".weight"].float().contiguous()
        b = sd64[wk + ".bias"]
        bf = b.float().contiguous()
        X = torch.randn((M + 1, K), generator=g).cuda()
        X[M] = 1e30
        if alias:
            ybuf = torch.randn((M + 1, Nout), generator=g).cuda()
            ybuf[M] = float("nan")
        else:
            ybuf = torch.full((M + 1, Nout), float("nan"), device="cuda")
        y0 = ybuf[:M].clone()
        native.check(native.lib().sampt_linear_f32(_h(m), native.ptr(X), c_int(K), native.ptr(W), c_int(K), native.ptr(bf),
                                                   native.ptr(ybuf) if alias else native.ptr(None), c_int(Nout), native.ptr(ybuf),
                                                   c_int(Nout), c_int(M), c_int(Nout), c_int(K), c_int(act), native.stream_ptr()))
        torch.cuda.synchronize()
        assert torch.isnan(ybuf[M]).all(), "guard row written"
        x64, w64 = X[:M].double(), W.double()
        v = x64 @ w64.T + b
        tol = _gamma(K + 1) * (x64.abs() @ w64.abs().T + b.abs())
        if act == 3:
            tol = _gelu_tanh_bound(v, tol)
            v = F.gelu(v, approximate="tanh")
        if alias:
            v = v + y0.double()
            tol = tol + _U * v.abs()
        _report(f"sgemm {what} N={N} (M={M})", (ybuf[:M].double() - v).abs(), tol + 1e-45)


# ======================================================================================================= one UpdateFormer block
def _gemm_err(tc, X, e_X, W, b, v):
    """error of fl(X W^T + b) given |X - X_exact| <= e_X: the GEMM's own rounding (fp32 fma chain, or the three-pass fp16
    product of tests/test_gpu_gemm.py: 2^-21 sqrt(3K/16) + 2^-20 of the products, 2^-25 per fp16-subnormal lo operand, the
    fp32 epilogue) plus the propagated input error"""
    K = X.shape[-1]
    A = X.abs() @ W.abs().T
    if tc:
        own = ((2.0 ** -21 * (3 * K / 16) ** 0.5 + 2.0 ** -20) * A + 2.0 ** -25 * (W.abs().sum(1) + X.abs().sum(-1, keepdim=True))
               + 2.0 ** -20 * (v.abs() + b.abs()))
    else:
        own = _gamma(K + 1) * (A + b.abs())
    return own + e_X @ W.abs().T


def _block64(sd64, p, x, G, L, gstride, lstride, tc):
    """float64 AttnBlock on the fp32 input x (M, 384) and a first-order bound of the kernel chain: each stage's own rounding
    (groups LayerNorm, attention, sgemm / three-pass GEMM) plus the propagated error of its inputs"""
    x = x.double()
    h1, r1, e_h1 = _ln64(x)
    if tc:                                            # the fp16 hi | lo operand drops lo's rounding
        e_h1 = e_h1 + 2.0 ** -22 * h1.abs() + 2.0 ** -25
    wq, bq = sd64[p + "attn.qkv.weight"], sd64[p + "attn.qkv.bias"]
    qkv = h1 @ wq.T + bq
    e_qkv = _gemm_err(tc, h1, e_h1, wq, bq, qkv)
    rows, o, e_o, (q, k, v, pr, s) = _attn64(qkv, G, L, gstride, lstride)
    eq, ek, ev = [t.view(G, L, 8, 48).permute(0, 2, 1, 3) for t in e_qkv[rows].view(G, L, 3, 384).unbind(2)]
    sc = 48 ** -0.5
    ds = sc * (eq @ k.abs().transpose(-1, -2) + q.abs() @ ek.transpose(-1, -2))          # score perturbation
    e_o = e_o + pr @ ev + (pr * ds) @ v.abs() + (pr * ds).sum(-1, keepdim=True) * o.abs()     # |v_j - o_i| <= |v_j| + |o_i|
    att = torch.empty_like(x)
    e_att = torch.empty_like(x)
    att[rows.reshape(-1)] = o.permute(0, 2, 1, 3).reshape(-1, 384)
    e_att[rows.reshape(-1)] = e_o.permute(0, 2, 1, 3).reshape(-1, 384)
    if tc:
        e_att = e_att + 2.0 ** -22 * att.abs() + 2.0 ** -25
    wp, bp = sd64[p + "attn.proj.weight"], sd64[p + "attn.proj.bias"]
    pr_ = att @ wp.T + bp
    x1 = x + pr_
    e_x1 = _gemm_err(tc, att, e_att, wp, bp, pr_) + _U * x1.abs()
    h2, r2, e_h2 = _ln64(x1)
    e_h2 = e_h2 + _ln_propagate(x1, r2, e_x1)
    if tc:
        e_h2 = e_h2 + 2.0 ** -22 * h2.abs() + 2.0 ** -25
    w1, b1 = sd64[p + "mlp.fc1.weight"], sd64[p + "mlp.fc1.bias"]
    f1 = h2 @ w1.T + b1
    gl = F.gelu(f1, approximate="tanh")
    e_gl = _gelu_tanh_bound(f1, _gemm_err(tc, h2, e_h2, w1, b1, f1))
    if tc:
        e_gl = e_gl + 2.0 ** -22 * gl.abs() + 2.0 ** -25
    w2, b2 = sd64[p + "mlp.fc2.weight"], sd64[p + "mlp.fc2.bias"]
    f2 = gl @ w2.T + b2
    x2 = x1 + f2
    e_x2 = _gemm_err(tc, gl, e_gl, w2, b2, f2) + e_x1 + _U * x2.abs()
    return x2, e_x2


# Measured bar of one block: max |x - float64| / max |float64|.  The first-order bound above holds but, with the synthetic N(0, 1)
# block weights (saturated softmax, worst-case propagation through sums of 1536), it sits about 1e5 above the actual error, so
# it cannot see an error of 2^-12 in one GEMM.  Each path is therefore also held to 4x the largest relative error the fp32 path
# showed over these cases on an H100 80GB HBM3 (700 W): fp32 path 1.15e-7, tensor-core path 3.47e-7.  For scale, GELU(erf) in place
# of GELU(tanh) gives about 5e-6 on both paths, and dropping the A_lo.B_hi pass of the three-pass GEMM about 9e-6.
_BLOCK_BAR = 4.6e-7


@pytest.mark.parametrize("N", [4, 15, 16, 37, 84, 292])
@pytest.mark.parametrize("kind,blk", [(0, 0), (0, 5), (1, 0), (1, 5)])
def test_updateformer_block(model, kind, blk, N):
    """one time / space block in place, on the fp32 path and (N >= 16, M >= 128) the tensor-core path: each path within the
    first-order bound of its kernel chain and within the measured bar; the two paths agree within the sum of their bounds"""
    m, sd64 = model
    M = N * _S
    g = torch.Generator().manual_seed(N * 10 + kind * 7 + blk)
    x0 = torch.randn((M, _HID), generator=g) * 2
    x0[::5] += 30.0
    p = f"updateformer.{'space' if kind else 'time'}_blocks.{blk}."
    G, L, gs, ls = (N, _S, _S, 1) if kind == 0 else (_S, N, 1, _S)
    outs = {}
    for tc in ((0, 1) if N >= 16 else (0,)):
        xb, xg = _guarded(x0)
        xin = xg.clone()
        native.check(native.lib().sampt_test_cotracker_block(_h(m), c_int(kind), c_int(blk), c_int(tc), native.ptr(xb), c_int(N),
                                                             native.stream_ptr()), "test_cotracker_block")
        torch.cuda.synchronize()
        assert (xb[M * _HID:] == 1e30).all(), "a value past x was written"
        ref, tol = _block64(sd64, p, xin, G, L, gs, ls, tc)
        err = (xg.double() - ref).abs()
        _report(f"block {p} N={N} tc={tc}", err, tol + 1e-45)
        rel = err.max().item() / ref.abs().max().item()
        print(f"block {p} N={N} tc={tc}: max err / max |x| = {rel:.3g} (bar {_BLOCK_BAR:.3g})")
        assert rel <= _BLOCK_BAR, (p, N, tc, rel)
        outs[tc] = (xg.double().clone(), tol)
    if len(outs) == 2:
        _report(f"block {p} N={N} tc vs fp32", (outs[1][0] - outs[0][0]).abs(), outs[0][1] + outs[1][1] + 1e-45)


def test_block_tc_needs_w16(model):
    m = model[0]
    ctx = m.native_context()
    name = "cot.updateformer.time_blocks.0.attn.qkv.w16"
    saved = ctx._tensors[name]
    native.check(native.lib().sampt_unset_tensors(ctx.handle, name.encode()), "unset")
    x = torch.zeros((16 * _S, _HID), device="cuda")
    try:
        rc = native.lib().sampt_test_cotracker_block(ctx.handle, c_int(0), c_int(0), c_int(1), native.ptr(x), c_int(16),
                                                     native.stream_ptr())
        assert rc != 0 and b".w16" in native.lib().sampt_last_error()
    finally:
        ctx.set_tensor(name, saved)


# ======================================================================================================= update and visibility
@pytest.mark.parametrize("N", _NS)
def test_update_and_vis(model, N):
    """GroupNorm(1,128) (block sums of 128 threads: n = 8) -> Linear 128x128 (fma chain from the bias, n = 129) -> GELU(erf)
    (slope <= 1.13, 2 u) added to ffeats; coords += dxy on every slot (CoTracker does not lock slot 0); then the visibility
    head w . ffeat + b (fma chain, n = 129) of the kernel's own updated features"""
    m, sd64 = model
    M = N * _S
    g = torch.Generator().manual_seed(N + 5)
    delta = torch.randn((M, 130), generator=g)
    delta[:, :2] *= 50.0
    delta[:, 2:] += torch.randn((M, 1), generator=g) * 300                     # large common offsets: GroupNorm conditioning
    ffeats = torch.randn((N, _S, 128), generator=g).cuda()
    coords = (torch.rand((N, _S, 2), generator=g) * 200 - 50).cuda()
    db, dg = _guarded(delta)
    f0, c0 = ffeats.clone(), coords.clone()
    vbuf, vis = _nan_out((N, _S), _S)
    native.check(native.lib().sampt_test_cotracker_update(_h(m), native.ptr(db), native.ptr(coords), native.ptr(ffeats), c_int(N),
                                                          native.ptr(vbuf), native.stream_ptr()), "test_cotracker_update")
    _guard_ok(vbuf, vis.numel())
    assert torch.equal(coords, c0 + dg[:, :2].view(N, _S, 2)), "coords += delta on every slot"
    v = dg[:, 2:].double()
    mu = v.mean(-1, keepdim=True)
    dv = v - mu
    var = (dv ** 2).mean(-1, keepdim=True)
    rstd = 1 / torch.sqrt(var + 1e-5)
    gw, gb = sd64["norm.weight"], sd64["norm.bias"]
    gn = dv * rstd * gw + gb
    m_err = _gamma(8) * v.abs().mean(-1, keepdim=True) + _U * mu.abs()
    rel = 0.5 * (_gamma(9) * var + 2 * m_err * dv.abs().mean(-1, keepdim=True) + m_err ** 2) / (var + 1e-5) + 3 * _U
    e_gn = (rstd * (m_err + _U * dv.abs()) + dv.abs() * rstd * rel) * gw.abs() + 3 * _U * (dv.abs() * rstd * gw.abs() + gb.abs())
    W, b = sd64["ffeat_updater.0.weight"], sd64["ffeat_updater.0.bias"]
    acc = gn @ W.T + b
    e_acc = _gamma(129) * (gn.abs() @ W.abs().T + b.abs()) + e_gn @ W.abs().T
    up = F.gelu(acc)
    ref = f0.double().view(M, 128) + up
    tol = 1.13 * e_acc + 2 * _U * up.abs() + _U * ref.abs() + 1e-45
    _report(f"update ffeats N={N}", (ffeats.double().view(M, 128) - ref).abs(), tol)
    vw, vb = sd64["vis_predictor.0.weight"][0], sd64["vis_predictor.0.bias"]
    ff = ffeats.double().view(M, 128)
    vref = ff @ vw + vb
    _report(f"visibility N={N}", (vis.double().view(M) - vref).abs(), _gamma(129) * (ff.abs() @ vw.abs() + vb.abs()) + 1e-45)


# ======================================================================================================= window and tracker
# Whole-chain bars (trajectories in image px): 4x the largest error the fp32 UpdateFormer path (SAMPT_COT_TC=0) showed against
# the float64 oracle on an H100 80GB HBM3 (700 W), never above 1e-3 px.  Measured (fp32 path / tensor-core path, N = 16, 84, 292;
# N = 15, M = 120, always runs the fp32 path and gave 1.52e-5 px and 5.9e-5 px):
#   window, 1 iteration:  coords 1.53e-5 / 1.53e-5 px, visibility logits 8.7e-7 / 2.0e-6
#   window, 6 iterations: coords 1.26e-4 / 1.26e-4 px, visibility logits 3.39e-3 / 3.38e-3
#   tracker, 84 points, 21 frames: trajectories 9.4e-4 / 7.2e-4 px, sigmoid visibilities 2.0e-3 / 2.2e-3
# The tracker's bar is the 1e-3 px cap, not 4x its measured error: the cap binds, leaving 6 % headroom over the fp32 path's
# 9.4e-4 px and 28 % over the tensor-core path that runs by default.  The tensor-core path, which the window takes at M >= 128,
# must meet the same bars.
_WINDOW_BAR = {1: 6e-5, 6: 5e-4}
_WINDOW_VIS_BAR = {1: 3.5e-6, 6: 1.35e-2}
_TRACK_BAR = 1e-3
_TRACK_VIS_BAR = 8e-3


def _features(m, T, seed):
    clip = synth.make_clip(T, 384, 512, seed=seed)
    m.fnet_on_tensor_cores = False
    fm = torch.cat([m.fnet_frames(clip["frames"][i:i + 8].float().cuda()) for i in range(0, T, 8)])
    return clip, fm


@pytest.mark.parametrize("N", [15, 16, 84, 292])
@pytest.mark.parametrize("iters", [1, 6])
def test_window_vs_float64(model, N, iters):
    """sampt_cotracker_window against forward_iteration in float64 on the same encoder features"""
    m, sd64 = model
    _, fm = _features(m, _S, seed=N)
    pyr = m.build_pyramid(fm)
    g = torch.Generator().manual_seed(N + iters)
    c0 = torch.rand((N, 2), generator=g) * torch.tensor([_W4 - 1.0, _H4 - 1.0])
    coords = c0[:, None].repeat(1, _S, 1).cuda().contiguous()
    fmn = fm.permute(0, 3, 1, 2)
    ff0 = pips_ref.bilinear_sample2d(fmn[0:1], coords[None, :, 0, 0], coords[None, :, 0, 1]).permute(0, 2, 1)[0]      # (N, 128)
    ffeats = ff0[:, None].repeat(1, _S, 1).contiguous()
    tm = torch.ones((N, _S), device="cuda")
    tm[: N // 3, 5:] = 0.0
    vi = torch.full((N, _S), 10.0, device="cuda")
    fidx = torch.tensor([0, 0] + list(range(_S)), dtype=torch.int32, device="cuda")
    co_in, ff_in = coords.clone(), ffeats.clone()
    vis = torch.empty((N, _S), device="cuda")
    native.check(native.lib().sampt_cotracker_window(
        _h(m), native.ptr(pyr[0]), native.ptr(pyr[1]), native.ptr(pyr[2]), native.ptr(pyr[3]), c_int(_H4), c_int(_W4), native.ptr(fidx),
        native.ptr(coords), native.ptr(ffeats), native.ptr(tm), native.ptr(vi), native.ptr(m._time_emb), c_int(N), c_int(iters),
        c_int(6), c_int(6), native.ptr(vis), native.stream_ptr()), "cotracker_window")
    torch.cuda.synchronize()
    preds, v64 = R.forward_iteration(sd64, fmn.double()[None], co_in.double().permute(1, 0, 2)[None], ff_in.double().permute(1, 0, 2)[None],
                                     vi.double().t()[None, :, :, None], tm.bool().t()[None, :, :, None], iters=iters)
    err = (coords.double() * 4.0 - preds[-1][0].permute(1, 0, 2)).abs().max().item()
    verr = (vis.double() - v64[0].t()).abs().max().item()
    print(f"window N={N} iters={iters} (M={8 * N}): max |coords - float64| = {err:.3g} px, max |vis logit - float64| = {verr:.3g}")
    assert err <= _WINDOW_BAR[iters] and verr <= _WINDOW_VIS_BAR[iters]


@pytest.mark.parametrize("reverse", [False, True])
def test_track_vs_float64(model, reverse):
    """CoTracker.track at the C3 count (84 points) over 21 frames: births at frames 0, 5, 12 and 13, so a window grows the active
    set while carried-over state exists; the last window is partial.  Identity and reversed frame order."""
    m, sd64 = model
    T, N = 21, 84
    clip, fm = _features(m, T, seed=77)
    pyr = m.build_pyramid(fm)
    q = synth.make_query_points(clip, N, seed=3)[0].clone()
    q[:, 0] = torch.tensor([0.0, 5.0, 12.0, 13.0]).repeat(N // 4)
    order = list(range(T))[::-1] if reverse else list(range(T))
    traj, vis = m.track(pyr, q.cuda(), order, iters=6)
    torch.cuda.synchronize()
    fmn = fm.permute(0, 3, 1, 2)[order].double()
    rgbs = torch.zeros((1, T, 3, 4, 4), dtype=torch.float64, device="cuda")
    t64, v64 = R.cotracker_forward(sd64, rgbs, q.cuda().double()[None], iters=6, fmaps_all=fmn)
    err = (traj.double() - t64[0]).abs().max().item()
    verr = (vis.double() - v64[0]).abs().max().item()
    print(f"track N={N} T={T} reverse={reverse}: max |traj - float64| = {err:.3g} px, max |vis - float64| = {verr:.3g}")
    assert err <= _TRACK_BAR and verr <= _TRACK_VIS_BAR
