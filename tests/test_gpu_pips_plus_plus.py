"""GPU: the PIPS++ tracker (csrc/pips_plus_plus.cu) kernel by kernel against float64 through the sampt_test_pips_plus_plus_*
entries of include/sampt_b200.h, then the window chain and the tracker against the CPU oracle (oracle/pips_plus_plus_ref.py).

Single kernels: bounds from fp32 rounding, u = 2^-24, and the summation length n (gamma_n = n u / (1 - n u)); tensor-core
convolutions add the 2^-22 relative error of a product of fp16 hi|lo operands (three passes, DESIGN §5).  Outputs start as NaN
with a guard tail that must stay NaN.
Each residual block: a bound propagated through the block in float64 (_bounded_conv, _bounded_norm_relu): every split-precision
product carries at most 3 * 2^-22 of |a||w| plus 2^-25 |w| (an activation lo half that is an fp16 subnormal), the fp32 sum
gamma_K of the sum of |products| (K = 3 Cin), and the instance norm passes its input's error on scaled by rstd, plus the error of
its own statistics.
Chains, where such worst-case bounds compound past usefulness: the GPU's error against float64 is held to a multiple of the CPU
float32 oracle's own error against float64 plus 2^-20 of the largest value, and the ratio is printed.  The 16-iteration window:
16x (measured 2.9-4.1x on one H100).  The DeltaBlock alone, nine GEMM-bearing stages from one set of rows: 32x (measured
18.5-18.7x); its CPU float32 error is a few u of the output, the three-pass split products carry up to 4u each."""
import math
from ctypes import c_char_p, c_int

import pytest
import torch

from oracle import pips_plus_plus_ref as ref
from sampt_b200 import native, synth

pytestmark = pytest.mark.gpu

_U = 2.0 ** -24
_H8, _W8 = 16, 20          # 128 x 160 frames at stride 8
CHAIN_MULT = 16.0
DELTA_BLOCK_MULT = 32.0
_PROD = 3 * 2.0 ** -22      # relative error of one three-pass split product
_SUBN = 2.0 ** -25          # absolute error of an activation lo half that is an fp16 subnormal


def _gamma(n):
    return n * _U / (1 - n * _U)


def _report(what, err, bound):
    worst = (err / bound).max().item()
    print(f"{what}: max err {err.max().item():.3g}, worst err / bound {worst:.3g}")
    assert worst <= 1.0, (what, worst)


def _nan_out(shape, guard=64, dtype=torch.float32):
    n = math.prod(shape)
    buf = torch.full((n + guard,), float("nan"), device="cuda", dtype=dtype)
    return buf, buf[:n].view(shape)


def _guard_ok(buf, n):
    torch.cuda.synchronize()
    assert torch.isnan(buf[n:].float()).all(), "a value past the output was written"


@pytest.fixture(scope="module")
def model():
    from sam_pt.point_tracker.pips_plus_plus import PipsPlusPlus
    sd = synth.make_pips_plus_plus_state_dict()
    m = PipsPlusPlus(stride=8)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    return m, sd


def _pyramid(m, fm):
    """fm (S,H8,W8,128) cuda -> the 4 channels-last levels"""
    S, H8, W8, _ = fm.shape
    pyr = [fm.contiguous()] + [torch.empty((S, H8 >> l, W8 >> l, 128), device="cuda") for l in range(1, 4)]
    ctx = m.native_context()
    native.check(native.lib().sampt_pips_pyramid(ctx.handle, native.ptr(pyr[0]), c_int(S), c_int(H8), c_int(W8), native.ptr(pyr[1]),
                                                 native.ptr(pyr[2]), native.ptr(pyr[3]), native.stream_ptr()), "pyramid")
    return pyr


def _coords(S, N, gen):
    """(S,N,2) feature-map px: random inside, integral, on the border, one pixel outside and far outside"""
    c = torch.rand((S, N, 2), generator=gen, dtype=torch.float64) * torch.tensor([_W8 - 1, _H8 - 1], dtype=torch.float64)
    special = torch.tensor([[3.0, 4.0], [0.0, 0.0], [_W8 - 1.0, _H8 - 1.0], [-1.0, 5.5], [_W8 + 0.5, -1.0], [40.0, -30.0],
                            [7.5, 8.5]], dtype=torch.float64)
    for n in range(min(N, special.shape[0])):
        c[:, n] = special[n] + 0.25 * torch.arange(S, dtype=torch.float64)[:, None] * (n % 2)
    return c.float()


# ============================================================================================================== row kernel
@pytest.mark.parametrize("N,S", [(1, 2), (8, 8), (64, 8), (8, 50), (1, 128), (8, 128), (64, 50)])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_row(model, N, S, mode):
    m, _ = model
    gen = torch.Generator().manual_seed(100 * N + S + mode)
    fm = torch.randn((S, _H8, _W8, 128), generator=gen)
    pyr = _pyramid(m, fm.cuda())
    coords = _coords(S, N, gen)
    feats = torch.randn((3, S, N, 128), generator=gen)
    feats_d = feats.cuda().contiguous()
    M = N * S
    rbuf, row = _nan_out((M, 718))
    abuf, A = _nan_out((M, 2 * 2176), dtype=torch.float16)
    ctx = m.native_context()
    native.check(native.lib().sampt_test_pips_plus_plus_row(
        ctx.handle, *[native.ptr(p) for p in pyr], c_int(_H8), c_int(_W8), native.ptr(coords.cuda().contiguous()), native.ptr(feats_d),
        c_int(N), c_int(S), c_int(mode), native.ptr(row), native.ptr(A), native.stream_ptr()), "row")
    _guard_ok(rbuf, M * 718)
    _guard_ok(abuf, M * 2 * 2176)
    # float64 reference from the fp32 operands
    fm64 = fm.double().permute(0, 3, 1, 2)[None]
    c64 = coords.double()[None]
    pyr64 = ref.build_pyramid(fm64)
    f = feats.double()[:, None]
    if mode == 1:
        t = ref.sample_targets(fm64, c64, torch.zeros(S, dtype=torch.long))
        f1 = f2 = f4 = t
    elif mode == 2:
        f1 = f[0]
        f2 = ref.sample_targets(fm64, c64, (torch.arange(S) - 2).clip(min=0))
        f4 = ref.sample_targets(fm64, c64, (torch.arange(S) - 4).clip(min=0))
    else:
        f1, f2, f4 = f[0], f[1], f[2]
    want = ref.input_rows(pyr64, f1, f2, f4, c64).reshape(M, 718)
    got = row.double().cpu()
    # targets written back
    fgot = feats_d.double().cpu()
    for b, t in enumerate((f1, f2, f4)):
        terr = (fgot[b] - t[0]).abs()
        _report(f"row N={N} S={S} mode={mode} target {b}", terr, torch.full_like(terr, 8 * _U * fm.abs().max().item()))
    # correlation columns: 128-term dot products of the targets with the 4 neighbours of each sample, blended
    tmax = torch.stack([t[0] for t in (f1, f2, f4)]).abs().sum(-1).max().item()
    corr_bound = (_gamma(140) + 16 * _U * _W8) * tmax * fm.abs().max().item() / math.sqrt(128) * 4
    _report(f"row N={N} S={S} mode={mode} corr", (got[:, :588] - want[:, :588]).abs(), torch.full((M, 588), corr_bound, dtype=torch.float64))
    # flow columns: exact fp32 differences of the coords
    flow = coords[1:] - coords[:-1]
    flow = torch.cat([flow, flow[-1:]]).permute(1, 0, 2).reshape(M, 2)
    assert torch.equal(row[:, 716:].cpu(), flow)
    # posemb columns within ulps of torch's float32 sin / cos of the same flow
    pe = ref.posemb_sincos_2d_xy(flow.reshape(N, S, 2))[..., :128].reshape(M, 128)
    _report(f"row N={N} S={S} mode={mode} posemb", (got[:, 588:716] - pe.double()).abs(), torch.full((M, 128), 4 * 2.0 ** -23))
    # A operand: hi + lo of the row at tap k of row (n, s+1-k); zero taps at each point's window ends and in the K padding
    Ad = A.double().cpu().reshape(N, S, 2, 2176)
    val = Ad[:, :, 0] + Ad[:, :, 1]
    r3 = got.reshape(N, S, 718)
    for k in range(3):
        src = torch.zeros_like(r3)
        lo, hi = max(0, 1 - k), min(S, S + 1 - k)
        src[:, lo:hi] = r3[:, lo + k - 1:hi + k - 1]
        err = (val[:, :, k * 718:(k + 1) * 718] - src).abs()
        _report(f"row N={N} S={S} mode={mode} A tap {k}", err, src.abs() * 2.0 ** -21 + 2.0 ** -24)
    assert (val[:, :, 2154:] == 0).all()


# ============================================================================================================== single stages
def _oracle_sd(sd, dt):
    return {k: v.to(dt) for k, v in sd.items()}


@pytest.mark.parametrize("name,cin,cout,pre", [("first_block_conv", 718, 128, 0), ("basicblock_list.0.conv1", 128, 128, 1),
                                               ("basicblock_list.2.conv1", 128, 256, 2), ("basicblock_list.6.conv2", 1024, 1024, 2)])
@pytest.mark.parametrize("N,S", [(1, 2), (8, 8), (3, 128)])
def test_tconv(model, name, cin, cout, pre, N, S):
    m, sd = model
    gen = torch.Generator().manual_seed(cin + cout + S)
    x = torch.randn((N, S, cin), generator=gen) * 3 + 0.5
    M = N * S
    obuf, out = _nan_out((M, cout))
    ctx = m.native_context()
    native.check(native.lib().sampt_test_pips_plus_plus_tconv(ctx.handle, c_char_p(name.encode()), native.ptr(x.cuda().contiguous()),
                                                              c_int(N), c_int(S), c_int(cin), c_int(cout), c_int(pre), native.ptr(out),
                                                              native.stream_ptr()), "tconv")
    _guard_ok(obuf, M * cout)
    s64 = _oracle_sd(sd, torch.float64)
    xi = x.double().permute(0, 2, 1)
    if pre == 2:
        xi = torch.relu(ref._inorm1d(xi))
    elif pre == 1:
        xi = torch.relu(xi)
    want = ref._conv1d(s64, "delta_block." + name, xi).permute(0, 2, 1).reshape(M, cout)
    w = s64[f"delta_block.{name}.conv.weight"].abs()
    mag = torch.nn.functional.conv1d(torch.nn.functional.pad(xi.abs(), (1, 1)), w).permute(0, 2, 1).reshape(M, cout)
    rel = _gamma(3 * cin) + 2.0 ** -21 + (2.0 ** -19 if pre == 2 else 0.0)
    _report(f"tconv {name} N={N} S={S}", (out.double().cpu() - want).abs(), rel * mag + 2.0 ** -30)


@pytest.mark.parametrize("N,S,C,offset", [(1, 2, 128, 0.0), (8, 8, 256, 1e3), (3, 128, 1024, 10.0), (64, 50, 128, 1e4)])
def test_inorm(model, N, S, C, offset):
    m, _ = model
    gen = torch.Generator().manual_seed(S * C)
    x = torch.randn((N, S, C), generator=gen) + offset
    sbuf, stats = _nan_out((N, C, 2))
    native.check(native.lib().sampt_test_pips_plus_plus_inorm(m.native_context().handle, native.ptr(x.cuda().contiguous()), c_int(N),
                                                              c_int(S), c_int(C), native.ptr(stats), native.stream_ptr()), "inorm")
    _guard_ok(sbuf, N * C * 2)
    x64 = x.double()
    mean = x64.mean(1)
    var = x64.var(1, unbiased=False)
    got = stats.double().cpu()
    _report(f"inorm mean N={N} S={S} C={C}", (got[..., 0] - mean).abs(), _gamma(S + 1) * x64.abs().max(1).values + 1e-30)
    # two passes: a mean error d adds S d^2 to the sum of squares, the sum itself carries gamma_(S+2) of it
    rstd = 1 / torch.sqrt(var + 1e-5)
    d = _gamma(S + 1) * x64.abs().max(1).values
    _report(f"inorm rstd N={N} S={S} C={C}", (got[..., 1] - rstd).abs(), rstd * (_gamma(2 * S + 8) + d ** 2 / (var + 1e-5)))


def _chain_check(what, got, want64, want32, mult=CHAIN_MULT):
    e_gpu = (got.double() - want64).abs().max().item()
    e_cpu = (want32.double() - want64).abs().max().item()
    bound = mult * e_cpu + 2.0 ** -20 * want64.abs().max().item()
    print(f"{what}: GPU err {e_gpu:.3g}, CPU fp32 err {e_cpu:.3g}, GPU / CPU {e_gpu / max(e_cpu, 1e-300):.3g}, "
          f"err / bound {e_gpu / bound:.3g}")
    assert e_gpu <= bound, what


def _conv_abs(s64, name, a):
    return torch.nn.functional.conv1d(torch.nn.functional.pad(a, (1, 1)), s64[name + ".conv.weight"].abs())


def _bounded_conv(s64, name, x, ex):
    """Conv1dPad `name` on the float64 x (B,C,S) whose GPU counterpart is off by at most ex -> (y, bound on the GPU's y)"""
    y = ref._conv1d(s64, name, x)
    K = s64[name + ".conv.weight"].shape[1] * 3
    ey = ((_gamma(K) + _PROD) * _conv_abs(s64, name, x.abs()) + _SUBN * _conv_abs(s64, name, torch.ones_like(x))
          + _conv_abs(s64, name, ex) + _U * y.abs())
    return y, ey


def _bounded_norm_relu(x, ex):
    """ReLU(InstanceNorm1d(x)) over the last axis with its error bound: the input error through (x - mean) * rstd (the mean moves
    by at most max ex, the variance by 2 mean(|x - mean| (ex + max ex)) + (ex + max ex)^2), plus the two-pass statistics' own
    rounding; x2 for the linearisation of rstd"""
    S = x.shape[-1]
    m = x.mean(-1, keepdim=True)
    d = x - m
    var = (d * d).mean(-1, keepdim=True)
    r = 1 / torch.sqrt(var + 1e-5)
    xn = d * r
    emax = ex.amax(-1, keepdim=True)
    dvar = 2 * (d.abs() * (ex + emax)).mean(-1, keepdim=True) + ((ex + emax) ** 2).mean(-1, keepdim=True) \
        + _gamma(2 * S + 8) * var + (_gamma(S + 1) * x.abs().amax(-1, keepdim=True)) ** 2
    e = 2 * (r * (ex + emax) + xn.abs() * dvar / (var + 1e-5) + _gamma(2 * S + 8) * xn.abs())
    return torch.relu(xn), e


def _bounded_block(s64, i, x, ex):
    ci, co = ref.BLOCK_CHANNELS[i]
    p = f"delta_block.basicblock_list.{i}."
    xin, exin = (torch.relu(x), ex) if i == 0 else _bounded_norm_relu(x, ex)
    y, ey = _bounded_conv(s64, p + "conv1", xin, exin)
    z, ez = _bounded_norm_relu(y, ey)
    out, eout = _bounded_conv(s64, p + "conv2", z, ez)
    idt, eid = (torch.relu(x), ex) if i == 0 else (x, ex)
    if co != ci:
        ch1 = (co - ci) // 2
        idt, eid = (torch.nn.functional.pad(t, (0, 0, ch1, co - ci - ch1)) for t in (idt, eid))
    out = out + idt
    return out, eout + eid + _U * out.abs()


@pytest.mark.parametrize("block", list(range(8)) + [-1])
@pytest.mark.parametrize("N,S", [(2, 8), (4, 128)])
def test_residual_and_delta_block(model, block, N, S):
    m, sd = model
    gen = torch.Generator().manual_seed(block + 10 + S)
    cin = 718 if block < 0 else ref.BLOCK_CHANNELS[block][0]
    cout = 2 if block < 0 else ref.BLOCK_CHANNELS[block][1]
    x = torch.randn((N, S, cin), generator=gen)
    if block == 0:
        x = torch.relu(x)
    M = N * S
    obuf, out = _nan_out((M, cout))
    x_d = x.cuda().contiguous()
    native.check(native.lib().sampt_test_pips_plus_plus_residual(m.native_context().handle, c_int(block), native.ptr(x_d), c_int(N),
                                                                 c_int(S), native.ptr(out), native.stream_ptr()), "residual")
    _guard_ok(obuf, M * cout)
    s64 = _oracle_sd(sd, torch.float64)
    if block < 0:
        _chain_check(f"DeltaBlock N={N} S={S}", out.cpu(), ref.delta_block_rows(s64, x.double()).reshape(M, 2),
                     ref.delta_block_rows(_oracle_sd(sd, torch.float32), x).reshape(M, 2), DELTA_BLOCK_MULT)
        return
    h = x.double().permute(0, 2, 1)
    want, bound = (t.permute(0, 2, 1).reshape(M, cout) for t in _bounded_block(s64, block, h, torch.zeros_like(h)))
    _report(f"residual block {block} N={N} S={S}", (out.double().cpu() - want).abs(), bound)


def test_update(model):
    m, _ = model
    gen = torch.Generator().manual_seed(3)
    N, S = 7, 9
    coords = torch.randn((S, N, 2), generator=gen) * 10
    lock = torch.randn((N, 2), generator=gen)
    delta = torch.randn((N, S, 2), generator=gen)
    c_d, lock_d, delta_d = coords.cuda().contiguous(), lock.cuda().contiguous(), delta.cuda().contiguous()
    pbuf, pre = _nan_out((S, N, 2))
    native.check(native.lib().sampt_test_pips_plus_plus_update(m.native_context().handle, native.ptr(c_d), native.ptr(lock_d),
                                                               native.ptr(delta_d), c_int(N), c_int(S), c_int(8), native.ptr(pre),
                                                               native.stream_ptr()), "update")
    _guard_ok(pbuf, S * N * 2)
    new = coords + delta.permute(1, 0, 2)
    assert torch.equal(pre.cpu(), new * 8)
    new[0] = lock
    assert torch.equal(c_d.cpu(), new)


# ============================================================================================================== window chain
def test_window_16_iterations(model):
    m, sd = model
    S, N = 8, 8
    clip = synth.make_clip(S, 128, 160, seed=81)
    q = synth.make_query_points(clip, N, seed=81)[0, :, 1:]
    tr = q[None, None].repeat(1, S, 1, 1)
    rgbs = clip["frames"][None]
    p1, p2, feats, _ = m(tr.cuda(), rgbs.cuda(), iters=16)
    # the oracle runs on the GPU encoder's features so that the chain alone is compared
    fm = m.encode_frames(rgbs[0].cuda())[0].permute(0, 3, 1, 2)[None].cpu()
    r64 = ref.pips_plus_plus_forward(_oracle_sd(sd, torch.float64), tr.double(), None, 16, fmaps=fm.double())
    r32 = ref.pips_plus_plus_forward(_oracle_sd(sd, torch.float32), tr.float(), None, 16, fmaps=fm.float())
    for i in (0, 7, 15, 16):
        _chain_check(f"window coords iteration {i}", p1[i].cpu(), r64[0][i], r32[0][i])
    _chain_check("window feats2", feats[1].cpu(), r64[2][1], r32[2][1])
    assert len(p1) == 17 and len(p2) == 18
    assert torch.equal(p2[0].cpu(), tr) and torch.equal(p2[3][:, 0].cpu(), tr[:, 0])


def test_window_matches_reference_golden(model, golden_dir):
    import os
    m, sd = model
    g = torch.load(os.path.join(golden_dir, "pips_plus_plus_golden.pt"))
    for key in ("window_S8", "window_S128"):
        cfg = g[key]["cfg"]
        clip = synth.make_clip(cfg["S"], 128, 160, seed=cfg["seed"])
        q = synth.make_query_points(clip, cfg["N"], seed=cfg["seed"])[0, :, 1:]
        tr = q[None, None].repeat(1, cfg["S"], 1, 1)
        p1, _, feats, _ = m(tr.cuda(), clip["frames"][None].float().cuda(), iters=cfg["iters"])
        err = (torch.stack(p1)[:, 0].cpu() - g[key]["preds1"]).abs().max().item()
        ferr = (torch.stack(feats)[:, 0].cpu() - g[key]["feats"]).abs().max().item()
        print(f"{key}: GPU vs reference golden: coords {err:.3g} px, feats {ferr:.3g}")
        assert err < 1e-3 and ferr < 1e-3


# ============================================================================================================== tracker
def test_tracker_140_frames_mixed_timesteps(model):
    from sam_pt.point_tracker.pips_plus_plus import PipsPlusPlusPointTracker
    m, sd = model
    T = 140
    clip = synth.make_clip(T, 128, 160, seed=82)
    q = torch.cat([synth.make_query_points(clip, 2, seed=82, t=t) for t in (0, 70, 139)], dim=1)
    trk = PipsPlusPlusPointTracker(checkpoint_path=None, stride=8, max_sequence_length=128, iters=4, image_size=None)
    trk.model.load_state_dict(sd)
    traj, vis = trk(clip["frames"][None].cuda(), q.cuda())
    want, _ = ref.pips_plus_plus_tracker_forward(_oracle_sd(sd, torch.float32), clip["frames"][None].float(), q, iters=4)
    err = (traj.cpu() - want).abs().max().item()
    print(f"tracker 140 frames, query frames 0 / 70 / 139: max |dcoord| {err:.3g} px")
    assert traj.shape == (1, T, 6, 2) and err < 1e-3
    assert torch.equal(traj[0, 139, 4:].cpu(), q[0, 4:, 1:]) and bool((vis == 1).all())


def test_alternating_with_pips_is_bitwise_stable(model):
    from oracle import pips_ref
    from sam_pt.point_tracker.pips import Pips
    m, _ = model
    p = Pips(S=8, stride=4)
    p.load_state_dict(synth.condition_pips(synth.make_state_dict(pips_ref.pips_state_dict_shapes(), 7201)))
    p = p.cuda().eval()
    clip = synth.make_clip(8, 128, 160, seed=83)
    rgbs = clip["frames"][None].cuda()
    q = synth.make_query_points(clip, 4, seed=83)[:, :, 1:].cuda()
    tr = q[:, None].repeat(1, 8, 1, 1)

    def run_pips():
        return p(q, rgbs, iters=6)[0][-1].clone()

    def run_ppp():
        return m(tr, rgbs, iters=4)[0][-1].clone()
    a1, b1 = run_pips(), run_ppp()
    a2, b2, a3 = run_pips(), run_ppp(), run_pips()
    assert torch.equal(a1, a2) and torch.equal(a1, a3) and torch.equal(b1, b2)


def test_window_feat_init_matches_reference_golden(model, golden_dir):
    """sampt_pips_plus_plus_window with feat_init (the targets of an earlier window, used as all three at iteration 0)"""
    import os
    m, _ = model
    g = torch.load(os.path.join(golden_dir, "pips_plus_plus_golden.pt"))["window_S8"]
    cfg = g["cfg"]
    clip = synth.make_clip(cfg["S"], 128, 160, seed=cfg["seed"])
    q = synth.make_query_points(clip, cfg["N"], seed=cfg["seed"])[0, :, 1:]
    tr = q[None, None].repeat(1, cfg["S"], 1, 1) + 1.5
    fi = tuple(g["feats"][b][None].cuda() for b in range(3))
    p1, _, feats, _ = m(tr.cuda(), clip["frames"][None].float().cuda(), iters=4, feat_init=fi)
    err = (torch.stack(p1)[:, 0].cpu() - g["feat_init_preds1"]).abs().max().item()
    ferr = (torch.stack(feats)[:, 0].cpu() - g["feat_init_feats"]).abs().max().item()
    print(f"window with feat_init: GPU vs reference golden: coords {err:.3g} px, feats {ferr:.3g}")
    assert err < 1e-3 and ferr < 1e-3


@pytest.mark.parametrize("float_frames", [False, True])
def test_tracker_image_size_and_float_frames(model, float_frames):
    """The image_size path (resize of rgbs/255, x scaled by image_size[0]/H and y by image_size[1]/W in place, and back), on
    uint8 frames and on non-integer float frames, which are used as given, against the oracle"""
    from sam_pt.point_tracker.pips_plus_plus import PipsPlusPlusPointTracker
    m, sd = model
    clip = synth.make_clip(6, 128, 160, seed=84)
    frames = clip["frames"][None]
    if float_frames:
        frames = frames.float() + torch.rand(frames.shape, generator=torch.Generator().manual_seed(84)) * 0.9
    q = synth.make_query_points(clip, 3, seed=84)
    trk = PipsPlusPlusPointTracker(checkpoint_path=None, image_size=(160, 192), iters=3)
    trk.model.load_state_dict(sd)
    q_d = q.clone().cuda()
    traj, _ = trk(frames.cuda(), q_d)
    want, _ = ref.pips_plus_plus_tracker_forward(_oracle_sd(sd, torch.float32), frames.float(), q, iters=3, image_size=(160, 192))
    err = (traj.cpu() - want).abs().max().item()
    print(f"tracker image_size (float frames {float_frames}): max |dcoord| {err:.3g} px")
    assert err < 1e-3
    assert torch.equal(q_d[0, :, 1].cpu(), q[0, :, 1] * (160 / 128)) and torch.equal(q_d[0, :, 2].cpu(), q[0, :, 2] * (192 / 160))


def _c2_golden_mod():
    import importlib.util
    import os
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_golden_pips_plus_plus_c2.py")
    spec = importlib.util.spec_from_file_location("make_golden_pips_plus_plus_c2", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_sampt_vit_b_c2_16_frames(golden_dir):
    """SamPt (ViT-B + PIPS++, 12 refinements) on the first 16 frames of C2 (480x854, seed 72, 8 points) against the committed
    golden of the unmodified reference tracker and the SAM oracle chain (tests/golden/make_golden_pips_plus_plus_c2.py): the
    stride-8 encoder and the pyramid at 60x106 (levels 30x53, 15x26, 7x13); every frame within 1e-3 px, mask IoU >= 0.999."""
    import os

    import numpy as np
    from sampt_b200 import factory
    g = _c2_golden_mod()
    gold = dict(np.load(os.path.join(golden_dir, "pips_plus_plus_c2_16.npz")))
    sd = synth.make_pips_plus_plus_state_dict()
    vid = g.video()
    q_before = vid["query_points"].clone()
    model = factory.build_sam_pt("vit_b", g.sam_state_dict(), None, positive_points_per_mask=g.P, sam_iou_threshold=-1e9,
                                 iterative_refinement_iterations=g.REFINEMENTS, pips_plus_plus_state_dict=sd)
    # the tracker alone, against the reference tracker's own output
    frames = torch.stack(vid["image"]).cuda()
    ttraj, _ = model.point_tracker(frames[None], vid["query_points"].reshape(1, -1, 3).cuda())
    terr_trk = (ttraj[0].cpu() - torch.from_numpy(gold["tracker_traj"])).abs().amax(dim=(1, 2))
    out = model(vid)
    terr = (out["trajectories"].cpu() - torch.from_numpy(gold["traj"])).abs().amax(dim=(1, 2, 3))
    assert torch.equal(out["visibilities"].cpu(), torch.from_numpy(gold["vis"]))
    assert torch.equal(vid["query_points"], q_before)
    ref_masks = np.unpackbits(gold["masks"], axis=1)[:, :g.H * g.W].reshape(g.T, g.H, g.W).astype(bool)
    ious = []
    for f in range(g.T):
        a = (out["logits"][0][f] > 0).cpu().numpy()
        u = (a | ref_masks[f]).sum()
        ious.append(1.0 if u == 0 else float((a & ref_masks[f]).sum() / u))
    print(f"C2 16 frames ViT-B + PIPS++: tracker max |dcoord| {terr_trk.max().item():.2e} px, SamPt max |dcoord| "
          f"{terr.max().item():.2e} px, min IoU {min(ious):.5f}")
    assert (terr_trk <= 1e-3).all() and (terr <= 1e-3).all() and min(ious) >= 0.999, (terr, ious)
