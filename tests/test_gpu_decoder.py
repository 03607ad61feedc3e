"""GPU: the SAM prompt encoder and mask decoder (csrc/decoder.cu) stage by stage against float64, through the unit-test entries
of include/sampt_b200.h (sampt_test_sam_attention / _prompt / _upscale / _postprocess), then whole predict_torch calls against the
float64 oracle, then the bitwise invariants of the refinement chain and its CUDA graphs.

Kernel bounds are derived from fp32 rounding, u = 2^-24, and the sequential summation length n of the kernel under test
(gamma_n = n u / (1 - n u)).  Each group prints its worst error / bound."""
import math
from ctypes import c_int

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import sam_ref
from sampt_b200 import factory, native, synth

pytestmark = pytest.mark.gpu

_U = 2.0 ** -24
_G = 64                  # image-embedding grid of every SAM model (1024 / 16)
_NOUT = 5                # output tokens: iou + 4 mask tokens


def _gamma(n):
    return n * _U / (1 - n * _U)


def _report(what, err, bound):
    worst = (err / bound).max().item()
    print(f"{what}: max err {err.max().item():.3g}, worst err / bound {worst:.3g}")
    assert worst <= 1.0, (what, worst)


def _sd(seed=41, hq=False):
    return synth.condition_sam(synth.make_state_dict(sam_ref.sam_state_dict_shapes(sam_ref.VIT_TEST, hq=hq), seed))


@pytest.fixture(scope="module")
def model():
    sd = _sd()
    sam = factory.build_sam("vit_test", sd).cuda()
    return sam, sd, {k: v.double() for k, v in sd.items()}


def _ctx(sam):
    """the shared context with `sam`'s decoder weights registered (another model of the session may have replaced them)"""
    return sam.native_context()


# ======================================================================================================= attention cores
def _attn_inputs(Tq, Nk, dh, spread, seed, key_scale=None):
    """q [Tq, 8 dh], k/v [Nk, 8 dh] fp32; q scaled so that the largest |logit| of every head is `spread`"""
    g = torch.Generator().manual_seed(seed)
    q = torch.randn((Tq, 8 * dh), generator=g)
    k = torch.randn((Nk, 8 * dh), generator=g)
    v = torch.randn((Nk, 8 * dh), generator=g)
    if key_scale is not None:
        k = k * key_scale[:, None]
    s = torch.einsum("thd,jhd->htj", q.double().view(Tq, 8, dh), k.double().view(Nk, 8, dh)) / math.sqrt(dh)
    m = s.abs().amax(dim=(1, 2))                                   # per head
    q = (q.view(Tq, 8, dh) * (spread / m).float()[None, :, None]).reshape(Tq, 8 * dh)
    return q, k, v


def _attn_expected(q, k, v, dh, n, kind_terms):
    """float64 attention over the kernel's own fp32 operands and its bound (first order, x1.05 for the second-order rest):
    logit j carries E_j = u ((dh + 2) sum_d |q_d k_jd| / sqrt(dh)   dot product, q scaling, 1/sqrt(dh) rounding
                            + (m - s_j)                             rounding of the exponent's argument s_j - max
                            + kind_terms)                           expf ulps and kernel-specific rescalings
    and moves the output by <= sum_j P_j E_j |v_j| + (sum_j P_j E_j) (P |V|); the numerator and denominator sums of length n
    add 2 gamma_n P |V|; the final division u |o|."""
    Tq, Nk = q.shape[0], k.shape[0]
    Q = q.cuda().double().view(Tq, 8, dh).transpose(0, 1)
    K = k.cuda().double().view(Nk, 8, dh).transpose(0, 1)
    V = v.cuda().double().view(Nk, 8, dh).transpose(0, 1)
    S = Q @ K.transpose(1, 2) / math.sqrt(dh)
    M = Q.abs() @ K.abs().transpose(1, 2) / math.sqrt(dh)
    P = torch.softmax(S, dim=-1)
    O = P @ V
    PV = P @ V.abs()
    E = _U * ((dh + 2) * M + (S.amax(-1, keepdim=True) - S) + kind_terms)
    PE = P * E
    tol = 1.05 * (PE @ V.abs() + PE.sum(-1, keepdim=True) * PV) + 2 * _gamma(n) * PV + 3 * _U * O.abs() + 1e-30
    back = lambda t: t.transpose(0, 1).reshape(Tq, 8 * dh)
    return back(O), back(tol), S


def _run_attention(sam, kind, q, k, v, T, Nk, out_rows, width):
    """out (+ one guard row) starts as NaN: rows the kernel does not write stay NaN, and the guard row must stay NaN"""
    ctx = _ctx(sam)
    out = torch.full((out_rows + 1, width), float("nan"), device="cuda")
    native.check(native.lib().sampt_test_sam_attention(ctx.handle, c_int(kind), native.ptr(q), native.ptr(k), native.ptr(v),
                                                       native.ptr(out), c_int(T), c_int(Nk), native.stream_ptr()), "test_sam_attention")
    torch.cuda.synchronize()
    assert torch.isnan(out[out_rows]).all(), "a row past the output was written"
    return out[:out_rows]


def _with_guard(t):
    """t plus one row of huge values: a kernel that reads past the last row turns its output into garbage"""
    return torch.cat([t, torch.full((1, t.shape[1]), 1e30)]).cuda().contiguous()


@pytest.mark.parametrize("T", [1, 7, 8, 16, 17, 31, 32, 33, 64, 65, 263, 327])
def test_token_self_attention(model, T):
    """kind 0 (attn_q_small_kernel: each thread sums every 256th key, then a 5-level warp tree and 8 warps, n = ceil(T/256) + 13)
    and kind 1 (attn_tok_self_kernel: one lane sums all T keys in order, n = T + 1), at every T, against float64 and each other"""
    sam = model[0]
    q, k, v = _attn_inputs(T, T, 32, 30.0, seed=T)
    qg, kg, vg = _with_guard(q), _with_guard(k), _with_guard(v)
    outs = []
    for kind, n in ((0, math.ceil(T / 256) + 13), (1, T + 1)):
        exp, tol, _ = _attn_expected(q, k, v, 32, n, 4.0)
        out = _run_attention(sam, kind, qg, kg, vg, T, T, T, 256)
        assert torch.isfinite(out).all(), (kind, T)
        _report(f"self-attention kind {kind} T={T}", (out.double() - exp).abs(), tol)
        outs.append((out.double(), tol))
    (o0, t0), (o1, t1) = outs
    _report(f"self-attention kind 0 vs kind 1 T={T}", (o0 - o1).abs(), t0 + t1)


@pytest.mark.parametrize("T,N", [(7, 4096), (32, 4096), (33, 4096), (64, 4096), (65, 4096), (263, 4096), (327, 4096),
                                 (70, 4001), (33, 100)])
def test_image_to_token_attention(model, T, N):
    """attn_kv_small_kernel: one pass over the T tokens in chunks of 32 with an online softmax.  Each term passes through the
    later rescales corr = expf(m_old - m_new): their arguments add up to at most m - s_j (already in E_j) and each costs an
    expf and an fma rounding, <= 3 u per token, so kind_terms = 3 T + 4 and n = T.  The keys' scale grows along the tokens, so
    the running maximum of most queries first appears in a later chunk."""
    sam = model[0]
    key_scale = torch.linspace(0.3, 3.0, T)
    q, k, v = _attn_inputs(N, T, 16, 30.0, seed=1000 + T, key_scale=key_scale)
    exp, tol, S = _attn_expected(q, k, v, 16, T, 3.0 * T + 4)
    if T > 32:
        late = (S.argmax(-1) >= 32).double().mean().item()
        print(f"T={T} N={N}: {late:.2f} of the (query, head) pairs have their maximum after the first chunk")
        assert late > 0.05
    out = _run_attention(sam, 3, q.cuda(), k.cuda(), v.cuda(), T, N, N, 128)
    assert torch.isfinite(out).all()
    _report(f"image->token attention T={T} N={N}", (out.double() - exp).abs(), tol)


@pytest.mark.parametrize("Nk", [4096, 4000, 300])
@pytest.mark.parametrize("T", [7, 263])
def test_token_to_image_attention(model, T, Nk):
    """attn_t2i_partial_kernel + attn_t2i_combine_kernel: per split of 256 keys each lane sums 8 keys, then a 5-level warp tree;
    the combine sums the splits in order (n = 8 + 5 + nsplit + 1).  A key's weight is expf(s_j - m_split) expf(m_split - m): the
    two arguments add up to m - s_j, two expf ulps and a product rounding give kind_terms = 8.  The splits have very different
    scales (logit spread up to +-30, most of the mass in a few splits); query 0 is dominated by one key."""
    sam = model[0]
    nsplit = (Nk + 255) // 256
    g = torch.Generator().manual_seed(Nk + T)
    split_scale = torch.rand(nsplit, generator=g) * 2.5 + 0.1
    key_scale = split_scale.repeat_interleave(256)[:Nk]
    q, k, v = _attn_inputs(T, Nk, 16, 30.0, seed=2000 + T + Nk, key_scale=key_scale)
    j = Nk - 7                                                     # in the last (possibly partial) split
    u = F.normalize(torch.randn((8, 16), generator=g), dim=1)      # per head: q_0 = 4 u, k_j = 40 u -> logit 40, the rest ~N(0, 2.6)
    q[0] = (4.0 * u).flatten()
    k[j] = (40.0 * u).flatten()
    exp, tol, S = _attn_expected(q, k, v, 16, 8 + 5 + nsplit + 1, 8.0)
    P0 = torch.softmax(S[:, 0], dim=-1)
    assert (P0[:, j] > 0.99).all()                                 # query 0: one key holds the mass in every head
    out = _run_attention(sam, 2, q.cuda(), k.cuda(), v.cuda(), T, Nk, T, 128)
    assert torch.isfinite(out).all()
    _report(f"token->image attention T={T} Nk={Nk}", (out.double() - exp).abs(), tol)


# ======================================================================================================= prompt encoder
def _ln2d_bound(v, dv, w, b, eps):
    """LayerNorm2d over dim 1 + affine, first order: (z exact, bound).  mean and var are sums of C terms; rstd = 1/sqrtf(var +
    eps) is 3 roundings; (v - mean) rstd and the fma with the affine weight 2 more"""
    C = v.shape[1]
    sh = (1, C) + (1,) * (v.dim() - 2)
    mean = v.mean(1, keepdim=True)
    d = v - mean
    var = (d * d).mean(1, keepdim=True)
    r = 1.0 / torch.sqrt(var + eps)
    dmean = dv.mean(1, keepdim=True) + _gamma(C) * v.abs().mean(1, keepdim=True)
    dd = dv + dmean + _U * d.abs()
    dvar = 2 * (d.abs() * dd).mean(1, keepdim=True) + _gamma(C + 1) * var
    dr = r * (0.5 * dvar / (var + eps) + 3 * _U)
    y = d * r
    dy = r * dd + d.abs() * dr + _U * y.abs()
    z = w.view(sh) * y + b.view(sh)
    return z, w.abs().view(sh) * dy + _U * z.abs()


def _gelu_bound(z, dz):
    """GELU(erf): |GELU'| <= 1.13; erff (2 ulp), the products and the sum <= 4 u (|z| + |GELU(z)|)"""
    g = F.gelu(z)
    return g, 1.13 * dz + 4 * _U * (z.abs() + g.abs())


def _dense_expected(sd64, mask, feat):
    """src = feat + mask_downscaling(mask) in float64 and its bound: conv 2x2 s2 (4 fma) -> LN2d(4) -> GELU -> conv 2x2 s2
    (16 fma) -> LN2d(16) -> GELU -> conv 1x1 (16 fma) -> + feat"""
    p = "prompt_encoder.mask_downscaling."
    m = mask.cuda().double().view(1, 1, 256, 256)
    W = {k[len(p):]: v.cuda() for k, v in sd64.items() if k.startswith(p)}
    conv = lambda x, w, b, s: F.conv2d(x, w, b, stride=s)
    v1 = conv(m, W["0.weight"], W["0.bias"], 2)
    dv1 = _gamma(5) * (conv(m.abs(), W["0.weight"].abs(), W["0.bias"].abs(), 2))
    h1, dh1 = _gelu_bound(*_ln2d_bound(v1, dv1, W["1.weight"], W["1.bias"], 1e-6))
    v2 = conv(h1, W["3.weight"], W["3.bias"], 2)
    dv2 = conv(dh1, W["3.weight"].abs(), None, 2) + _gamma(17) * conv(h1.abs(), W["3.weight"].abs(), W["3.bias"].abs(), 2)
    h2, dh2 = _gelu_bound(*_ln2d_bound(v2, dv2, W["4.weight"], W["4.bias"], 1e-6))
    d = conv(h2, W["6.weight"], W["6.bias"], 1)
    dd = conv(dh2, W["6.weight"].abs(), None, 1) + _gamma(17) * conv(h2.abs(), W["6.weight"].abs(), W["6.bias"].abs(), 1)
    tok = lambda x: x[0].flatten(1).t()
    src = feat.cuda().double() + tok(d)
    print(f"mask_downscaling variances: LN(4) {v1.var(1, unbiased=False).min().item():.2g} .. "
          f"{v1.var(1, unbiased=False).max().item():.2g}, LN(16) {v2.var(1, unbiased=False).min().item():.2g} .. "
          f"{v2.var(1, unbiased=False).max().item():.2g}")
    return src, tok(dd) + _U * src.abs()


def _pe_bound(sd64, xy):
    """bound of the kernel's PE of fp32 points xy [n, 2]: x + 0.5 (u), / 1024 (exact), 2 c - 1 (u), c_x g_0 + c_y g_1 (a product
    and an fma), * fp32(2 pi) (relative 2 u with the constant's own rounding) -> |d arg|; sinf / cosf add 2 ulp <= 4 u"""
    gm = sd64["prompt_encoder.pe_layer.positional_encoding_gaussian_matrix"].cuda()
    xn = (xy.cuda().double() + 0.5) / 1024
    c = 2 * xn - 1
    dc = _U * (2 * xn.abs() + 2 * c.abs())
    v = c @ gm
    dv = dc @ gm.abs() + _U * (c.abs() @ gm.abs() + v.abs())
    arg = 2 * math.pi * v
    darg = 2 * math.pi * dv + 2 * _U * arg.abs()
    print(f"PE: |arg| up to {arg.abs().max().item():.1f} rad")
    return torch.cat([darg, darg], dim=1) + 4 * _U


_PROMPTS = {
    # name: (coords, labels, box)
    "labels -1/0/1": ([[10.0, 20.0], [500.5, 300.25], [0.0, 0.0], [1023.5, 1023.5], [700.0, 100.0]], [1, 0, -1, 1, 0], None),
    "labels 2/3 on user points": ([[100.0, 200.0], [640.0, 480.0], [12.0, 900.0]], [2, 3, 1], None),
    "off-frame points": ([[-250.0, 40.0], [1500.0, -300.0], [1023.5, 2000.0], [-1000.0, -1000.0]], [1, 0, 1, 1], None),
    "box and points": ([[300.0, 300.0], [0.0, 1023.5]], [1, 0], [100.0, 150.0, 700.0, 440.0]),
    "box, edge corners": ([[512.0, 512.0]], [1], [0.0, 0.0, 1023.5, 1023.5]),
    "box, off-frame corners": ([[-20.0, 30.0], [40.0, 50.0]], [0, -1], [-100.0, -50.0, 1300.0, 1100.0]),
}


@pytest.fixture(scope="module")
def small_var_model():
    """weights whose 16-channel LayerNorm2d sees variances below its eps: mask_downscaling.3 scaled by 1e-3"""
    sd = _sd()
    for k in ("prompt_encoder.mask_downscaling.3.weight", "prompt_encoder.mask_downscaling.3.bias"):
        sd[k] = sd[k] * 1e-3
    sam = factory.build_sam("vit_test", sd).cuda()
    return sam, sd, {k: v.double() for k, v in sd.items()}


def _mask_bands(seed):
    """256 x 256 mask in four row bands of scale 0, 1e-4, 1 and 1e3: the 4-channel LayerNorm2d sees variances from the bias-only
    ~1e-3 up to ~1e5"""
    g = torch.Generator().manual_seed(seed)
    m = torch.randn((256, 256), generator=g)
    scale = torch.tensor([0.0, 1e-4, 1.0, 1e3]).repeat_interleave(64)
    return (m * scale[:, None]).contiguous()


@pytest.mark.parametrize("which,mask", [("model", False), ("model", True), ("small_var_model", True)])
@pytest.mark.parametrize("prompt", list(_PROMPTS))
def test_prompt_encoder(request, which, mask, prompt):
    """prompt_tokens_kernel + dense_src_kernel against float64 prompt_encode.  Labels other than -1 / 0 / 1 on user points
    get the positional encoding alone (upstream PromptEncoder._embed_points); the box corners get point_embeddings 2 / 3."""
    sam, sd, sd64 = request.getfixturevalue(which)
    coords, labels, box = _PROMPTS[prompt]
    K = len(labels)
    xy = torch.tensor(coords, dtype=torch.float32)
    lab = torch.tensor(labels, dtype=torch.int32)
    bx = torch.tensor(box, dtype=torch.float32) if box is not None else None
    g = torch.Generator().manual_seed(K)
    feat = torch.randn((_G * _G, 256), generator=g)
    m = _mask_bands(K) if mask else None
    T = _NOUT + K + (2 if box is not None else 1)
    ctx = _ctx(sam)
    tokens = torch.full((T, 256), float("nan"), device="cuda")
    src = torch.full((_G * _G, 256), float("nan"), device="cuda")
    # device copies held in locals: a temporary inside the call's argument list could be freed and its block reused before the
    # kernel reads it
    d_feat, d_xy, d_lab = feat.cuda(), xy.cuda(), lab.cuda()
    d_bx = bx.cuda() if bx is not None else None
    d_m = m.cuda() if m is not None else None
    native.check(native.lib().sampt_test_sam_prompt(
        ctx.handle, native.ptr(d_feat), c_int(_G), native.ptr(d_xy), native.ptr(d_lab), c_int(K), native.ptr(d_bx), native.ptr(d_m),
        native.ptr(tokens), native.ptr(src), native.stream_ptr()), "test_sam_prompt")
    torch.cuda.synchronize()
    # output tokens: copies
    out_tok = torch.cat([sd["mask_decoder.iou_token.weight"], sd["mask_decoder.mask_tokens.weight"]]).cuda()
    assert torch.equal(tokens[:_NOUT], out_tok)
    # point / pad / box tokens
    sparse, dense = sam_ref.prompt_encode(sd64, (xy.double()[None], lab.long()[None]),
                                          bx.double()[None] if bx is not None else None,
                                          m.double().view(1, 1, 256, 256) if m is not None else None)
    pts = xy if box is None else torch.cat([xy, bx.view(2, 2)])
    if box is None:
        pts = torch.cat([pts, torch.zeros((1, 2))])
    tol = _pe_bound(sd64, pts)
    not_pt = torch.tensor(labels + ([-1] if box is None else [0, 0])) == -1
    tol[not_pt.cuda()] = 0.0                                    # not_a_point_embed: copied
    tol = tol + _U * sparse[0].cuda().abs()                     # + the learned embedding
    _report(f"prompt tokens ({prompt})", (tokens[_NOUT:].double() - sparse[0].cuda()).abs(), tol + 1e-30)
    # dense part
    if m is None:
        exp = feat.cuda().double() + sd64["prompt_encoder.no_mask_embed.weight"].cuda().view(1, 256)
        _report(f"src, no mask ({prompt})", (src.double() - exp).abs(), _U * exp.abs() + 1e-30)
    else:
        exp, tol_d = _dense_expected(sd64, m, feat)
        assert (exp - (feat.cuda().double() + dense[0].cuda().flatten(1).t())).abs().max() < 1e-9
        _report(f"src with mask_in ({which}, {prompt})", (src.double() - exp).abs(), tol_d + 1e-30)


# ======================================================================================================= upscaling tail
@pytest.mark.parametrize("n_masks,with_u", [(1, False), (1, True), (3, False), (3, True)])
def test_upscale_tail(model, n_masks, with_u):
    """upscale_mask_kernel on a given first-ConvT output u1: LN2d(64) -> GELU -> ConvT(64->32) (64 fma) -> GELU -> hyper . (32 fma)"""
    sam, sd, sd64 = model
    g = torch.Generator().manual_seed(n_masks)
    u1 = torch.randn((_G * _G, 256), generator=g) * 2.0
    hyper = torch.randn((n_masks, 32), generator=g)
    ctx = _ctx(sam)
    R = 4 * _G
    low = torch.full((n_masks, R, R), float("nan"), device="cuda")
    u_out = torch.full((R * R, 32), float("nan"), device="cuda") if with_u else None
    d_u1, d_hyper = u1.cuda(), hyper.cuda()
    native.check(native.lib().sampt_test_sam_upscale(ctx.handle, native.ptr(d_u1), native.ptr(d_hyper), c_int(n_masks), c_int(_G),
                                                     native.ptr(low), native.ptr(u_out), native.stream_ptr()), "test_sam_upscale")
    torch.cuda.synchronize()
    p = "mask_decoder.output_upscaling."
    x = u1.cuda().double().view(_G, _G, 2, 2, 64).permute(4, 0, 2, 1, 3).reshape(1, 64, 2 * _G, 2 * _G)
    a, da = _gelu_bound(*_ln2d_bound(x, torch.zeros_like(x), sd64[p + "1.weight"].cuda(), sd64[p + "1.bias"].cuda(), 1e-6))
    w3, b3 = sd64[p + "3.weight"].cuda(), sd64[p + "3.bias"].cuda()
    c = F.conv_transpose2d(a, w3, b3, stride=2)
    dc = F.conv_transpose2d(da, w3.abs(), None, stride=2) + _gamma(65) * F.conv_transpose2d(a.abs(), w3.abs(), b3.abs(), stride=2)
    u, du = _gelu_bound(c, dc)
    u, du = u[0].flatten(1), du[0].flatten(1)                 # [32, R*R]
    h = hyper.cuda().double()
    exp = h @ u
    tol = h.abs() @ du + _gamma(32) * (h.abs() @ u.abs())
    _report(f"upscale low_res n_masks={n_masks} u_out={with_u}", (low.view(n_masks, -1).double() - exp).abs(), tol + 1e-30)
    if with_u:
        _report("upscale u_out", (u_out.double() - u.t()).abs(), du.t() + 1e-30)


# ======================================================================================================= postprocess
def _axis(in_size, out_size):
    """the kernel's src_index in fp32, exactly: scale = fp32(in / out), s = fmaf(scale, dst + 0.5, -0.5) (the fp32 product is
    exact in float64, so float64 then one rounding is the fma), clamp at 0, i0 = trunc(s) clamped to in - 1, l1 = s - i0,
    l0 = fp32(1 - l1).  Returns the [out, in] interpolation matrix with those weights."""
    sc = np.float32(in_size) / np.float32(out_size)
    s = (np.float64(sc) * (np.arange(out_size, dtype=np.float64) + 0.5) - 0.5).astype(np.float32)
    s = np.maximum(s, np.float32(0))
    i0 = np.minimum(s.astype(np.int64), in_size - 1)
    i1 = i0 + (i0 < in_size - 1)
    l1 = (s - i0.astype(np.float32)).astype(np.float32)
    l0 = (np.float32(1) - l1).astype(np.float32)
    A = np.zeros((out_size, in_size))
    np.add.at(A, (np.arange(out_size), i0), l0.astype(np.float64))
    np.add.at(A, (np.arange(out_size), i1), l1.astype(np.float64))
    return torch.from_numpy(A)


def _pp_matrices(in_h, in_w, H, W):
    """composite [H, 256] / [W, 256] matrices of 256 -> 1024 (no crop needed: rows >= in_h are never read) -> in x -> H x W"""
    up = _axis(4 * _G, 16 * _G)
    return (_axis(in_h, H) @ up[:in_h]).cuda(), (_axis(in_w, W) @ up[:in_w]).cuda()


def _run_pp(sam, low, in_hw, HW):
    n = low.shape[0]
    ctx = _ctx(sam)
    out = torch.full((n,) + HW, float("nan"), device="cuda")
    bbox = torch.full((5,), -7, dtype=torch.int32, device="cuda")
    box4 = torch.full((4,), -7.0, device="cuda")
    skip = torch.full((1,), 5, dtype=torch.int32, device="cuda")
    ndone = torch.full((1,), 5, dtype=torch.int32, device="cuda")
    d_low = low.cuda().contiguous()
    native.check(native.lib().sampt_test_sam_postprocess(
        ctx.handle, native.ptr(d_low), c_int(n),c_int(_G), c_int(in_hw[0]), c_int(in_hw[1]), c_int(HW[0]),
        c_int(HW[1]), native.ptr(out), native.ptr(bbox), native.ptr(box4), native.ptr(skip), native.ptr(ndone),
        native.stream_ptr()), "test_sam_postprocess")
    torch.cuda.synchronize()
    return out, bbox.cpu(), box4.cpu(), int(skip.item()), int(ndone.item())


def _check_ctl(out, bbox, box4, skip, ndone, what):
    """bbox / count exactly as the host computes them from the kernel's own mask 0; the break test and its outputs"""
    pos = (out[0] > 0).nonzero().cpu()
    cnt = pos.shape[0]
    assert int(bbox[4]) == cnt, (what, int(bbox[4]), cnt)
    if cnt:
        exp = [int(pos[:, 1].min()), int(pos[:, 0].min()), int(pos[:, 1].max()), int(pos[:, 0].max())]
        assert bbox[:4].tolist() == exp, (what, bbox.tolist(), exp)
    else:
        assert bbox[:4].tolist() == [0x7FFFFFFF, 0x7FFFFFFF, -1, -1], (what, bbox.tolist())
    assert skip == (1 if cnt < 2 else 0), (what, cnt, skip)
    if cnt >= 2:
        assert ndone == 1 and box4.tolist() == [float(x) for x in bbox[:4].tolist()], (what, ndone, box4.tolist())
    else:
        assert ndone == 0 and box4.tolist() == [-7.0] * 4, (what, ndone, box4.tolist())
    return cnt, bbox[:4].tolist()


_GEOMS = [(480, 854), (240, 320), (1080, 1920), (1920, 1080), (97, 131), (481, 855), (1024, 1024)]


@pytest.mark.parametrize("H,W", _GEOMS)
def test_postprocess_values(model, H, W):
    """both bilinear resizes against float64 with the kernel's own fp32 source coordinates: each resize is 2 fma levels on
    non-negative weights, so |err| <= gamma_6 (|A| |low| |B|^T) for the composite matrices A, B"""
    sam = model[0]
    in_hw = sam_ref.get_preprocess_shape(H, W)
    g = torch.Generator().manual_seed(H + W)
    low = torch.randn((3, 4 * _G, 4 * _G), generator=g) * 8.0
    out, bbox, box4, skip, ndone = _run_pp(sam, low, in_hw, (H, W))
    A, B = _pp_matrices(in_hw[0], in_hw[1], H, W)
    L = low.cuda().double()
    exp = A @ L @ B.t()
    tol = _gamma(6) * (A @ L.abs() @ B.t()) + 1e-30
    _report(f"postprocess {H}x{W} (input {in_hw[0]}x{in_hw[1]})", (out.double() - exp).abs(), tol)
    ref = sam_ref.postprocess_masks(low.double()[None], in_hw, (H, W))[0].cuda()
    print(f"  against F.interpolate in float64 (coordinates in float64): max diff {(out.double() - ref).abs().max().item():.3g}")
    _check_ctl(out, bbox, box4, skip, ndone, f"{H}x{W} random")


def _impulse_level(A, B, a, b, k):
    """low_res = -1 everywhere and v at (a, b): out = -1 + (v + 1) A[:, a] B[:, b]^T.  Returns v for exactly k positive pixels
    (threshold halfway between the k-th and (k+1)-th largest weights), or None when those weights are too close to separate"""
    w = torch.sort((A[:, a][:, None] * B[:, b][None, :]).flatten(), descending=True).values
    if w[k - 1] <= 0 or w[k - 1] - w[k] < 1e-3 * w[k - 1]:
        return None
    return 2.0 / (w[k - 1] + w[k]).item() - 1.0


@pytest.mark.parametrize("H,W", _GEOMS)
def test_postprocess_bbox_and_break(model, H, W):
    """area 0, 1 and 2 (the break fires below 2), positives on row 0 / column 0 / row H-1 / column W-1, and a mask 0 that is
    empty while masks 1 and 2 are not: bbox and count equal the host's box and count of the kernel's mask 0"""
    sam = model[0]
    in_hw = sam_ref.get_preprocess_shape(H, W)
    A, B = _pp_matrices(in_hw[0], in_hw[1], H, W)
    R = 4 * _G
    base = -torch.ones((1, R, R))
    counts = set()
    # low-res pixels that some output pixel reads with a large weight (a downscale reads only some of them)
    cands = [(int(A[H * i // 7].argmax()), int(B[W * j // 7].argmax())) for i in range(1, 7) for j in range(1, 7)]
    for k in (1, 2):
        for a, b in cands:
            v = _impulse_level(A, B, a, b, k)
            if v is not None:
                low = base.clone()
                low[0, a, b] = v
                cnt, _ = _check_ctl(*_run_pp(sam, low, in_hw, (H, W)), f"{H}x{W} impulse k={k}")
                assert cnt == k, (k, cnt)
                counts.add(cnt)
                break
    if (H, W) in ((480, 854), (240, 320), (481, 855)):   # an upscale's impulse response has tied maxima: no single pixel
        assert counts == {1, 2}, counts
    cnt, _ = _check_ctl(*_run_pp(sam, base, in_hw, (H, W)), "all negative")
    assert cnt == 0
    # corners of the valid region
    low = base.clone()
    low[0, 0, 0] = 50.0
    cnt, box = _check_ctl(*_run_pp(sam, low, in_hw, (H, W)), "top-left")
    assert box[0] == 0 and box[1] == 0, box
    low = base.clone()
    a, b = int(A[H - 1].argmax()), int(B[W - 1].argmax())
    low[0, a, b] = 50.0
    cnt, box = _check_ctl(*_run_pp(sam, low, in_hw, (H, W)), "bottom-right")
    assert box[2] == W - 1 and box[3] == H - 1, box
    # mask 0 empty, masks 1 / 2 full
    low3 = torch.cat([base, -base, -base])
    out, *ctl = _run_pp(sam, low3, in_hw, (H, W))
    assert _check_ctl(out, *ctl, "mask 0 empty of 3")[0] == 0
    assert (out[1:] > 0).all()


# ======================================================================================================= whole predict_torch calls
@pytest.fixture(scope="module")
def predictor(model):
    from segment_anything.predictor import SamPredictor
    sam, sd, sd64 = model
    g = torch.Generator().manual_seed(9)
    feats = torch.randn((1, 256, _G, _G), generator=g)
    pred = SamPredictor(sam)
    pred.set_frames_features((480, 854), feats.cuda())
    refs = []
    for s, f in ((sd, feats), (sd64, feats.double())):
        r = sam_ref.RefSamPredictor(s, sam_ref.VIT_TEST)
        r.features, r.original_size, r.input_size = f, (480, 854), (576, 1024)
        refs.append(r)
    return pred, refs[0], refs[1], feats


def _vs_oracle(what, gpu, cpu32, f64):
    """as accurate as an fp32 implementation: |GPU - float64| <= 4 |CPU float32 oracle - float64| + 2^-20 max |float64|"""
    f64 = f64.double().cpu()
    e_gpu = (gpu.double().cpu() - f64).abs().max().item()
    e_cpu = (cpu32.double().cpu() - f64).abs().max().item()
    bound = 4 * e_cpu + 2.0 ** -20 * f64.abs().max().item()
    print(f"{what}: GPU err {e_gpu:.3g}, CPU fp32 err {e_cpu:.3g}, GPU err / bound {e_gpu / bound if bound else 0.0:.3g}")
    assert e_gpu <= bound, (what, e_gpu, bound)


def _prompt(K, seed, box_mask):
    g = torch.Generator().manual_seed(seed)
    pts = torch.rand((1, K, 2), generator=g) * torch.tensor([1020.0, 570.0])
    labels = (torch.rand((1, K), generator=g) < 0.7).int()
    box = mask = None
    if box_mask:
        box = torch.tensor([[100.0, 150.0, 700.0, 440.0]])
        mask = torch.randn((1, 1, 256, 256), generator=g) * 4.0
    return pts, labels, box, mask


def _predict_all(pred, r32, r64, pts, labels, box, mask, multimask):
    cu = lambda t: t.cuda() if t is not None else None
    d = lambda t: t.double() if t is not None else None
    gpu = pred.predict_torch(cu(pts), cu(labels), cu(box[:, None]) if box is not None else None, cu(mask), multimask, True)
    c32 = r32.predict_torch(pts, labels, box, mask, multimask, True)
    c64 = r64.predict_torch(d(pts), labels, d(box), d(mask), multimask, True)
    return gpu, c32, c64


@pytest.mark.parametrize("box_mask", [False, True])
@pytest.mark.parametrize("K", [1, 10, 11, 26, 27, 58, 59, 256, 320])
def test_predict_torch_prompt_sizes(predictor, K, box_mask):
    """T = 5 + K + 1 (points) or 5 + K + 2 (box) on both sides of 16, 32 and 64, up to the slot capacity"""
    pred, r32, r64, _ = predictor
    (m, i, l), (m32, i32, l32), (m64, i64, l64) = _predict_all(pred, r32, r64, *_prompt(K, K, box_mask), False)
    T = _NOUT + K + (2 if box_mask else 1)
    for name, a, b, c in (("low_res", l, l32, l64), ("logits", m, m32, m64), ("iou", i, i32, i64)):
        _vs_oracle(f"predict_torch K={K} T={T} box+mask={box_mask} {name}", a, b, c)


def test_predict_torch_multimask_box_mask(predictor):
    pred, r32, r64, _ = predictor
    (m, i, l), (m32, i32, l32), (m64, i64, l64) = _predict_all(pred, r32, r64, *_prompt(9, 77, True), True)
    assert m.shape == (1, 3, 480, 854) and l.shape == (1, 3, 256, 256)
    for name, a, b, c in (("low_res", l, l32, l64), ("logits", m, m32, m64), ("iou", i, i32, i64)):
        _vs_oracle(f"predict_torch multimask {name}", a, b, c)


@pytest.fixture(scope="module")
def hq():
    from segment_anything_hq.predictor import SamPredictor
    sd = _sd(43, hq=True)
    sd64 = {k: v.double() for k, v in sd.items()}
    sam = factory.build_sam("vit_test", sd, hq=True).cuda()
    g = torch.Generator().manual_seed(19)
    feats = torch.randn((1, 256, _G, _G), generator=g)
    interm = torch.randn((1, _G, _G, sam_ref.VIT_TEST.embed_dim), generator=g)
    pred = SamPredictor(sam)
    pred.set_frames_features((480, 854), (feats.cuda(), interm.cuda()))
    refs = []
    for s, f, it in ((sd, feats, interm), (sd64, feats.double(), interm.double())):
        r = sam_ref.RefSamPredictor(s, sam_ref.VIT_TEST, hq=True)
        r.features, r.interm, r.original_size, r.input_size = f, [it], (480, 854), (576, 1024)
        refs.append(r)
    return pred, refs[0], refs[1], sd, sd64, feats, interm


def _hq_features_ref(sd, feats, interm):
    p = "mask_decoder."
    e = F.conv_transpose2d(feats, sd[p + "embedding_encoder.0.weight"], sd[p + "embedding_encoder.0.bias"], stride=2)
    e = F.gelu(sam_ref._ln2d(e, sd[p + "embedding_encoder.1.weight"], sd[p + "embedding_encoder.1.bias"]))
    e = F.conv_transpose2d(e, sd[p + "embedding_encoder.3.weight"], sd[p + "embedding_encoder.3.bias"], stride=2)
    cv = F.conv_transpose2d(interm.permute(0, 3, 1, 2), sd[p + "compress_vit_feat.0.weight"], sd[p + "compress_vit_feat.0.bias"],
                            stride=2)
    cv = F.gelu(sam_ref._ln2d(cv, sd[p + "compress_vit_feat.1.weight"], sd[p + "compress_vit_feat.1.bias"]))
    cv = F.conv_transpose2d(cv, sd[p + "compress_vit_feat.3.weight"], sd[p + "compress_vit_feat.3.bias"], stride=2)
    return (e + cv)[0].flatten(1).t()                         # [(4G)^2, 32] channels-last


def test_hq_features_and_predict_c5_shape(hq):
    """sampt_sam_hq_features against float64 embedding_encoder + compress_vit_feat, then one HQ predict_torch at K = 256
    (T = 6 + 256 + 1 = 263, the C5 shape)"""
    pred, r32, r64, sd, sd64, feats, interm = hq
    got = pred._hq_features()
    _vs_oracle("hq_features", got, _hq_features_ref(sd, feats, interm), _hq_features_ref(sd64, feats.double(), interm.double()))
    (m, i, l), (m32, i32, l32), (m64, i64, l64) = _predict_all(pred, r32, r64, *_prompt(256, 5, False), False)
    for name, a, b, c in (("low_res", l, l32, l64), ("logits", m, m32, m64), ("iou", i, i32, i64)):
        _vs_oracle(f"HQ predict_torch K=256 T=263 {name}", a, b, c)
    with pytest.raises(RuntimeError):
        pred.predict_torch(*[t.cuda() for t in _prompt(4, 1, False)[:2]], multimask_output=True)


# ======================================================================================================= chain and graph invariants
def _refine(pred, pts, labels, n_refine, slot=0):
    out = torch.empty(pred.original_size, device="cuda")
    iou, low, nd = pred.predict_refine(pts.cuda(), labels.cuda(), 0, n_refine, out, slot=slot)
    return out, iou, low, nd


def _same(a, b, what):
    for x, y in zip(a, b):
        assert torch.equal(x, y), what


def _eager(ctx, fn):
    """run fn with no decoder slab (the eager chain out of the shared workspace), then restore the slab"""
    ctx.clear_decoder_workspace()
    try:
        return fn()
    finally:
        ctx.set_decoder_workspace()


def test_chain_invariants(predictor, model):
    pred, r32, r64, feats = predictor
    sam = model[0]
    ctx = _ctx(sam)
    pts, labels, _, _ = _prompt(8, 3, False)
    # predict == predict_refine(n_refine = 0)
    m, i, l = pred.predict_torch(pts.cuda(), labels.cuda(), None, None, False, True)
    out, iou, low, nd = _refine(pred, pts[0], labels[0], 0)
    _same((m[0, 0], i[0], l[0, 0]), (out, iou, low), "sampt_sam_predict vs predict_refine(0)")
    assert int(nd.item()) == 0
    # the 1 + 12 chain: CUDA graph vs eager
    graph = _refine(pred, pts[0], labels[0], 12)
    eager = _eager(ctx, lambda: _refine(pred, pts[0], labels[0], 12))
    print(f"1 + 12 chain: {int(graph[3].item())} refinements")
    assert int(graph[3].item()) >= 1
    _same(graph, eager, "graph vs eager chain")
    # one slot: K = 6, K = 40, K = 6 again
    p6, l6, _, _ = _prompt(6, 11, False)
    p40, l40, _, _ = _prompt(40, 12, False)
    first = _refine(pred, p6[0], l6[0], 12, slot=3)
    _refine(pred, p40[0], l40[0], 12, slot=3)
    _same(first, _refine(pred, p6[0], l6[0], 12, slot=3), "slot 3: K=6 after K=40")
    # K = 400 > DEC_KCAP_MIN: the slot is re-carved
    p400, l400, _, _ = _prompt(400, 13, False)
    big = _refine(pred, p400[0], l400[0], 12, slot=3)
    _same(big, _eager(ctx, lambda: _refine(pred, p400[0], l400[0], 12)), "K=400 graph vs eager")


def test_concurrent_slots(predictor, model):
    """two slots on two streams, two feature maps, concurrently == one after the other"""
    from segment_anything.predictor import SamPredictor
    pred, _, _, _ = predictor
    sam = model[0]
    _ctx(sam)
    pred2 = SamPredictor(sam)
    g = torch.Generator().manual_seed(99)
    pred2.set_frames_features((480, 854), torch.randn((1, 256, _G, _G), generator=g).cuda())
    pa, la, _, _ = _prompt(12, 21, False)
    pb, lb, _, _ = _prompt(30, 22, False)
    seq_a = _refine(pred, pa[0], la[0], 12, slot=5)
    seq_b = _refine(pred2, pb[0], lb[0], 12, slot=6)
    torch.cuda.synchronize()
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    sa.wait_stream(torch.cuda.current_stream())
    sb.wait_stream(torch.cuda.current_stream())
    for _ in range(3):
        with torch.cuda.stream(sa):
            ca = _refine(pred, pa[0], la[0], 12, slot=5)
        with torch.cuda.stream(sb):
            cb = _refine(pred2, pb[0], lb[0], 12, slot=6)
        torch.cuda.synchronize()
        _same(seq_a, ca, "slot 5 concurrent")
        _same(seq_b, cb, "slot 6 concurrent")


def test_empty_first_mask_stops_chain(predictor):
    """hyper-network 0 zeroed: the first mask is empty, the chain stops at once (n_done = 0) as the oracle's loop does"""
    from segment_anything.predictor import SamPredictor
    _, _, _, feats = predictor
    sd = _sd()
    for k in ("mask_decoder.output_hypernetworks_mlps.0.layers.2.weight", "mask_decoder.output_hypernetworks_mlps.0.layers.2.bias"):
        sd[k] = torch.zeros_like(sd[k])
    sam = factory.build_sam("vit_test", sd).cuda()
    pred = SamPredictor(sam)
    pred.set_frames_features((480, 854), feats.cuda())
    pts, labels, _, _ = _prompt(8, 3, False)
    out, iou, low, nd = _refine(pred, pts[0], labels[0], 12)
    assert int(nd.item()) == 0
    assert (out <= 0).all() and (low <= 0).all()
    refs = []
    for s in (sd, {k: v.double() for k, v in sd.items()}):
        r = sam_ref.RefSamPredictor(s, sam_ref.VIT_TEST)
        r.features, r.original_size, r.input_size = feats.to(next(iter(s.values())).dtype), (480, 854), (576, 1024)
        refs.append(r.predict_torch(pts.to(r.features.dtype), labels, None, None, False, True))
    assert int((refs[1][0][0, 0] > 0).sum()) < 2                # the oracle's loop breaks before its first refinement
    for name, a, j in (("logits", out, 0), ("iou", iou, 1), ("low_res", low, 2)):
        _vs_oracle(f"empty first mask {name}", a, refs[0][j][0, 0] if j != 1 else refs[0][j][0],
                   refs[1][j][0, 0] if j != 1 else refs[1][j][0])
