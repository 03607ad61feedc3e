"""GPU: the SAM ViT image encoder (csrc/vit_pipeline.cu, csrc/vit_kernels.cu) kernel by kernel against float64 -- patch
embedding, the LayerNorm rows in every layout and with every row map, one block at every precision, the neck -- and the
padding-window skip end to end.

Bounds.  u = 2^-24.  A hi | lo operand reproduces its value to |v - hi - lo| <= 2^-22 |v| (2^-25 absolute where lo is an fp16
subnormal, which the 2^s weight scaling keeps away from the weights).  A GEMM's error is judged by its relative rms over the
whole output, where rounding errors of random sign average out and the bars below separate the forms of the product:
  - three fp16 passes: 2^-17.  The operands alone would allow ~5e-8 (a CPU emulation with fp32 round-to-nearest sums), but the
    tensor cores' fp32 accumulation is not round-to-nearest and dominates: on one H100 the patch embedding (K = 768) measures
    4.0e-6 and the neck 1.9e-6 to 2.2e-6;
  - e4m3 correction segments (precision 6): 4 x 1.0e-5 (DESIGN section 5);
  - fp16 activations (precision 1 and 2): 2^-10 (the fp16 rounding of each operand is 2^-12 rms).
A block's MLP half chains two GEMMs (K up to 5120) through GELU and is held to 2^-14 at three passes (measured 2.0e-5 to 3.3e-5;
a dropped 2^-12 correction segment costs ~2e-4); its attention half to twice the error
of a float64 emulation of the attention path's fp16 storage, plus the GEMM bars of qkv and proj.
Element-wise kernels (im2col, LayerNorm, the e4m3 bytes) are held element by element.  Outputs start as NaN, so anything a
kernel should write and does not shows up, and rows a kernel must not write keep their old bits."""
from ctypes import c_float, c_int

import pytest
import torch
import torch.nn.functional as F

from oracle import sam_ref

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
MEAN = sam_ref.PIXEL_MEAN
STD = sam_ref.PIXEL_STD
G, P, WS = 64, 16, 14
NW = 5
REL_3PASS = 2.0 ** -17
REL_3PASS_MLP = 2.0 ** -14
REL_F8 = 4.0e-5
REL_F16 = 2.0 ** -10


def _n():
    from sampt_b200 import native
    return native


def _rel_gemm(passes, f8=False):
    return REL_F8 if f8 else (REL_3PASS if passes == 3 else REL_F16)


def _prec(p):
    """(passes of the MLP / embed / neck GEMMs, of qkv, of proj, attention output carried as hi | lo) of sampt_vit_encode"""
    p_qkv = 2 if p in (3, 5) else (3 if p >= 4 else p)
    p_proj = 2 if p == 3 else (3 if p >= 4 else p)
    return min(p, 3), p_qkv, p_proj, p >= 4


def _encoder(D, heads, depth=2, globals_=(1,), seed=0, hq=False):
    """ImageEncoderViT on the GPU with its seeded weights, LayerNorm affines perturbed away from (1, 0)"""
    if hq:
        from segment_anything_hq.modeling.image_encoder import ImageEncoderViT
    else:
        from segment_anything.modeling.image_encoder import ImageEncoderViT
    enc = ImageEncoderViT(embed_dim=D, depth=depth, num_heads=heads, use_rel_pos=True, window_size=WS,
                          global_attn_indexes=globals_)
    g = torch.Generator().manual_seed(seed + D)
    with torch.no_grad():
        for k, v in enc.named_parameters():
            if "norm" in k or "neck.1." in k or "neck.3." in k:
                v.copy_((1.0 if k.endswith("weight") else 0.0) + 0.2 * torch.randn(v.shape, generator=g))
    return enc.cuda()


@pytest.fixture(scope="module")
def vit_h():
    return _encoder(1280, 16, seed=1)


@pytest.fixture(scope="module")
def vit_b():
    return _encoder(768, 12, seed=2)


def _sd64(enc):
    return {"image_encoder." + k: v.detach().double() for k, v in enc.state_dict().items()}


def _ctx(enc, precision, B):
    enc.precision = precision
    ctx = enc.native_context()
    ctx.ensure_vit_workspace(enc.workspace_bytes(B))
    return ctx


def _rel_rms(err, ref):
    return (err.double().pow(2).mean().sqrt() / ref.double().pow(2).mean().sqrt()).item()


# ------------------------------------------------------------------------------------------------------ patch embedding
def _frames(B, Hr, Wr, seed):
    g = torch.Generator().manual_seed(seed)
    u8 = torch.randint(0, 256, (B, 3, Hr, Wr), generator=g, dtype=torch.uint8)
    u8[:, :, :5, :] = 255
    u8[:, :, -3:, -7:] = 0
    return u8


def _preprocess(u8):
    """Sam.preprocess in torch float32: one subtraction and one IEEE division per value, zero padding to 1024^2"""
    x = (u8.float() - torch.tensor(MEAN).view(1, 3, 1, 1)) / torch.tensor(STD).view(1, 3, 1, 1)
    return F.pad(x, (0, 1024 - u8.shape[3], 0, 1024 - u8.shape[2]))


def _im2col(x):
    """(B,3,1024,1024) -> [B*G*G, 3*P*P], column c*P*P + iy*P + ix"""
    B = x.shape[0]
    return x.view(B, 3, G, P, G, P).permute(0, 2, 4, 1, 3, 5).reshape(B * G * G, 3 * P * P)


def _embed(enc, image, is_f32, B, Hr, Wr, precision):
    n = _n()
    ctx = _ctx(enc, precision, B)
    asp = 2 if precision >= 3 else 1
    K = 3 * P * P
    a = torch.full((B * G * G, K * asp), float("nan"), device="cuda").half()
    x = torch.full((B * G * G, enc.embed_dim), float("nan"), device="cuda")
    m, s = (c_float * 3)(*MEAN), (c_float * 3)(*STD)
    img = image.cuda().contiguous()
    n.check(n.lib().sampt_test_vit_embed(ctx.handle, n.ptr(img), c_int(is_f32), c_int(B), c_int(Hr), c_int(Wr),
                                         c_int(enc.embed_dim), c_int(1024), c_int(P), c_int(precision), m, s, n.ptr(a),
                                         n.ptr(x), n.stream_ptr()), "vit_embed")
    torch.cuda.synchronize()
    return a, x


def _embed_ref(enc, x32):
    sd = _sd64(enc)
    w = sd["image_encoder.patch_embed.proj.weight"].cuda()
    y = F.conv2d(x32.double().cuda(), w, stride=P).permute(0, 2, 3, 1)
    mag = F.conv2d(x32.double().abs().cuda(), w.abs(), stride=P).permute(0, 2, 3, 1)
    full = y + sd["image_encoder.patch_embed.proj.bias"].cuda() + sd["image_encoder.pos_embed"].cuda()
    D = enc.embed_dim
    return y.reshape(-1, D), mag.reshape(-1, D), full.reshape(-1, D)


def _check_embed(enc, a, x, x32, precision, what):
    asp = 2 if precision >= 3 else 1
    K = 3 * P * P
    want = _im2col(x32).cuda()
    hi = want.half()
    assert torch.equal(a[:, :K].view(torch.int16), hi.view(torch.int16)), f"{what}: hi operand"
    if asp == 2:
        lo = (want - hi.float()).half()
        assert torch.equal(a[:, K:].view(torch.int16), lo.view(torch.int16)), f"{what}: lo operand"
    y, mag, full = _embed_ref(enc, x32)
    err = x.double() - full
    assert torch.isfinite(x).all(), what
    # element-wise: the representation of both operands, fp32 accumulation over K, + bias + pos_embed
    passes = min(precision, 3)
    rep = 3 * 2.0 ** -22 if passes == 3 else 2.0 ** -10
    bound = (rep + K * U) * mag + 4 * U * full.abs()
    assert (err.abs() <= bound).all(), (what, (err.abs() / bound).max().item())
    r = _rel_rms(err, y)
    print(f"{what}: relative rms {r:.3e} (bar {_rel_gemm(passes):.3e})")
    assert r <= _rel_gemm(passes), (what, r)


@pytest.mark.parametrize("precision", [1, 2, 6])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("Hr,Wr", [(576, 1024), (1024, 576), (1024, 683), (1024, 1024)])
def test_embed_u8(vit_b, Hr, Wr, B, precision):
    """Normalisation, zero padding and the im2col bit for bit (torch's fp32 (u8 - mean) / std split into hi | lo), then the
    patch GEMM + bias + pos_embed against float64.  683 leaves a partial patch column."""
    u8 = _frames(B, Hr, Wr, Hr * 7 + Wr + B)
    a, x = _embed(vit_b, u8, 0, B, Hr, Wr, precision)
    _check_embed(vit_b, a, x, _preprocess(u8), precision, f"embed u8 {Hr}x{Wr} B{B} p{precision}")


@pytest.mark.parametrize("precision", [1, 6])
def test_embed_f32(vit_h, precision):
    """The float image path (upstream forward(x)): im2col_f32 bit for bit, including values whose lo is an fp16 subnormal."""
    g = torch.Generator().manual_seed(5)
    x32 = torch.randn((2, 3, 1024, 1024), generator=g) * 2
    x32[0, 0, :16, :16] = 1e-6 * torch.randn((16, 16), generator=g)
    a, x = _embed(vit_h, x32, 1, 2, 1024, 1024, precision)
    _check_embed(vit_h, a, x, x32, precision, f"embed f32 p{precision}")


# ------------------------------------------------------------------------------------------------------------- ln_rows
def _window_map(B, ny, nx):
    """window_map_kernel / live_window_map_kernel: window-partitioned row -> token row, -1 for padding"""
    L = WS * WS
    r = torch.arange(B * ny * nx * L)
    t, wb = r % L, r // L
    w, b = wb % (ny * nx), wb // (ny * nx)
    y, x = (w // nx) * WS + t // WS, (w % nx) * WS + t % WS
    return torch.where((y < G) & (x < G), b * G * G + y * G + x, torch.full_like(r, -1)).int()


def _token_map(B, rows, cols):
    """live_token_map_kernel"""
    r = torch.arange(B * rows * cols)
    i, b = r % (rows * cols), r // (rows * cols)
    return (b * G * G + (i // cols) * G + i % cols).int()


MAPS = {
    "identity": lambda B: None,
    "window": lambda B: _window_map(B, NW, NW),
    "live3x5": lambda B: _window_map(B, 3, 5),
    "live5x3": lambda B: _window_map(B, 5, 3),
    "tokens": lambda B: _token_map(B, 42, 64),
}


def _ln_rows_input(D, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((2 * G * G, D), generator=g)
    out = torch.rand((2 * G * G,), generator=g) < 0.05
    idx = torch.randint(0, D, (2 * G * G, 3), generator=g)
    x[out.nonzero()[:, 0, None], idx[out]] *= 100.0                # a few x100 outlier channels
    for b in range(2):
        r = b * G * G
        x[r + 5] = 0.375                                             # constant row: zero variance
        x[r + 6] = 1e3 + torch.randn((D,), generator=g)              # large mean
        x[r + 9] = -0.5 + 1e-3 * torch.randn((D,), generator=g)      # variance 1e-6 = eps
    return x


def _e4m3_ord(b):
    """e4m3 byte -> signed ordinal of its code (adjacent codes differ by one)"""
    b = b.to(torch.int32)
    return torch.where(b >= 128, -(b - 128), b)


@pytest.mark.parametrize("mapname", list(MAPS))
@pytest.mark.parametrize("D", [128, 640, 768, 1024, 1280, 1536])
def test_ln_rows(D, mapname):
    """ln_rows against float64 LayerNorm (eps 1e-6) in all three layouts; -1 rows of a map are zeros in every layout.

    fp32 bound: a lane sums D/32 values, then 5 shuffle levels, so |d mean| <= (D/32 + 5) u mean|x| and the variance is
    computed to (D/32 + 7) u relative plus the square of that mean error; x_hat then errs by |d mean| rstd + |x_hat| (half the
    variance error + 3 u), and gamma x_hat + beta adds 3 u of its terms."""
    n = _n()
    from sampt_b200 import native
    ctx = native.get_context(torch.device("cuda"))
    g = torch.Generator().manual_seed(D)
    x = _ln_rows_input(D, D + len(mapname))
    gamma = 1.0 + 0.3 * torch.randn((D,), generator=g)
    beta = 0.2 * torch.randn((D,), generator=g)
    smap = MAPS[mapname](2)
    M = x.shape[0] if smap is None else smap.numel()
    src = torch.arange(M) if smap is None else smap.long()
    valid = src >= 0
    xs = torch.zeros((M, D), dtype=torch.float64)
    xs[valid] = x[src[valid]].double()
    mu = xs.mean(1, keepdim=True)
    var = (xs - mu).pow(2).mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + 1e-6)
    xh = (xs - mu) * rstd
    ref = xh * gamma.double() + beta.double()
    e_mu = (D / 32 + 5) * U * xs.abs().mean(1, keepdim=True)
    e_var = (D / 32 + 7) * U + (e_mu * rstd) ** 2
    bnd = (e_mu * rstd + xh.abs() * (0.5 * e_var + 3 * U)) * gamma.double().abs() + 3 * U * (
        (xh * gamma.double()).abs() + beta.double().abs())
    ref[~valid] = 0
    bnd[~valid] = 0
    xg, gg, bg = x.cuda(), gamma.cuda(), beta.cuda()
    sg = smap.cuda() if smap is not None else None
    for normalize in ((1, 0) if mapname == "identity" else (1,)):
        want, b = (ref, bnd) if normalize else (xs, torch.zeros_like(bnd))
        for layout in (0, 1, 2):
            out = torch.full((M, 2 * D if layout else D), float("nan"), device="cuda").half()
            n.check(n.lib().sampt_test_vit_ln(ctx.handle, n.ptr(xg), c_int(D), n.ptr(sg), c_int(M), c_int(D), c_int(normalize),
                                              n.ptr(gg), n.ptr(bg), c_int(layout), n.ptr(out), n.stream_ptr()), "vit_ln")
            torch.cuda.synchronize()
            what = f"ln D{D} {mapname} norm{normalize} layout{layout}"
            o = out.cpu()
            hi = o[:, :D].double()
            assert torch.isfinite(hi).all(), what
            if layout == 1:
                v = hi + o[:, D:].double()
                tol = b + 2.0 ** -22 * want.abs() + 2.0 ** -25
            else:
                v = hi
                tol = b + 2.0 ** -11 * want.abs() + 2.0 ** -25
            assert ((v - want).abs() <= tol).all(), (what, ((v - want).abs() / tol).max().item())
            if layout == 2:
                by = o[:, D:].contiguous().view(torch.uint8)            # [M, 2D] bytes: lo8 block, then hi8 block
                lo8, hi8 = by[:, :D], by[:, D:]
                r_hi = (want * 0.125).float().clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8)
                # hi8 rounds the kernel's fp32 value, which is within tol of the float64 one: one code either way
                assert ((_e4m3_ord(hi8) - _e4m3_ord(r_hi)).abs() <= 1).all(), what + " hi8"
                # lo8 carries (v - hi) 2^12, small enough that the fp32 LayerNorm error can move it by several codes: check the
                # value it restores (e4m3 rounds to 2^-4 relative, 2^-10 absolute below its normal range).  The layout covers
                # |v| < 2^7, where (v - hi) 2^12 stays inside e4m3's 448; beyond that the byte may saturate (only the cast-only
                # rows with outliers reach it: LayerNorm outputs stay far below).
                lo = lo8.view(torch.float8_e4m3fn).double() / 4096.0
                tol8 = b + 2.0 ** -4 * (want - hi).abs() + 2.0 ** -22
                inside = want.abs() < 128
                assert ((hi + lo - want).abs() <= tol8)[inside].all(), what + " lo8"
            if smap is not None:
                pad = ~valid
                assert (o[pad].view(torch.int16) == 0).all(), what + ": padding rows must be +0 in every byte"


# ----------------------------------------------------------------------------------------------------------- one block
def _run_block(enc, blk, is_global, x, precision, B, Hr=1024, Wr=1024, live_only=0, want_mid=True):
    n = _n()
    ctx = _ctx(enc, precision, B)
    xg = x.cuda().contiguous().clone()
    mid = torch.full_like(xg, float("nan")) if want_mid else None
    n.check(n.lib().sampt_test_vit_block(ctx.handle, c_int(blk), c_int(is_global), n.ptr(xg), n.ptr(mid), c_int(B), c_int(Hr),
                                         c_int(Wr), c_int(live_only), c_int(enc.embed_dim), c_int(enc.num_heads), c_int(WS),
                                         c_int(1024), c_int(P), c_int(precision), n.stream_ptr()), "vit_block")
    torch.cuda.synchronize()
    return xg, mid


def _attn_core_fp16(qkv, rel_pos_h, rel_pos_w, H, W, heads):
    """sam_ref.vit_attention_core in float64 with the attention kernels' fp16 storage: q * scale, the two rel-pos dot products
    (from the unscaled q) and the unnormalised probabilities exp(s - max) are rounded to fp16; the row sum is not."""
    B, L, D3 = qkv.shape
    hd = D3 // 3 // heads
    t = qkv.reshape(B, L, 3, heads, hd).permute(2, 0, 3, 1, 4).reshape(3, B * heads, L, hd)
    q, k, v = t[0], t[1], t[2]
    r16 = lambda a: a.half().double()
    s = r16(q * hd ** -0.5) @ k.transpose(-2, -1)
    Rh, Rw = sam_ref.get_rel_pos(H, H, rel_pos_h), sam_ref.get_rel_pos(W, W, rel_pos_w)
    rq = q.reshape(-1, H, W, hd)
    rel_h = r16(torch.einsum("bhwc,hkc->bhwk", rq, Rh))
    rel_w = r16(torch.einsum("bhwc,wkc->bhwk", rq, Rw))
    s = (s.view(-1, H, W, H, W) + rel_h[:, :, :, :, None] + rel_w[:, :, :, None, :]).view(-1, L, L)
    e = torch.exp(s - s.amax(-1, keepdim=True))
    o = (r16(e) @ v) / e.sum(-1, keepdim=True)
    return o.view(B, heads, L, hd).permute(0, 2, 1, 3).reshape(B, L, -1)


def _attn_half64(sd, p, x, heads, is_global, qkv_round=False, out_round=False):
    """x + proj(attention(LN1(x))) in float64 on the GPU, one frame at a time; qkv_round emulates the fp16 storage of qkv and
    of the attention kernels' operands, out_round the fp16 attention output (proj's operand at precision 1 to 3)."""
    outs = []
    for b in range(x.shape[0]):
        xb = x[b:b + 1]
        h = F.layer_norm(xb, (xb.shape[-1],), sd[p + "norm1.weight"], sd[p + "norm1.bias"], 1e-6)
        if not is_global:
            h, pad_hw = sam_ref.window_partition(h, WS)
        Bw, H, W, D = h.shape
        qkv = F.linear(h, sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"]).reshape(Bw, H * W, -1)
        if qkv_round:
            o = _attn_core_fp16(qkv.half().double(), sd[p + "attn.rel_pos_h"], sd[p + "attn.rel_pos_w"], H, W, heads)
        else:
            o = sam_ref.vit_attention_core(qkv, sd[p + "attn.rel_pos_h"], sd[p + "attn.rel_pos_w"], H, W, heads)
        if out_round:
            o = o.half().double()
        o = F.linear(o.reshape(Bw, H, W, D), sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"])
        if not is_global:
            o = sam_ref.window_unpartition(o, WS, pad_hw, (G, G))
        outs.append(xb + o)
    return torch.cat(outs)


def _mlp_half64(sd, p, x):
    y = F.layer_norm(x, (x.shape[-1],), sd[p + "norm2.weight"], sd[p + "norm2.bias"], 1e-6)
    y = F.gelu(F.linear(y, sd[p + "mlp.lin1.weight"], sd[p + "mlp.lin1.bias"]))
    return F.linear(y, sd[p + "mlp.lin2.weight"], sd[p + "mlp.lin2.bias"])


def _block_case(enc, blk, is_global, B, precision):
    D = enc.embed_dim
    g = torch.Generator().manual_seed(blk * 10 + B + D)
    x = torch.randn((B * G * G, D), generator=g)
    # a few rows per frame of variance ~1e-6, where norm1's eps moves the output by a large fraction
    for b in range(B):
        for r in (b * G * G + 3, b * G * G + 2000, b * G * G + G * G - 1):
            x[r] = 0.3 + 1e-3 * torch.randn((D,), generator=g)
    out, mid = _run_block(enc, blk, is_global, x, precision, B)
    what = f"block D{D} {'global' if is_global else 'windowed'} B{B} p{precision}"
    assert torch.isfinite(out).all() and torch.isfinite(mid).all(), what
    sd = {k: v.cuda() for k, v in _sd64(enc).items()}
    p = f"image_encoder.blocks.{blk}."
    passes, p_qkv, p_proj, att_split = _prec(precision)
    f8 = precision == 6
    # MLP half, from the kernel's own x_mid
    m64 = mid.double().view(B, G, G, D)
    delta = _mlp_half64(sd, p, m64).reshape(-1, D)
    err = out.double() - (mid.double() + delta)
    bar = REL_F8 if f8 else (REL_3PASS_MLP if passes == 3 else REL_F16)
    r_mlp = ((err.pow(2).mean().sqrt() - 2 * U * out.double().pow(2).mean().sqrt()) / delta.pow(2).mean().sqrt()).item()
    print(f"{what}: MLP half relative rms {r_mlp:.3e} (bar {bar:.3e})")
    assert r_mlp <= bar, (what, r_mlp, bar)
    # attention half: the fp16 storage of qkv is the floor
    x64 = x.double().cuda().view(B, G, G, D)
    ref = _attn_half64(sd, p, x64, enc.num_heads, is_global).reshape(-1, D)
    emu = _attn_half64(sd, p, x64, enc.num_heads, is_global, qkv_round=True, out_round=not att_split).reshape(-1, D)
    d_attn = (ref - x64.reshape(-1, D)).pow(2).mean().sqrt()
    e_emu = (emu - ref).pow(2).mean().sqrt()
    gemm = (_rel_gemm(p_qkv, f8) + _rel_gemm(p_proj, f8)) * d_attn
    e = (mid.double() - ref).pow(2).mean().sqrt()
    ratio = ((e - gemm) / e_emu).item()
    print(f"{what}: attention half rms {e.item():.3e}, fp16-qkv emulation {e_emu.item():.3e}, ratio after GEMM terms {ratio:.3f}")
    assert e <= 2 * e_emu + gemm, (what, ratio)


@pytest.mark.parametrize("precision", [1, 2, 3, 4, 5, 6])
@pytest.mark.parametrize("is_global,B", [(0, 1), (0, 2), (1, 1), (1, 2)])
def test_block_vit_h(vit_h, is_global, B, precision):
    """ViT-H (1280 wide, 16 heads of 80): windowed block 0 (S = 14, 25 windows of which 9 hold padding) and global block 1
    (S = 64)."""
    _block_case(vit_h, is_global, bool(is_global), B, precision)


@pytest.mark.parametrize("precision", [1, 4, 6])
@pytest.mark.parametrize("is_global,B", [(0, 2), (1, 2)])
def test_block_vit_b(vit_b, is_global, B, precision):
    """ViT-B (768 wide, 12 heads of 64)."""
    _block_case(vit_b, is_global, bool(is_global), B, precision)


@pytest.mark.parametrize("precision", [3, 6])
def test_block_live_only(vit_h, precision):
    """The padding-window skip's compacted block for 576x1024 frames (3 x 5 live windows, tokens y < 42): live rows equal the
    full block's bit for bit, every other row keeps its old bits."""
    B, D = 2, 1280
    g = torch.Generator().manual_seed(99)
    x = torch.randn((B * G * G, D), generator=g)
    full, _ = _run_block(vit_h, 0, 0, x, precision, B, want_mid=False)
    live, _ = _run_block(vit_h, 0, 0, x, precision, B, 576, 1024, live_only=1, want_mid=False)
    tok = torch.arange(B * G * G)
    is_live = ((tok % (G * G)) // G) < 42
    assert torch.equal(live[is_live.cuda()], full[is_live.cuda()])
    assert torch.equal(live[~is_live.cuda()].cpu(), x[~is_live])


# ---------------------------------------------------------------------------------------------------------------- neck
def _neck64(sd, x, B, D):
    p = "image_encoder."
    h = x.view(B, G, G, D).permute(0, 3, 1, 2)
    h = F.conv2d(h, sd[p + "neck.0.weight"])
    h = sam_ref._ln2d(h, sd[p + "neck.1.weight"], sd[p + "neck.1.bias"])
    h = F.conv2d(h, sd[p + "neck.2.weight"], padding=1)
    return sam_ref._ln2d(h, sd[p + "neck.3.weight"], sd[p + "neck.3.bias"])


@pytest.mark.parametrize("precision", [1, 6])
@pytest.mark.parametrize("B", [1, 2, 3])
@pytest.mark.parametrize("D", [768, 1280])
def test_neck(vit_b, vit_h, D, B, precision):
    """conv1x1 -> LayerNorm2d -> conv3x3 (pad 1) -> LayerNorm2d in NCHW.  Both LayerNorms divide by the channel std, so the
    relative rms of the GEMMs carries through; rows and columns 0 and 63 (where the 3x3 taps reach the zero padding) are held
    apart from the interior."""
    enc = vit_b if D == 768 else vit_h
    n = _n()
    ctx = _ctx(enc, precision, B)
    g = torch.Generator().manual_seed(D + B)
    x = torch.randn((B * G * G, D), generator=g) * 2
    xg = x.cuda()
    out = torch.full((B, 256, G, G), float("nan"), device="cuda")
    n.check(n.lib().sampt_test_vit_neck(ctx.handle, n.ptr(xg), c_int(B), c_int(D), c_int(1024), c_int(P), c_int(256),
                                        c_int(precision), n.ptr(out), n.stream_ptr()), "vit_neck")
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    sd = {k: v.cuda() for k, v in _sd64(enc).items()}
    ref = _neck64(sd, x.double().cuda(), B, D)
    err = out.double() - ref
    bar = _rel_gemm(min(precision, 3))
    border = torch.zeros((G, G), dtype=torch.bool, device="cuda")
    border[0, :] = border[-1, :] = border[:, 0] = border[:, -1] = True
    for name, sel in (("border", border), ("interior", ~border)):
        r = _rel_rms(err[:, :, sel], ref[:, :, sel])
        print(f"neck D{D} B{B} p{precision} {name}: relative rms {r:.3e} (bar {bar:.3e})")
        assert r <= bar, (name, r, bar)


# ------------------------------------------------------------------------------------------------ padding-window skip
SKIP_D, SKIP_HEADS, SKIP_DEPTH, SKIP_GLOBALS = 1280, 16, 3, (2,)


@pytest.fixture(scope="module")
def skip_preds():
    """SamPredictors of a SAM and an HQ-SAM encoder of equal shapes (ViT-H width, depth 3, first global block 2)"""
    from segment_anything.modeling.mask_decoder import MaskDecoder
    from segment_anything.modeling.prompt_encoder import PromptEncoder
    from segment_anything.modeling.sam import Sam
    from segment_anything.modeling.transformer import TwoWayTransformer
    from segment_anything.predictor import SamPredictor
    preds = []
    for seed, hq in ((11, False), (12, True)):
        enc = _encoder(SKIP_D, SKIP_HEADS, SKIP_DEPTH, SKIP_GLOBALS, seed=seed, hq=hq)
        enc.precision = 6
        pe = PromptEncoder(embed_dim=256, image_embedding_size=(64, 64), input_image_size=(1024, 1024), mask_in_chans=16)
        md = MaskDecoder(num_multimask_outputs=3, transformer=TwoWayTransformer(depth=2, embedding_dim=256, mlp_dim=2048, num_heads=8),
                         transformer_dim=256, iou_head_depth=3, iou_head_hidden_dim=256)
        preds.append(SamPredictor(Sam(enc, pe, md).cuda()))
    return preds


def _encode(pred, frames):
    f, i = pred.encode_frames(frames.cuda(), want_interm=True)
    torch.cuda.synchronize()
    return f.clone(), i.clone()


def _forward_float(pred, frames):
    """upstream ImageEncoderViT.forward on Sam.preprocess of the same resized frames (a path that never skips)"""
    x = _preprocess(pred.resize_frames_u8(frames.cuda()).cpu()).cuda()
    f = pred.model.image_encoder(x)
    torch.cuda.synchronize()
    return f


# original frame sizes -> resized: 480x854 -> 576x1024, 854x480 -> 1024x576, 720x480 -> 1024x683 and 480x720 -> 683x1024 (a
# partial last patch column / row)
@pytest.mark.parametrize("H,W", [(480, 854), (854, 480), (720, 480), (480, 720)])
def test_skip_pad_bitwise(skip_preds, H, W):
    """SamPredictor.encode_frames: the first encode of a shape runs in full and saves the padding rows; the second runs
    compacted.  Both agree bit for bit, at B = 3 and then frame by frame, features and interm, and equal forward(float) of
    the same preprocessed image."""
    pred = skip_preds[0]
    frames = _frames(3, H, W, H + W)
    f0, i0 = _encode(pred, frames)          # full (a shape not seen before on this context)
    f1, i1 = _encode(pred, frames)          # compacted
    assert torch.equal(f0, f1) and torch.equal(i0, i1)
    for b in range(3):
        fb, ib = _encode(pred, frames[b:b + 1])
        assert torch.equal(fb[0], f0[b]) and torch.equal(ib[0], i0[b]), b
    assert torch.equal(_forward_float(pred, frames), f1)


def test_skip_pad_weight_change_and_alternation(skip_preds):
    """An in-place weight change re-registers the weights and drops the saved rows: the next encodes (full, then compacted)
    match forward(float) of the new weights.  A SAM and an HQ-SAM encoder of equal shapes alternating on one context each match
    their own forward(float)."""
    sam, hq = skip_preds
    frames = _frames(2, 480, 854, 3)
    _encode(sam, frames)
    _encode(sam, frames)
    with torch.no_grad():
        getattr(sam.model.image_encoder.blocks, "0").mlp.lin1.weight.mul_(1.25)
    for _ in range(2):
        f, _ = _encode(sam, frames)
        assert torch.equal(f, _forward_float(sam, frames))
    for _ in range(2):
        for p in (sam, hq):
            f, _ = _encode(p, frames)
            assert torch.equal(f, _forward_float(p, frames))


def test_skip_pad_square_frame_saves_nothing(skip_preds):
    """A square frame has no padding windows: no rows are saved and the second call launches what the first did."""
    pred = skip_preds[0]
    n = _n()
    frames = _frames(1, 1024, 1024, 8)
    ctx = pred.model.image_encoder.native_context()
    counts = []
    for _ in range(2):
        c0 = n.lib().sampt_launch_count(ctx.handle)
        _encode(pred, frames)
        counts.append(n.lib().sampt_launch_count(ctx.handle) - c0)
    assert counts[0] == counts[1], counts
