"""GPU: one ViT attention block between its qkv GEMM and proj -- operand preparation (rel-pos folding) + the attention kernel,
include/sampt_b200.h: sampt_test_vit_attention -- against float64.

Checked separately: the operands the preparation builds (Q' = [fp16(q scale) | rel_h | rel_w | 0], K' = [k | onehot(ky) |
onehot(kx) | 0], V^T), the result over those operands, and the result against the oracle's restatement of upstream Attention +
add_decomposed_rel_pos (oracle.sam_ref.vit_attention_core)."""
from ctypes import c_int

import pytest
import torch

from oracle.sam_ref import vit_attention_core

pytestmark = pytest.mark.gpu

_U = 2.0 ** -11   # unit roundoff of fp16


def _dims(S, D, nheads):
    """vit_pipeline.cu: head dim, K dimension of Q'K'^T, V^T row pitch (windowed rows are padded to whole 64-key tiles)"""
    HD, L = D // nheads, S * S
    return HD, ((HD + 2 * S + 63) // 64) * 64, L if L > 256 else ((L + 63) // 64) * 64


def _inputs(nwb, S, D, nheads, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    HD = D // nheads
    qkv = torch.randn((nwb * S * S, 3 * D), generator=g, device="cuda").half()
    rph = torch.randn((2 * S - 1, HD), generator=g, device="cuda") * 0.25
    rpw = torch.randn((2 * S - 1, HD), generator=g, device="cuda") * 0.25
    return qkv, rph, rpw


def _run(qkv, rph, rpw, nwb, nheads, S, D, split_off=0, out_f8=0):
    """operands and output buffers start as NaN: whatever the call does not write stays NaN"""
    from sampt_b200 import native
    ctx = native.get_context("cuda")
    HD, DK, Lkp = _dims(S, D, nheads)
    BH, L = nwb * nheads, S * S
    nan = float("nan")
    Qx = torch.full((BH, L, DK), nan, device="cuda", dtype=torch.float16)
    Kx = torch.full((BH, L, DK), nan, device="cuda", dtype=torch.float16)
    Vt = torch.full((BH, HD, Lkp), nan, device="cuda", dtype=torch.float16)
    ld_out = 2 * D if split_off else D
    out = torch.full((nwb * L, ld_out), nan, device="cuda", dtype=torch.float16)
    native.check(native.lib().sampt_test_vit_attention(
        ctx.handle, native.ptr(qkv), native.ptr(rph), native.ptr(rpw), c_int(nwb), c_int(nheads), c_int(S), c_int(D), c_int(DK),
        c_int(Lkp), native.ptr(Qx), native.ptr(Kx), native.ptr(Vt), native.ptr(out), c_int(ld_out), c_int(split_off), c_int(out_f8),
        native.stream_ptr()), "test_vit_attention")
    torch.cuda.synchronize()
    return Qx, Kx, Vt, out


def _heads(qkv, nwb, S, nheads):
    """qkv rows (wb, t) -> q, k, v as [nwb * nheads, L, HD] (bh = wb * nheads + h)"""
    L = S * S
    x = qkv.view(nwb, L, 3, nheads, -1).permute(2, 0, 3, 1, 4)
    return [t.reshape(nwb * nheads, L, -1) for t in x.unbind(0)]


def _fp16_ulp(x):
    e = torch.floor(torch.log2(x.abs().clamp(min=2.0 ** -14)))
    return torch.pow(2.0, e - 10)


def _report(what, err, bound):
    worst = (err / bound).max().item()
    print(f"{what}: max err {err.max().item():.3g}, worst err / bound {worst:.3g}")
    assert worst <= 1.0, (what, worst)


# windowed blocks: S = 14, one (25 windows) or two (50) 1024^2 frames and an odd count; global blocks: S = 64, frames 1-3 (the
# persistent preparation kernel's items then divide unevenly over the SMs).  D / heads: ViT-B (768 / 12, HD 64),
# ViT-L (1024 / 16, HD 64), ViT-H (1280 / 16, HD 80).
_CASES = [(S, nwb, D, nh) for S, nwbs in ((14, (25, 50, 7)), (64, (1, 2, 3))) for D, nh in ((768, 12), (1280, 16)) for nwb in nwbs] + [
    (14, 25, 1024, 16), (64, 1, 1024, 16)]


@pytest.mark.parametrize("S,nwb,D,nheads", _CASES)
def test_vit_attention_operands(S, nwb, D, nheads):
    """K' bit-exact, V^T = v^T bit-exact, Q' = fp16(q scale) bit-exact and its rel-pos columns within one fp16 ulp of the
    float64 products q . R[qy - j + S - 1] (plus 2^-20 sum |q| |R| for their fp32 accumulation, which matters only where the
    product cancels) -- and correctly rounded for at least 99% of them: the table is carried as fp16 hi + lo, ~2^-22
    accurate, so only values that close to a rounding boundary may round the other way (with the hi half alone, ~2^-12
    accurate, a large share would)"""
    qkv, rph, rpw = _inputs(nwb, S, D, nheads, seed=S * 100 + nwb + D)
    Qx, Kx, Vt, _ = _run(qkv, rph, rpw, nwb, nheads, S, D)
    HD, DK, Lkp = _dims(S, D, nheads)
    L = S * S
    q, k, v = _heads(qkv, nwb, S, nheads)
    t = torch.arange(L, device="cuda")
    ty, tx = t // S, t % S
    kext = torch.zeros((L, DK - HD), device="cuda", dtype=torch.float16)
    kext[t, ty] = 1.0
    kext[t, S + tx] = 1.0
    kexp = torch.cat([k, kext.expand(k.shape[0], L, DK - HD)], dim=2)
    assert torch.equal(Kx.view(torch.int16), kexp.view(torch.int16))
    assert torch.equal(Vt[:, :, :L].view(torch.int16), v.transpose(1, 2).contiguous().view(torch.int16))
    scale = torch.tensor(1.0, dtype=torch.float32) / torch.sqrt(torch.tensor(float(HD), dtype=torch.float32))
    assert torch.equal(Qx[:, :, :HD].view(torch.int16), (q.float() * scale.cuda()).half().view(torch.int16))
    assert torch.equal(Qx[:, :, HD + 2 * S:], torch.zeros_like(Qx[:, :, HD + 2 * S:]))
    j = torch.arange(S, device="cuda")
    for name, R, pos, c0 in (("rel_h", rph, ty, HD), ("rel_w", rpw, tx, HD + S)):
        idx = (pos[:, None] - j[None, :] + S - 1).expand(q.shape[0], L, S)
        exp = torch.gather(q.double() @ R.double().T, 2, idx)          # [BH, L, S] of [BH, L, 2S-1]
        mag = torch.gather(q.double().abs() @ R.double().abs().T, 2, idx)
        got = Qx[:, :, c0: c0 + S].double()
        exact = (got == exp.half().double()).double().mean().item()
        print(f"{name} S={S} nwb={nwb} HD={HD}: correctly rounded fraction {exact:.5f}")
        _report(f"{name} S={S} nwb={nwb} HD={HD}", (got - exp).abs(), _fp16_ulp(exp) + 2.0 ** -20 * mag)
        assert exact >= 0.99, exact


def _expected(qkv, rph, rpw, nwb, nheads, S, D, Qx, Kx, Vt):
    """float64: the oracle's result, the exact attention over the kernel's own operands, and the two bounds (see below)"""
    HD, DK, Lkp = _dims(S, D, nheads)
    L = S * S
    chunk = max(1, (1 << 26) // (L * L))          # heads per float64 block of logits
    core, o2, tol_k, tol_c = [], [], [], []
    fchunk = max(1, chunk // nheads)
    for f0 in range(0, nwb, fchunk):
        f1 = min(nwb, f0 + fchunk)
        x = qkv[f0 * L: f1 * L].double().view(f1 - f0, L, 3 * D)
        core.append(vit_attention_core(x, rph.double(), rpw.double(), S, S, nheads).reshape(-1, D))
    for b0 in range(0, nwb * nheads, chunk):
        b1 = min(nwb * nheads, b0 + chunk)
        Q2, K2 = Qx[b0:b1].double(), Kx[b0:b1].double()
        V = Vt[b0:b1, :, :L].double().transpose(1, 2)
        P = torch.softmax(Q2 @ K2.transpose(1, 2), dim=-1)
        o = P @ V
        pv = P @ V.abs()
        # kernel over its operands: P rounded to fp16 (each weight relative 2^-11, normalised by the unrounded fp32 sum), the
        # fp16 output rounding, and a 2^-20 allowance for ex2.approx and fp32 accumulation
        tk = 1.05 * _U * (pv + o.abs()) + 2.0 ** -20 * pv + 2.0 ** -24
        # operand roundings: every Q' entry is fp16 (relative 2^-11; K' is exact), so logit j moves by at most
        # E_j = 2^-11 sum_c |Q'_c K'_jc| (+ 2^-16 for the fp32 rel-pos products); to first order the output moves by
        # sum_j P_j |E_j - sum_k P_k E_k| |v_j| <= (P o E) |V| + (P . E) (P |V|)
        E = 1.05 * _U * (Q2.abs() @ K2.abs().transpose(1, 2)) + 2.0 ** -16
        tc = (P * E) @ V.abs() + (P * E).sum(-1, keepdim=True) * pv + tk
        del P, E, Q2, K2
        o2.append(o)
        tol_k.append(tk)
        tol_c.append(tc)
    rows = lambda lst: torch.cat(lst).view(nwb, nheads, L, HD).permute(0, 2, 1, 3).reshape(-1, D)   # bh -> (wb, t) rows
    return torch.cat(core), rows(o2), rows(tol_k), rows(tol_c)


@pytest.mark.parametrize("S,nwb,D,nheads", _CASES)
def test_vit_attention_matches_oracle(S, nwb, D, nheads):
    qkv, rph, rpw = _inputs(nwb, S, D, nheads, seed=S * 100 + nwb + D)
    Qx, Kx, Vt, out = _run(qkv, rph, rpw, nwb, nheads, S, D)
    assert torch.isfinite(out).all()   # V^T's row padding [S*S, Lkp) started as NaN and must not reach the output
    core, o2, tol_k, tol_c = _expected(qkv, rph, rpw, nwb, nheads, S, D, Qx, Kx, Vt)
    _report(f"S={S} nwb={nwb} D={D}: vs float64 over the kernel's operands", (out.double() - o2).abs(), tol_k)
    _report(f"S={S} nwb={nwb} D={D}: vs vit_attention_core", (out.double() - core).abs(), tol_c)


def _ordinal(b):
    """e4m3 byte -> signed position on the e4m3 number line (+0 and -0 both 0)"""
    m = (b & 0x7F).int()
    return torch.where((b & 0x80) != 0, -m, m)


@pytest.mark.parametrize("S,nwb,D,nheads", [(14, 7, 1280, 16), (64, 2, 768, 12)])
def test_vit_attention_split_and_f8_outputs(S, nwb, D, nheads):
    """the A operand of proj: hi | lo fp16 (precision 5) and hi | e4m3 bytes (precision 6), from the same inputs"""
    qkv, rph, rpw = _inputs(nwb, S, D, nheads, seed=S * 100 + nwb + D + 1)
    Qx, Kx, Vt, out = _run(qkv, rph, rpw, nwb, nheads, S, D)
    _, _, _, outs = _run(qkv, rph, rpw, nwb, nheads, S, D, split_off=D)
    _, _, _, out8 = _run(qkv, rph, rpw, nwb, nheads, S, D, split_off=D, out_f8=1)
    hi, lo = outs[:, :D], outs[:, D:]
    assert torch.equal(hi.view(torch.int16), out.view(torch.int16))
    assert torch.equal(out8[:, :D].view(torch.int16), out.view(torch.int16))
    _, o2, tol_k, _ = _expected(qkv, rph, rpw, nwb, nheads, S, D, Qx, Kx, Vt)
    rec = hi.double() + lo.double()
    # hi + lo is the fp32 result to 2^-22: only the P rounding remains of tol_k
    tol_rec = tol_k - 1.05 * _U * o2.abs() + 2.0 ** -21 * o2.abs()
    _report(f"S={S} nwb={nwb}: hi + lo vs float64 over the kernel's operands", (rec - o2).abs(), tol_rec)
    e_rec, e_hi = (rec - o2).pow(2).mean().sqrt().item(), (hi.double() - o2).pow(2).mean().sqrt().item()
    print(f"rms error hi + lo {e_rec:.3g}, hi alone {e_hi:.3g}")
    assert e_rec < e_hi, (e_rec, e_hi)
    # e4m3 blocks: e4m3((hi + lo - hi) 2^12) at byte 2 D + col, e4m3((hi + lo) 2^-3) at byte 3 D + col, within one code
    raw = out8.view(torch.uint8)
    lo8, hi8 = raw[:, 2 * D: 3 * D], raw[:, 3 * D: 4 * D]
    e4 = lambda t: t.float().clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8)
    d_lo = (_ordinal(lo8) - _ordinal(e4(lo.double() * 4096.0))).abs().max().item()
    d_hi = (_ordinal(hi8) - _ordinal(e4(rec * 0.125))).abs().max().item()
    print(f"e4m3 code distance: lo block {d_lo}, hi block {d_hi}")
    assert d_lo <= 1 and d_hi <= 1, (d_lo, d_hi)
