"""GPU: tensor-core flash-attention kernel (pre-extended operands) against a float64 softmax(QK^T)V reference."""
from ctypes import c_int

import pytest
import torch

pytestmark = pytest.mark.gpu


def _run(Q, K, V, Lk, NT, nheads, HD, ld_pad=0, nan_pad=False):
    """Q (BH,Lq,DK) K (BH,Lk,DK) V (BH,Lk,HD) fp32 cpu -> out (B*Lq, nheads*HD + ld_pad) fp16.  The columns past nheads*HD
    start as a sentinel; nan_pad: V^T's row padding (keys in [Lk, Lkp)) holds NaN instead of zeros."""
    from sampt_b200 import native
    ctx = native.get_context("cuda")
    BH, Lq, DK = Q.shape
    Lkp = ((Lk + 63) // 64) * 64
    Vt = torch.full((BH, HD, Lkp), float("nan") if nan_pad else 0.0, dtype=torch.float16)
    Vt[:, :, :Lk] = V.transpose(1, 2).half()
    Qd, Kd, Vd = Q.half().cuda().contiguous(), K.half().cuda().contiguous(), Vt.cuda().contiguous()
    B = BH // nheads
    ld_out = nheads * HD + ld_pad
    out = torch.full((B * Lq, ld_out), -3.5, dtype=torch.float16, device="cuda")
    native.check(native.lib().sampt_attention_f16(
        ctx.handle, native.ptr(Qd), native.ptr(Kd), native.ptr(Vd), c_int(BH), c_int(Lq), c_int(Lk), c_int(Lkp), c_int(DK),
        c_int(HD), c_int(NT), c_int(nheads), native.ptr(out), c_int(ld_out), c_int(0), native.stream_ptr()), "attention")
    torch.cuda.synchronize()
    out = out.cpu()
    assert torch.equal(out[:, nheads * HD:], torch.full_like(out[:, nheads * HD:], -3.5))   # nothing written past the heads
    return out[:, :nheads * HD]


def _ref(Q, K, V, nheads):
    Qh, Kh, Vh = Q.half().double().cuda(), K.half().double().cuda(), V.half().double().cuda()
    P = torch.softmax(Qh @ Kh.transpose(1, 2), dim=-1)
    O = P @ Vh  # (BH, Lq, HD)
    BH, Lq, HD = O.shape
    return O.view(BH // nheads, nheads, Lq, HD).permute(0, 2, 1, 3).reshape(-1, nheads * HD).cpu()


_ROWS = [
    (4, 196, 196, 128, 80, 208, 2),     # SAM ViT-H windowed block: 14x14 window, hd 80 (+28 rel-pos dims -> 128)
    (3, 196, 196, 128, 64, 208, 3),     # ViT-B windowed (hd 64)
    (2, 512, 512, 256, 80, 128, 2),     # global-style multi-tile online softmax (ViT-H: 80+128 -> 256)
    (2, 300, 260, 192, 64, 128, 1),     # ragged sizes, ViT-B global DK=192
    (1, 64, 64, 64, 64, 64, 1),
    # head dims off the 64 / 80 templates and on the 96 / 128 ones
    (2, 130, 130, 64, 16, 64, 2), (2, 200, 150, 64, 48, 64, 1), (2, 130, 196, 128, 96, 64, 2), (2, 64, 100, 128, 112, 64, 1),
    (1, 256, 256, 128, 128, 64, 1),
    # key counts around one 64-key tile
    (2, 100, 1, 64, 64, 64, 2), (2, 100, 63, 64, 64, 64, 2), (2, 100, 64, 64, 64, 64, 2), (2, 100, 65, 64, 64, 64, 2),
    (1, 4096, 4096, 256, 80, 64, 1),    # ViT-H global block: 64 key tiles of online softmax
    # extras: ld_pad = unused output columns past the heads; last_max = logits rising from -30 to +30 over the keys, so every
    # row's maximum is in the last tile and each tile rescales the running output; nan_pad = NaN in V^T's row padding
    (4, 196, 196, 128, 80, 64, 2, "ld_pad"), (2, 100, 65, 64, 48, 64, 2, "ld_pad"),
    (2, 256, 1000, 128, 64, 64, 1, "last_max"), (2, 128, 4096, 256, 80, 64, 2, "last_max"),
    (2, 100, 65, 64, 64, 64, 2, "nan_pad"), (3, 196, 196, 128, 80, 208, 3, "nan_pad"),
]


@pytest.mark.parametrize("BH,Lq,Lk,DK,HD,NT,nheads,extra", [r + ("",) * (8 - len(r)) for r in _ROWS],
                         ids=["-".join(str(v) for v in r) for r in _ROWS])
def test_attention_matches_reference(BH, Lq, Lk, DK, HD, NT, nheads, extra):
    g = torch.Generator().manual_seed(BH * 1000 + Lq + DK)
    Q = torch.randn((BH, Lq, DK), generator=g) * 0.5
    K = torch.randn((BH, Lk, DK), generator=g) * 0.5
    V = torch.randn((BH, Lk, HD), generator=g)
    if extra == "last_max":
        Q, K = Q * 0.02, K * 0.02
        Q[:, :, -1] = 1.0
        K[:, :, -1] = torch.linspace(-30.0, 30.0, Lk)
        logits = Q.half().double() @ K.half().double().transpose(1, 2)
        assert (logits.argmax(-1) >= ((Lk - 1) // 64) * 64).all()
    out = _run(Q, K, V, Lk, NT, nheads, HD, ld_pad=64 if extra == "ld_pad" else 0, nan_pad=extra == "nan_pad")
    ref = _ref(Q, K, V, nheads)
    err = (out.double() - ref).abs().max().item()
    assert err < 4e-3, err  # fp16 P and fp16 output rounding
