"""GPU: tensor-core flash-attention kernel (pre-extended operands) against a float64 softmax(QK^T)V reference."""
from ctypes import c_int

import pytest
import torch

pytestmark = pytest.mark.gpu


def _run(Q, K, V, Lk, NT, nheads, HD):
    """Q (BH,Lq,DK) K (BH,Lk,DK) V (BH,Lk,HD) fp32 cpu -> out (B*Lq, nheads*HD) fp16."""
    from sampt_b200 import native
    ctx = native.get_context("cuda")
    BH, Lq, DK = Q.shape
    Lkp = ((Lk + 63) // 64) * 64
    Vt = torch.zeros((BH, HD, Lkp), dtype=torch.float16)
    Vt[:, :, :Lk] = V.transpose(1, 2).half()
    Qd, Kd, Vd = Q.half().cuda().contiguous(), K.half().cuda().contiguous(), Vt.cuda().contiguous()
    B = BH // nheads
    out = torch.zeros((B * Lq, nheads * HD), dtype=torch.float16, device="cuda")
    native.check(native.lib().sampt_attention_f16(
        ctx.handle, native.ptr(Qd), native.ptr(Kd), native.ptr(Vd), c_int(BH), c_int(Lq), c_int(Lk), c_int(Lkp), c_int(DK),
        c_int(HD), c_int(NT), c_int(nheads), native.ptr(out), c_int(nheads * HD), c_int(0), native.stream_ptr()), "attention")
    torch.cuda.synchronize()
    return out.cpu()


def _ref(Q, K, V, nheads):
    Qh, Kh, Vh = Q.half().double(), K.half().double(), V.half().double()
    P = torch.softmax(Qh @ Kh.transpose(1, 2), dim=-1)
    O = P @ Vh  # (BH, Lq, HD)
    BH, Lq, HD = O.shape
    return O.view(BH // nheads, nheads, Lq, HD).permute(0, 2, 1, 3).reshape(-1, nheads * HD)


@pytest.mark.parametrize("BH,Lq,Lk,DK,HD,NT,nheads", [
    (4, 196, 196, 128, 80, 208, 2),     # SAM ViT-H windowed block: 14x14 window, hd 80 (+28 rel-pos dims -> 128)
    (3, 196, 196, 128, 64, 208, 3),     # ViT-B windowed (hd 64)
    (2, 512, 512, 256, 80, 128, 2),     # global-style multi-tile online softmax (ViT-H: 80+128 -> 256)
    (2, 300, 260, 192, 64, 128, 1),     # ragged sizes, ViT-B global DK=192
    (1, 64, 64, 64, 64, 64, 1),
])
def test_attention_matches_reference(BH, Lq, Lk, DK, HD, NT, nheads):
    g = torch.Generator().manual_seed(BH * 1000 + Lq + DK)
    Q = torch.randn((BH, Lq, DK), generator=g) * 0.5
    K = torch.randn((BH, Lk, DK), generator=g) * 0.5
    V = torch.randn((BH, Lk, HD), generator=g)
    out = _run(Q, K, V, Lk, NT, nheads, HD)
    ref = _ref(Q, K, V, nheads)
    err = (out.double() - ref).abs().max().item()
    assert err < 4e-3, err  # fp16 P and fp16 output rounding
