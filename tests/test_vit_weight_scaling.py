"""CPU: the fp16 weight operands ImageEncoderViT registers for csrc/vit_pipeline.cu.  Each GEMM weight is stored as w 2^s (fp16
hi | lo) with the scale 2^-s next to it, so that (hi + lo) 2^-s restores w to 2^-22 |w|.  Unscaled, weights of size ~1/sqrt(K) --
every ViT linear and conv -- have fp16-subnormal lo halves, which restore w only to 2^-25 absolute: 3x to 30x worse."""
import math

import pytest
import torch


def _enc(precision, D=256, heads=2, depth=2):
    from segment_anything.modeling.image_encoder import ImageEncoderViT
    enc = ImageEncoderViT(embed_dim=D, depth=depth, num_heads=heads, use_rel_pos=True, window_size=14, global_attn_indexes=(1,))
    enc.precision = precision
    return enc


@pytest.mark.parametrize("K", [768, 1280, 2304, 5120])
def test_w16_restores_weights_to_2pow_minus22(K):
    """ViT-like weights (uniform with bound 1/sqrt(K), as torch's default init) and a few tiny ones."""
    from segment_anything.modeling.image_encoder import ImageEncoderViT
    g = torch.Generator().manual_seed(K)
    w = (torch.rand((64, K), generator=g) * 2 - 1) / math.sqrt(K)
    w[0, :8] = 1e-6 * torch.randn((8,), generator=g)
    w16, scale = ImageEncoderViT._w16(w, True)
    assert w16.dtype == torch.float16 and w16.shape == (64, 2 * K)
    s = scale.item()
    assert s == 2.0 ** round(math.log2(s))                               # a power of two: the epilogue's multiply is exact
    assert 2.0 ** 14 <= w.abs().max().item() / s < 2.0 ** 15
    v = (w16[:, :K].double() + w16[:, K:].double()) * s
    err = (v - w.double()).abs()
    assert (err <= 2.0 ** -22 * w.double().abs() + 2.0 ** -40).all(), (err / w.double().abs()).max().item()
    hi, sc1 = ImageEncoderViT._w16(w, False)
    assert sc1.item() == s and torch.equal(hi, w16[:, :K])


@pytest.mark.parametrize("precision", [1, 3, 6])
def test_every_w16_has_its_scale(precision):
    """Every ".w16" the encoder registers has a ".w16s" = 2^-s next to it that restores the weight, for the patch embedding,
    the four linears of every block and both neck convs."""
    enc = _enc(precision)
    t = enc.native_weights()
    names = sorted(k[:-len(".w16")] for k in t if k.endswith(".w16"))
    want = ["patch_embed", "neck.0", "neck.2"] + [f"blocks.{i}.{n}" for i in range(enc.depth)
                                                  for n in ("attn.qkv", "attn.proj", "mlp.lin1", "mlp.lin2")]
    assert names == sorted(want)
    sd = enc.state_dict()
    D, C = enc.embed_dim, enc.out_chans
    ref = {"patch_embed": sd["patch_embed.proj.weight"].reshape(D, -1), "neck.0": sd["neck.0.weight"].reshape(C, D),
           "neck.2": sd["neck.2.weight"].permute(0, 2, 3, 1).reshape(C, 9 * C)}
    for n in names:
        w = ref[n] if n in ref else sd[n + ".weight"]
        K = w.shape[1]
        w16, s = t[n + ".w16"], t[n + ".w16s"]
        assert s.dtype == torch.float32 and s.shape == (1,)
        v = w16[:, :K].double() + (w16[:, K:].double() if precision >= 2 else 0)
        v = v * s.item()
        rel = 2.0 ** -22 if precision >= 2 else 2.0 ** -11
        assert ((v - w.double()).abs() <= rel * w.double().abs() + 2.0 ** -40).all(), n
        assert w16.shape[1] == (2 * K if precision >= 2 else K), n
    assert all((k + "s") in t for k in t if k.endswith(".w8"))
    assert any(k.endswith(".w8") for k in t) == (precision == 6)
