"""CPU: structural pins of the TinyViT-5M restatement (oracle/tinyvit_ref.py) and of the drop-in module's state dict
(mobile_sam/modeling/tiny_vit_sam.py): key set and shapes, parameter counts, the attention-bias indexing, float32 against
float64, and the size of a whole MobileSAM checkpoint."""
import math

import pytest
import torch

from oracle import tinyvit_ref


def _shapes():
    from mobile_sam.modeling.tiny_vit_sam import state_dict_shapes
    return state_dict_shapes()


def test_state_dict_keys_and_shapes():
    from mobile_sam.modeling.tiny_vit_sam import TinyViT
    from sampt_b200 import factory
    s = _shapes()
    assert len(s) == 302
    m = TinyViT(**factory.TINY_VIT_CFG)
    sd = m.state_dict()
    assert set(sd) == set(s)
    assert all(tuple(sd[k].shape) == tuple(v) for k, v in s.items())
    assert s["layers.1.blocks.0.attn.attention_biases"] == (4, 49)
    assert s["layers.2.blocks.5.attn.attention_biases"] == (5, 196)
    assert s["layers.3.blocks.1.attn.qkv.weight"] == (960, 320)
    assert s["layers.2.downsample.conv2.c.weight"] == (320, 1, 3, 3)
    assert "attention_bias_idxs" not in " ".join(s)   # non-persistent buffer upstream
    # BatchNorm running statistics are buffers, as in torch
    bufs = {k for k, _ in m.named_buffers()}
    assert bufs == {k for k in s if k.endswith((".running_mean", ".running_var", ".num_batches_tracked"))}


def test_parameter_count():
    from mobile_sam.modeling.tiny_vit_sam import TinyViT
    from sampt_b200 import factory
    m = TinyViT(**factory.TINY_VIT_CFG)
    n = sum(p.numel() for p in m.parameters())
    head = sum(p.numel() for k, p in m.named_parameters() if k.startswith(("head.", "norm_head.")))
    assert n == 6_065_532
    assert head == 321_640
    assert n - head == 5_743_892


@pytest.mark.parametrize("ws", [7, 14])
def test_bias_index_rule(ws):
    """attention_biases[h, |dr|*ws + |dc|] is what upstream's offset dict gathers."""
    idx = tinyvit_ref.attention_bias_idxs(ws)
    L = ws * ws
    r = torch.arange(L) // ws
    c = torch.arange(L) % ws
    closed = (r[:, None] - r[None, :]).abs() * ws + (c[:, None] - c[None, :]).abs()
    assert torch.equal(idx, closed)


def test_unsupported_architecture_raises():
    from mobile_sam.modeling import TinyViT
    from sampt_b200 import factory
    cfg = dict(factory.TINY_VIT_CFG, embed_dims=[96, 192, 384, 576])
    with pytest.raises(NotImplementedError):
        TinyViT(**cfg)
    with pytest.raises(NotImplementedError):
        TinyViT(**dict(factory.TINY_VIT_CFG, img_size=224))


def test_float32_agrees_with_float64():
    """Whole encoder on one seeded image.  Bound: float32 rounding errors of a length-K dot product grow like u sqrt(K) with
    u = 2^-24 (random-walk accumulation of independent roundings; the worst case K u is ~50x looser), and the restatement chains
    about 40 such layers, the longest sum being the neck's K = 2304, on unit-scale (LayerNorm2d) outputs: u sqrt(2304) * 40 =
    1.1e-4 absolute for the features, and the same relative to the largest value for layers.1's output (measured: 2.8e-6 and
    7e-8, i.e. 2.5 % and 0.3 % of the bound).  A float32 path that lost two orders of magnitude of precision would fail."""
    from sampt_b200 import synth
    sd = synth.make_tinyvit_state_dict(5)
    g = torch.Generator().manual_seed(3)
    x = torch.randn((1, 3, 1024, 1024), generator=g)
    f64, i64 = tinyvit_ref.tinyvit_forward({k: v.double() if v.is_floating_point() else v for k, v in sd.items()}, x.double())
    f32, i32 = tinyvit_ref.tinyvit_forward(sd, x)
    assert f32.dtype == torch.float32 and f64.dtype == torch.float64
    assert f64.shape == (1, 256, 64, 64) and i64[0].shape == (1, 64, 64, 160)
    bound = 2.0 ** -24 * math.sqrt(2304) * 40
    assert (f32.double() - f64).abs().max().item() < bound
    assert (i32[0].double() - i64[0]).abs().max().item() < bound * i64[0].abs().max().item()


def test_mobile_sam_checkpoint_size():
    """Encoder + prompt encoder + mask decoder floats: 38-40 MiB of float32, like the 39M sam_mobile_vit_t.pth."""
    from sampt_b200 import factory
    sam = factory.build_sam(factory.TINY_VIT)
    sd = sam.state_dict()
    enc = sum(v.numel() for k, v in sd.items() if k.startswith("image_encoder.") and v.is_floating_point())
    rest = sum(v.numel() for k, v in sd.items() if not k.startswith("image_encoder.") and v.is_floating_point()
               and k not in ("pixel_mean", "pixel_std"))
    assert enc == 6_075_388
    assert rest == 4_064_816
    mib = (enc + rest) * 4 / 2 ** 20
    assert 38.0 <= mib <= 40.0
    assert math.isclose(mib, 38.7, abs_tol=0.05)
