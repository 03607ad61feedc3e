"""CPU restatement of MobileSAM's TinyViT-5M image encoder (mobile_sam/modeling/tiny_vit_sam.py; sam-hq's copy returns
layers.1's output as interm_embeddings[0]) as functions over a state dict under upstream key names.

dtype-generic: every op runs in the dtype of the input image (float32 or float64; the state dict is cast to it).  Unpinned
against upstream (its package is not available here): the structural pins are the key set and shapes, the parameter count
and the attention-bias indexing (tests/test_oracle_tinyvit.py).
"""
from __future__ import annotations

import itertools
from typing import Dict, List, Tuple

import torch
import torch.nn.functional as F

from oracle import sam_ref

EMBED_DIMS = (64, 128, 160, 320)
DEPTHS = (2, 2, 6, 2)
NUM_HEADS = (2, 4, 5, 10)
WINDOW_SIZES = (7, 7, 14, 7)
BN_EPS = 1e-5
LN_EPS = 1e-5


def _t(sd, k, x):
    return sd[k].to(x.dtype)


def conv_bn(sd, p: str, x: torch.Tensor, stride: int = 1, pad: int = 0, groups: int = 1) -> torch.Tensor:
    """Conv2d_BN in eval mode on NCHW x: conv (no bias) then BatchNorm2d with running statistics."""
    y = F.conv2d(x, _t(sd, p + ".c.weight", x), None, stride, pad, 1, groups)
    return F.batch_norm(y, _t(sd, p + ".bn.running_mean", x), _t(sd, p + ".bn.running_var", x), _t(sd, p + ".bn.weight", x),
                        _t(sd, p + ".bn.bias", x), False, 0.0, BN_EPS)


def attention_bias_idxs(ws: int) -> torch.Tensor:
    """(L, L) index into attention_biases[h], built as upstream Attention.__init__ does: offsets numbered in order of first
    appearance over itertools.product of the window's points."""
    points = list(itertools.product(range(ws), range(ws)))
    offsets: Dict[Tuple[int, int], int] = {}
    idxs = []
    for p1 in points:
        for p2 in points:
            off = (abs(p1[0] - p2[0]), abs(p1[1] - p2[1]))
            if off not in offsets:
                offsets[off] = len(offsets)
            idxs.append(offsets[off])
    return torch.tensor(idxs, dtype=torch.long).view(len(points), len(points))


def stem(sd, x: torch.Tensor) -> torch.Tensor:
    """patch_embed.seq on the preprocessed (B,3,1024,1024) image -> NCHW (B,64,256,256)."""
    x = F.gelu(conv_bn(sd, "patch_embed.seq.0", x, 2, 1))
    return conv_bn(sd, "patch_embed.seq.2", x, 2, 1)


def mbconv(sd, p: str, x: torch.Tensor) -> torch.Tensor:
    h = x.shape[1] * 4
    y = F.gelu(conv_bn(sd, p + ".conv1", x))
    y = F.gelu(conv_bn(sd, p + ".conv2", y, 1, 1, groups=h))
    y = conv_bn(sd, p + ".conv3", y)
    return F.gelu(y + x)


def patch_merging(sd, p: str, x: torch.Tensor, out_dim: int) -> torch.Tensor:
    """NCHW in, NCHW out."""
    s = 1 if out_dim in (320, 448, 576) else 2
    y = F.gelu(conv_bn(sd, p + ".conv1", x))
    y = F.gelu(conv_bn(sd, p + ".conv2", y, s, 1, groups=out_dim))
    return conv_bn(sd, p + ".conv3", y)


def attention(sd, p: str, x: torch.Tensor, heads: int, ws: int) -> torch.Tensor:
    """Attention.forward on windows x (nW, L, C) (eval: the bias table gathered through attention_bias_idxs)."""
    n, L, C = x.shape
    kd = 32
    x = F.layer_norm(x, (C,), _t(sd, p + ".norm.weight", x), _t(sd, p + ".norm.bias", x), LN_EPS)
    qkv = F.linear(x, _t(sd, p + ".qkv.weight", x), _t(sd, p + ".qkv.bias", x))
    q, k, v = qkv.view(n, L, heads, -1).split([kd, kd, kd], dim=3)
    q, k, v = q.permute(0, 2, 1, 3), k.permute(0, 2, 1, 3), v.permute(0, 2, 1, 3)
    ab = _t(sd, p + ".attention_biases", x)[:, attention_bias_idxs(ws)]
    attn = (q @ k.transpose(-2, -1)) * (kd ** -0.5) + ab
    attn = attn.softmax(dim=-1)
    y = (attn @ v).transpose(1, 2).reshape(n, L, heads * kd)
    return F.linear(y, _t(sd, p + ".proj.weight", x), _t(sd, p + ".proj.bias", x))


def block_attn(sd, p: str, x: torch.Tensor, heads: int, ws: int) -> torch.Tensor:
    """x (B,H,W,C) -> x + attn(window_partition(zero_pad(x))) cropped back (TinyViTBlock.forward's first half)."""
    B, H, W, C = x.shape
    pb, pr = (ws - H % ws) % ws, (ws - W % ws) % ws
    y = F.pad(x, (0, 0, 0, pr, 0, pb)) if (pb or pr) else x
    pH, pW = H + pb, W + pr
    nH, nW = pH // ws, pW // ws
    y = y.view(B, nH, ws, nW, ws, C).transpose(2, 3).reshape(B * nH * nW, ws * ws, C)
    y = attention(sd, p + "attn", y, heads, ws)
    y = y.view(B, nH, nW, ws, ws, C).transpose(2, 3).reshape(B, pH, pW, C)[:, :H, :W]
    return x + y


def block(sd, p: str, x: torch.Tensor, heads: int, ws: int) -> torch.Tensor:
    """TinyViTBlock on x (B,H,W,C)."""
    x = block_attn(sd, p, x, heads, ws)
    C = x.shape[-1]
    x = conv_bn(sd, p + "local_conv", x.permute(0, 3, 1, 2), 1, 1, groups=C).permute(0, 2, 3, 1)
    y = F.layer_norm(x, (C,), _t(sd, p + "mlp.norm.weight", x), _t(sd, p + "mlp.norm.bias", x), LN_EPS)
    y = F.gelu(F.linear(y, _t(sd, p + "mlp.fc1.weight", x), _t(sd, p + "mlp.fc1.bias", x)))
    return x + F.linear(y, _t(sd, p + "mlp.fc2.weight", x), _t(sd, p + "mlp.fc2.bias", x))


def stage(sd, i: int, x: torch.Tensor) -> torch.Tensor:
    """layers.i with its downsample on token-major x (B, R*R, C) -> (B, R'*R', C')."""
    B, L, C = x.shape
    R = int(round(L ** 0.5))
    x = x.view(B, R, R, C)
    for j in range(DEPTHS[i]):
        p = f"layers.{i}.blocks.{j}."
        if i == 0:
            x = mbconv(sd, p[:-1], x.permute(0, 3, 1, 2)).permute(0, 2, 3, 1)
        else:
            x = block(sd, p, x, NUM_HEADS[i], WINDOW_SIZES[i])
    if i + 1 < len(EMBED_DIMS):
        x = patch_merging(sd, f"layers.{i}.downsample", x.permute(0, 3, 1, 2), EMBED_DIMS[i + 1]).permute(0, 2, 3, 1)
    return x.reshape(B, -1, x.shape[-1])


def layer_norm_2d(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, eps: float = 1e-6) -> torch.Tensor:
    u = x.mean(1, keepdim=True)
    s = (x - u).pow(2).mean(1, keepdim=True)
    x = (x - u) / torch.sqrt(s + eps)
    return w[:, None, None] * x + b[:, None, None]


def neck(sd, x: torch.Tensor) -> torch.Tensor:
    """(B, 4096, 320) tokens -> (B, 256, 64, 64)."""
    B = x.shape[0]
    x = x.view(B, 64, 64, -1).permute(0, 3, 1, 2)
    x = F.conv2d(x, _t(sd, "neck.0.weight", x))
    x = layer_norm_2d(x, _t(sd, "neck.1.weight", x), _t(sd, "neck.1.bias", x))
    x = F.conv2d(x, _t(sd, "neck.2.weight", x), padding=1)
    return layer_norm_2d(x, _t(sd, "neck.3.weight", x), _t(sd, "neck.3.bias", x))


def preprocess_u8(resized: torch.Tensor, mean, std, dtype=torch.float32, size: int = 1024) -> torch.Tensor:
    """Sam.preprocess of resized uint8 frames (B,3,Hr,Wr): (x - mean) / std in `dtype`, zero-padded to size^2."""
    x = resized.to(dtype)
    m = torch.tensor(list(mean), dtype=dtype).view(1, 3, 1, 1)
    s = torch.tensor(list(std), dtype=dtype).view(1, 3, 1, 1)
    x = (x - m) / s
    return F.pad(x, (0, size - x.shape[-1], 0, size - x.shape[-2]))


def tinyvit_forward(sd, x: torch.Tensor) -> Tuple[torch.Tensor, List[torch.Tensor]]:
    """Preprocessed (B,3,1024,1024) image -> (features (B,256,64,64), [layers.1's output (B,64,64,160)])."""
    y = stem(sd, x)
    B = y.shape[0]
    y = y.permute(0, 2, 3, 1).reshape(B, -1, y.shape[1])
    interm = []
    for i in range(len(EMBED_DIMS)):
        y = stage(sd, i, y)
        if i == 1:
            interm.append(y.view(B, 64, 64, -1))
    return neck(sd, y), interm



class RefTinySamPredictor(sam_ref.RefSamPredictor):
    """sam_ref.RefSamPredictor with the TinyViT encoder (MobileSAM; Light HQ-SAM with hq=True): the state dict holds
    `image_encoder.*` under TinyViT's keys and the prompt encoder / mask decoder under SAM's."""

    def __init__(self, sd, hq: bool = False):
        super().__init__(sd, sam_ref.VitCfg(img_size=1024), hq=hq)
        self.enc_sd = {k[len("image_encoder."):]: v for k, v in sd.items() if k.startswith("image_encoder.")}

    @torch.no_grad()
    def set_image(self, image_hwc_u8):
        x, self.input_size = sam_ref.preprocess(image_hwc_u8, 1024, 1024)
        self.original_size = tuple(image_hwc_u8.shape[:2])
        self.features, self.interm = tinyvit_forward(self.enc_sd, x.to(self.enc_sd["patch_embed.seq.0.c.weight"].dtype))
