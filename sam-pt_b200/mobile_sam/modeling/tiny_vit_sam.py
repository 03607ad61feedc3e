"""`TinyViT` with upstream constructor kwargs and state-dict keys (MobileSAM mobile_sam/modeling/tiny_vit_sam.py; kwargs per
configs/model/sam/sam_mobile_vit_tiny.yaml) executing in libsampt_b200 (csrc/tinyvit.cu: tensor-core GEMMs with three fp16
hi|lo passes, fp32 depthwise convs, LayerNorms and window attention).

Only the configuration the reference ships is built: TinyViT-5M at img_size 1024 (embed_dims 64/128/160/320, depths 2/2/6/2,
heads 2/4/5/10, windows 7/7/14/7, mlp_ratio 4, MBConv expansion 4, 3x3 local conv).  `norm_head` / `head` (the ImageNet
classifier) are in the checkpoint but never run, as upstream's forward does not run them either.

Kernel-native layouts registered under "sam.tinyvit." (include/sampt_b200.h):
  Conv2d_BN          BatchNorm folded in float64: w' = w g / sqrt(var + 1e-5), b' = beta - mean g / sqrt(var + 1e-5)
  1x1 convs, linears ".w16" [N, 2Kp] fp16 hi | lo of w 2^s, K zero-padded to Kp = a multiple of 64; ".w16s" [1] = 2^-s
  stem convs         im2col columns (ky*3 + kx)*Cin + ci, then as above (K 27 -> 64, 288 -> 320)
  depthwise convs    ".w" [9, C] tap-major fp32, ".b" [C]
  neck               as the ViT's neck (3x3 columns (ky*3 + kx)*256 + ci)
"""
from __future__ import annotations

from ctypes import c_float, c_int, c_size_t, byref
from typing import Dict, List, Sequence, Tuple

import torch
from torch import nn

from sampt_b200 import native
from sampt_b200.gemm_weights import split_scaled as _split
from sampt_b200.param_tree import build_param_tree

EMBED_DIMS = (64, 128, 160, 320)
DEPTHS = (2, 2, 6, 2)
NUM_HEADS = (2, 4, 5, 10)
WINDOW_SIZES = (7, 7, 14, 7)
IMG_SIZE = 1024
NECK_CHANS = 256
BN_EPS = 1e-5


def _pad64(k: int) -> int:
    return -(-k // 64) * 64


def pm_stride(out_dim: int) -> int:
    """PatchMerging keeps the resolution for out_dim 320 / 448 / 576 (upstream PatchMerging.__init__)."""
    return 1 if out_dim in (320, 448, 576) else 2


def _conv_bn(s: Dict[str, Tuple[int, ...]], p: str, cin: int, cout: int, ks: int, groups: int = 1) -> None:
    s[p + ".c.weight"] = (cout, cin // groups, ks, ks)
    for n in ("weight", "bias", "running_mean", "running_var"):
        s[p + ".bn." + n] = (cout,)
    s[p + ".bn.num_batches_tracked"] = ()


def state_dict_shapes(num_classes: int = 1000) -> Dict[str, Tuple[int, ...]]:
    """Every state-dict key of upstream TinyViT-5M (parameters and BatchNorm buffers) with its shape."""
    s: Dict[str, Tuple[int, ...]] = {}
    d0 = EMBED_DIMS[0]
    _conv_bn(s, "patch_embed.seq.0", 3, d0 // 2, 3)
    _conv_bn(s, "patch_embed.seq.2", d0 // 2, d0, 3)
    for i, (dim, depth) in enumerate(zip(EMBED_DIMS, DEPTHS)):
        lp = f"layers.{i}."
        for j in range(depth):
            bp = f"{lp}blocks.{j}."
            if i == 0:
                h = 4 * dim
                _conv_bn(s, bp + "conv1", dim, h, 1)
                _conv_bn(s, bp + "conv2", h, h, 3, groups=h)
                _conv_bn(s, bp + "conv3", h, dim, 1)
                continue
            ws = WINDOW_SIZES[i]
            s[bp + "attn.attention_biases"] = (NUM_HEADS[i], ws * ws)
            s[bp + "attn.norm.weight"] = (dim,)
            s[bp + "attn.norm.bias"] = (dim,)
            s[bp + "attn.qkv.weight"] = (3 * dim, dim)
            s[bp + "attn.qkv.bias"] = (3 * dim,)
            s[bp + "attn.proj.weight"] = (dim, dim)
            s[bp + "attn.proj.bias"] = (dim,)
            s[bp + "mlp.norm.weight"] = (dim,)
            s[bp + "mlp.norm.bias"] = (dim,)
            s[bp + "mlp.fc1.weight"] = (4 * dim, dim)
            s[bp + "mlp.fc1.bias"] = (4 * dim,)
            s[bp + "mlp.fc2.weight"] = (dim, 4 * dim)
            s[bp + "mlp.fc2.bias"] = (dim,)
            _conv_bn(s, bp + "local_conv", dim, dim, 3, groups=dim)
        if i + 1 < len(EMBED_DIMS):
            out = EMBED_DIMS[i + 1]
            _conv_bn(s, lp + "downsample.conv1", dim, out, 1)
            _conv_bn(s, lp + "downsample.conv2", out, out, 3, groups=out)
            _conv_bn(s, lp + "downsample.conv3", out, out, 1)
    d = EMBED_DIMS[-1]
    s["norm_head.weight"], s["norm_head.bias"] = (d,), (d,)
    s["head.weight"], s["head.bias"] = (num_classes, d), (num_classes,)
    s["neck.0.weight"] = (NECK_CHANS, d, 1, 1)
    s["neck.1.weight"], s["neck.1.bias"] = (NECK_CHANS,), (NECK_CHANS,)
    s["neck.2.weight"] = (NECK_CHANS, NECK_CHANS, 3, 3)
    s["neck.3.weight"], s["neck.3.bias"] = (NECK_CHANS,), (NECK_CHANS,)
    return s


def is_buffer(key: str) -> bool:
    return key.endswith((".running_mean", ".running_var", ".num_batches_tracked"))


def fold_conv_bn(sd: Dict[str, torch.Tensor], p: str) -> Tuple[torch.Tensor, torch.Tensor]:
    """Conv2d_BN in eval mode as one conv: (weight, bias) in float64."""
    w = sd[p + ".c.weight"].double()
    g, b = sd[p + ".bn.weight"].double(), sd[p + ".bn.bias"].double()
    rm, rv = sd[p + ".bn.running_mean"].double(), sd[p + ".bn.running_var"].double()
    scale = g / torch.sqrt(rv + BN_EPS)
    return w * scale.view(-1, 1, 1, 1), b - rm * scale


def native_weights(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """Upstream state dict -> {name under "sam.tinyvit.": tensor} in the layouts csrc/tinyvit.cu reads."""
    out: Dict[str, torch.Tensor] = {}

    def dense(p: str, name: str, im2col: bool = False) -> None:
        w, b = fold_conv_bn(sd, p)
        wm = w.permute(0, 2, 3, 1).reshape(w.shape[0], -1) if im2col else w.reshape(w.shape[0], -1)
        out[name + ".w16"], out[name + ".w16s"] = _split(wm, _pad64(wm.shape[1]))
        out[name + ".b"] = b.float()

    def dw(p: str, name: str) -> None:
        w, b = fold_conv_bn(sd, p)
        out[name + ".w"] = w.reshape(w.shape[0], 9).t().float().contiguous()
        out[name + ".b"] = b.float()

    dense("patch_embed.seq.0", "patch_embed.seq.0", im2col=True)
    dense("patch_embed.seq.2", "patch_embed.seq.2", im2col=True)
    for i, depth in enumerate(DEPTHS):
        lp = f"layers.{i}."
        for j in range(depth):
            bp = f"{lp}blocks.{j}."
            if i == 0:
                dense(bp + "conv1", bp + "conv1")
                dw(bp + "conv2", bp + "conv2")
                dense(bp + "conv3", bp + "conv3")
                continue
            for n in ("attn.norm.weight", "attn.norm.bias", "attn.qkv.bias", "attn.proj.bias", "attn.attention_biases",
                      "mlp.norm.weight", "mlp.norm.bias", "mlp.fc1.bias", "mlp.fc2.bias"):
                out[bp + n] = sd[bp + n].float().contiguous()
            for n in ("attn.qkv", "attn.proj", "mlp.fc1", "mlp.fc2"):
                wm = sd[bp + n + ".weight"].double()
                out[bp + n + ".w16"], out[bp + n + ".w16s"] = _split(wm, _pad64(wm.shape[1]))
            dw(bp + "local_conv", bp + "local_conv")
        if i + 1 < len(DEPTHS):
            dense(lp + "downsample.conv1", lp + "downsample.conv1")
            dw(lp + "downsample.conv2", lp + "downsample.conv2")
            dense(lp + "downsample.conv3", lp + "downsample.conv3")
    w0 = sd["neck.0.weight"].double()
    out["neck.0.w16"], out["neck.0.w16s"] = _split(w0.reshape(w0.shape[0], -1), _pad64(w0.shape[1]))
    w2 = sd["neck.2.weight"].double()
    out["neck.2.w16"], out["neck.2.w16s"] = _split(w2.permute(0, 2, 3, 1).reshape(w2.shape[0], -1), 9 * w2.shape[0])
    for n in ("neck.1.weight", "neck.1.bias", "neck.3.weight", "neck.3.bias"):
        out[n] = sd[n].float().contiguous()
    return out


class TinyViT(nn.Module):
    returns_interm = False          # sam-hq's subclass also returns interm_embeddings (layers.1's output)
    PREFIX = "sam.tinyvit."

    def __init__(self, img_size: int = 224, in_chans: int = 3, num_classes: int = 1000,
                 embed_dims: Sequence[int] = (96, 192, 384, 768), depths: Sequence[int] = (2, 2, 6, 2),
                 num_heads: Sequence[int] = (3, 6, 12, 24), window_sizes: Sequence[int] = (7, 7, 14, 7), mlp_ratio: float = 4.,
                 drop_rate: float = 0., drop_path_rate: float = 0.1, use_checkpoint: bool = False, mbconv_expand_ratio: float = 4.0,
                 local_conv_size: int = 3, layer_lr_decay: float = 1.0) -> None:
        super().__init__()
        cfg = (int(img_size), int(in_chans), tuple(int(x) for x in embed_dims), tuple(int(x) for x in depths),
               tuple(int(x) for x in num_heads), tuple(int(x) for x in window_sizes), float(mlp_ratio), float(mbconv_expand_ratio),
               int(local_conv_size))
        want = (IMG_SIZE, 3, EMBED_DIMS, DEPTHS, NUM_HEADS, WINDOW_SIZES, 4.0, 4.0, 3)
        if cfg != want:
            raise NotImplementedError("the H100 TinyViT implements MobileSAM's TinyViT-5M at img_size 1024 (embed_dims "
                                      "[64,128,160,320], depths [2,2,6,2], num_heads [2,4,5,10], window_sizes [7,7,14,7], "
                                      f"mlp_ratio 4, mbconv_expand_ratio 4, local_conv_size 3); got {cfg}")
        # drop_rate / drop_path_rate / use_checkpoint / layer_lr_decay only act in training; this module is inference-only
        self.img_size = IMG_SIZE
        self.num_classes = int(num_classes)
        self.embed_dims, self.depths, self.num_heads, self.window_sizes = EMBED_DIMS, DEPTHS, NUM_HEADS, WINDOW_SIZES
        from sampt_b200 import synth
        sd = synth.make_tinyvit_state_dict(seed=5, num_classes=self.num_classes)
        build_param_tree(self, {k: tuple(v.shape) for k, v in sd.items()}, values=sd, is_buffer=is_buffer)
        self._registered = None

    @property
    def _device(self) -> torch.device:
        return self.neck._modules["0"].weight.device

    # ------------------------------------------------------------------ weights -> libsampt_b200
    def native_context(self) -> native.Context:
        dev = self._device
        ctx = native.get_context(dev)
        key = (id(ctx), tuple(t._version for t in self.state_dict().values()), dev)
        if self._registered != key or not ctx.owns("sam.tinyvit", self):
            torch.cuda.synchronize(dev)   # nothing may still be reading the tensors this replaces
            sd = {k: v.detach().cpu() for k, v in self.state_dict().items()}
            ctx.unset_prefix(self.PREFIX)
            for k, v in native_weights(sd).items():
                ctx.set_tensor(self.PREFIX + k, v)
            self._registered = key
            ctx.claim("sam.tinyvit", self)
        return ctx

    @staticmethod
    def workspace_bytes(B: int) -> int:
        n = c_size_t(0)
        native.check(native.lib().sampt_tinyvit_workspace_bytes(c_int(B), byref(n)), "tinyvit_workspace_bytes")
        return int(n.value)

    def _encode(self, image: torch.Tensor, is_f32: bool, Hr: int, Wr: int, mean, std, want_interm: bool):
        ctx = self.native_context()
        B = image.shape[0]
        ctx.ensure_vit_workspace(self.workspace_bytes(B))
        g = IMG_SIZE // 16
        feats = torch.empty((B, NECK_CHANS, g, g), device=image.device, dtype=torch.float32)
        interm = torch.empty((B, g, g, EMBED_DIMS[2]), device=image.device, dtype=torch.float32) if want_interm else None
        m = (c_float * 3)(*[float(x) for x in mean])
        s = (c_float * 3)(*[float(x) for x in std])
        native.check(native.lib().sampt_tinyvit_encode(
            ctx.handle, native.ptr(image), c_int(1 if is_f32 else 0), c_int(B), c_int(Hr), c_int(Wr), m, s, native.ptr(feats),
            native.ptr(interm), native.stream_ptr()), "tinyvit_encode")
        return feats, interm

    def encode_resized_u8(self, resized: torch.Tensor, pixel_mean, pixel_std, want_interm: bool = False):
        """resized: (B,3,Hr,Wr) uint8 on the GPU (longest side == img_size) -> features (B,256,64,64) fp32 [+ layers.1's output
        (B,64,64,160) for Light HQ-SAM].  Normalisation and zero padding are fused into the stem's im2col."""
        assert resized.dtype == torch.uint8 and resized.is_cuda and resized.dim() == 4
        _, _, Hr, Wr = resized.shape
        feats, interm = self._encode(resized.contiguous(), False, Hr, Wr, pixel_mean, pixel_std, want_interm)
        return (feats, interm) if want_interm else feats

    def forward(self, x: torch.Tensor):
        """Upstream signature: x = preprocessed float image (B,3,1024,1024) (`Sam.preprocess` output) -> (B,256,64,64);
        sam-hq's variant returns (features, [interm_embeddings[0]])."""
        if x.dim() != 4 or x.shape[1] != 3 or x.shape[2] != IMG_SIZE or x.shape[3] != IMG_SIZE:
            raise ValueError(f"expected a (B,3,{IMG_SIZE},{IMG_SIZE}) image, got {tuple(x.shape)}")
        x = x.to(self._device, torch.float32).contiguous()
        feats, interm = self._encode(x, True, IMG_SIZE, IMG_SIZE, (0.0, 0.0, 0.0), (1.0, 1.0, 1.0), self.returns_interm)
        return (feats, [interm]) if self.returns_interm else feats


__all__: List[str] = ["TinyViT"]
