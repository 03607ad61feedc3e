"""`ImageEncoderViT` with upstream constructor kwargs / state-dict keys (segment_anything/modeling/image_encoder.py @ aac76a1;
kwargs per /root/reference/configs/model/sam/image_encoder/vit_base.yaml:1-16) executing in libsampt_b200:
tensor-core GEMMs + fused attention (csrc/gemm_tc.cu, attn_tc.cu, vit_kernels.cu, vit_pipeline.cu)."""
from __future__ import annotations

import math
import os
from ctypes import c_float, c_int
from typing import Dict, Tuple, Type

import torch
from torch import nn

from sampt_b200 import native
from sampt_b200.param_tree import build_param_tree

# GEMM accuracy dial (DESIGN.md "precision"): operands are carried as fp16 hi | lo (lo = fp16(x - hi)) and the tensor-core K loop runs
# over up to three segments A_hi.B_hi + A_lo.B_hi + A_hi.B_lo into one fp32 register accumulator.
#   1 = fp16 x fp16, one pass          2 = weights hi|lo, two passes          3 = MLP three passes, qkv / proj two
#   5 = MLP + proj three passes (attention output kept as hi|lo), qkv two     4 = three passes everywhere (~fp32 products)
#   6 = like 4, but the two correction segments of the qkv / proj / lin1 / lin2 GEMMs are e4m3 operands (e4m3 wgmma at twice
#       the fp16 rate, accumulated apart from the fp16 pass): they are 2^-12 of the result, e4m3's 2^-5 rounding leaves 2^-17,
#       so 2 fp16-pass equivalents instead of 3
# Measured at 6 on one H100 (400 W) against the FULL BASELINE clips (tests/test_gpu_full_configs.py: 50 frames of C2, 50 of C3,
# 8 of the C5 slice; bar: per-frame IoU >= 0.999), min IoU C2 / C3 / C5s: 0.99976 / 0.99971 / 0.99963.  With random weights the
# mask logits are noise-like and the 12-step box refinement amplifies a 1-pixel box change into ~1e-3 IoU, so settings that drop a
# correction term (2, 3, 5) sit close to or below the bar; 6 is the default.
DEFAULT_PRECISION = int(os.environ.get("SAMPT_VIT_PRECISION", "6"))


class ImageEncoderViT(nn.Module):
    def __init__(self, img_size: int = 1024, patch_size: int = 16, in_chans: int = 3, embed_dim: int = 768, depth: int = 12,
                 num_heads: int = 12, mlp_ratio: float = 4.0, out_chans: int = 256, qkv_bias: bool = True,
                 norm_layer: Type[nn.Module] = nn.LayerNorm, act_layer: Type[nn.Module] = nn.GELU, use_abs_pos: bool = True,
                 use_rel_pos: bool = False, rel_pos_zero_init: bool = True, window_size: int = 0,
                 global_attn_indexes: Tuple[int, ...] = ()) -> None:
        super().__init__()
        if not (use_abs_pos and use_rel_pos and qkv_bias and in_chans == 3 and int(mlp_ratio) == 4):
            raise NotImplementedError("the H100 encoder implements SAM's configuration: abs+rel pos, qkv bias, mlp_ratio 4")
        self.img_size, self.patch_size, self.embed_dim, self.depth = img_size, patch_size, embed_dim, depth
        self.num_heads, self.out_chans, self.window_size = num_heads, out_chans, window_size
        self.global_attn_indexes = tuple(int(i) for i in global_attn_indexes)
        self.precision = DEFAULT_PRECISION
        build_param_tree(self, self._shapes(), seed=1024 + depth)
        self._registered = None

    def _shapes(self) -> Dict[str, Tuple[int, ...]]:
        D, g, hd = self.embed_dim, self.img_size // self.patch_size, self.embed_dim // self.num_heads
        s: Dict[str, Tuple[int, ...]] = {"pos_embed": (1, g, g, D), "patch_embed.proj.weight": (D, 3, self.patch_size, self.patch_size),
                                         "patch_embed.proj.bias": (D,)}
        for i in range(self.depth):
            S = g if i in self.global_attn_indexes else self.window_size
            b = f"blocks.{i}."
            for n, shp in (("norm1.weight", (D,)), ("norm1.bias", (D,)), ("norm2.weight", (D,)), ("norm2.bias", (D,)),
                           ("attn.qkv.weight", (3 * D, D)), ("attn.qkv.bias", (3 * D,)), ("attn.proj.weight", (D, D)),
                           ("attn.proj.bias", (D,)), ("attn.rel_pos_h", (2 * S - 1, hd)), ("attn.rel_pos_w", (2 * S - 1, hd)),
                           ("mlp.lin1.weight", (4 * D, D)), ("mlp.lin1.bias", (4 * D,)), ("mlp.lin2.weight", (D, 4 * D)),
                           ("mlp.lin2.bias", (D,))):
                s[b + n] = shp
        C = self.out_chans
        s.update({"neck.0.weight": (C, D, 1, 1), "neck.1.weight": (C,), "neck.1.bias": (C,), "neck.2.weight": (C, C, 3, 3),
                  "neck.3.weight": (C,), "neck.3.bias": (C,)})
        return s

    # ------------------------------------------------------------------ weights -> kernel-native layouts
    @staticmethod
    def _w16(w: torch.Tensor, split: bool):
        """fp16 operand of w 2^s (hi, or hi | lo with lo = fp16(w 2^s - hi)) and the accumulator scale 2^-s, where s puts
        max|w| 2^s in [2^14, 2^15), so that (hi + lo) 2^-s restores w to 2^-22 |w|.  Unscaled, weights of size ~1/sqrt(K) leave
        every lo an fp16 subnormal, which restores w only to 2^-25 absolute."""
        w = w.detach().float()
        amax = float(w.abs().max())
        s = 15 - (math.frexp(amax)[1] if amax > 0 else 0)
        ws = w * (2.0 ** s)
        hi = ws.half()
        scale = torch.tensor([2.0 ** (-s)], dtype=torch.float32, device=w.device)
        if not split:
            return hi.contiguous(), scale
        lo = (ws - hi.float()).half()
        return torch.cat([hi, lo], dim=1).contiguous(), scale

    @staticmethod
    def _w8(w: torch.Tensor):
        """Weight operand of the fp8-corrected GEMM (include/sampt_b200.h: sampt_gemm_f8c): rows of 2K fp16 units
        [fp16(w 2^s) | e4m3(w 2^(s-12)) | e4m3((w 2^s - fp16(w 2^s)) 2^3)] and the accumulator scale 2^-s."""
        w = w.detach().float()
        amax = float(w.abs().max())
        s = 15 - (math.frexp(amax)[1] if amax > 0 else 0)         # |w| 2^s <= 2^15 (fp16 max 65504)
        ws = w * (2.0 ** s)
        hi = ws.half()
        rem = ws - hi.float()

        def e4m3(t):
            return t.clamp(-448.0, 448.0).to(torch.float8_e4m3fn).view(torch.uint8)

        hi8 = e4m3(w * (2.0 ** (s - 12)))
        lo8 = e4m3(rem * 8.0)
        packed = torch.cat([hi.view(torch.uint8), hi8, lo8], dim=1).contiguous()      # (N, 2K + K + K) bytes
        return packed.view(torch.float16), torch.tensor([2.0 ** (-s)], dtype=torch.float32, device=w.device)

    def native_weights(self) -> Dict[str, torch.Tensor]:
        """{name under "sam.image_encoder.": tensor} in the layouts csrc/vit_pipeline.cu reads at self.precision: every GEMM
        weight as "<layer>.w16" (fp16 w 2^s, hi | lo from precision 2 on) with its scale 2^-s as "<layer>.w16s", at precision
        6 also the fp8-corrected "<layer>.w8" / ".w8s" of the block linears."""
        split_b = self.precision >= 2   # (3, 4, 5: activations split as well, decided inside sampt_vit_encode)
        sd = self.state_dict()
        D, C = self.embed_dim, self.out_chans
        out: Dict[str, torch.Tensor] = {}

        def w16(name, w):
            out[name + ".w16"], out[name + ".w16s"] = self._w16(w, split_b)

        w16("patch_embed", sd["patch_embed.proj.weight"].reshape(D, -1))
        out["patch_embed.proj.bias"] = sd["patch_embed.proj.bias"].float()
        out["pos_embed"] = sd["pos_embed"].float().reshape(-1, D)
        for i in range(self.depth):
            b = f"blocks.{i}."
            for n in ("norm1.weight", "norm1.bias", "norm2.weight", "norm2.bias", "attn.qkv.bias", "attn.proj.bias",
                      "attn.rel_pos_h", "attn.rel_pos_w", "mlp.lin1.bias", "mlp.lin2.bias"):
                out[b + n] = sd[b + n].float()
            for n in ("attn.qkv", "attn.proj", "mlp.lin1", "mlp.lin2"):
                w16(b + n, sd[b + n + ".weight"])
                if self.precision == 6:
                    out[b + n + ".w8"], out[b + n + ".w8s"] = self._w8(sd[b + n + ".weight"])
        w16("neck.0", sd["neck.0.weight"].reshape(C, D))
        w16("neck.2", sd["neck.2.weight"].permute(0, 2, 3, 1).reshape(C, 9 * C))
        for n in ("neck.1.weight", "neck.1.bias", "neck.3.weight", "neck.3.bias"):
            out[n] = sd[n].float()
        return out

    def native_context(self, prefix: str = "sam.image_encoder.") -> native.Context:
        dev = self.pos_embed.device
        ctx = native.get_context(dev)
        key = (id(ctx), self.precision, tuple(p._version for p in self.parameters()), dev)
        if self._registered != key or not ctx.owns("sam.image_encoder", self):
            torch.cuda.synchronize(dev)  # nothing may still be reading the tensors this replaces
            native.check(native.lib().sampt_vit_cache_clear(ctx.handle), "vit_cache_clear")  # rows saved for the old weights
            for name, t in self.native_weights().items():
                ctx.set_tensor(prefix + name, t)
            self._registered = key
            ctx.claim("sam.image_encoder", self)
        return ctx

    def workspace_bytes(self, B: int) -> int:
        D, g = self.embed_dim, self.img_size // self.patch_size
        nW = -(-g // self.window_size)
        mtok, mwin = B * g * g, B * nW * nW * self.window_size ** 2
        asp = 2 if self.precision >= 3 else 1
        hd = D // self.num_heads
        dkw, dkg = -(-(hd + 2 * self.window_size) // 64) * 64, -(-(hd + 2 * g) // 64) * 64
        q = max(mwin * self.num_heads * dkw, mtok * self.num_heads * dkg) * 2
        v = max(mwin // self.window_size ** 2 * self.num_heads * hd * 256, B * self.num_heads * hd * g * g) * 2
        total = mtok * D * 4 + max(mwin, mtok) * max(D, 768) * asp * 2 + mwin * 3 * D * 2 + 2 * q + v + mwin * D * asp * 2 \
            + mtok * max(4 * D, 9 * self.out_chans) * asp * 2 + mtok * self.out_chans * 8 + mwin * 4
        return int(total * 1.02) + (64 << 20)

    def encode_resized_u8(self, resized: torch.Tensor, pixel_mean, pixel_std, want_interm: bool = False):
        """resized: (B,3,Hr,Wr) uint8 on the GPU (longest side == img_size) -> features (B,out_chans,g,g) fp32
        [+ first global block output (B,g,g,D) for HQ-SAM].  Normalisation + zero padding are fused into the patch im2col."""
        assert resized.dtype == torch.uint8 and resized.is_cuda and resized.dim() == 4
        ctx = self.native_context()
        B, _, Hr, Wr = resized.shape
        g = self.img_size // self.patch_size
        ctx.ensure_vit_workspace(self.workspace_bytes(B))
        feats = torch.empty((B, self.out_chans, g, g), device=resized.device, dtype=torch.float32)
        interm = torch.empty((B, g, g, self.embed_dim), device=resized.device, dtype=torch.float32) if want_interm else None
        gidx = (c_int * max(1, len(self.global_attn_indexes)))(*self.global_attn_indexes)
        mean = (c_float * 3)(*[float(x) for x in pixel_mean])
        std = (c_float * 3)(*[float(x) for x in pixel_std])
        native.check(native.lib().sampt_vit_encode(
            ctx.handle, native.ptr(resized.contiguous()), c_int(B), c_int(Hr), c_int(Wr), c_int(self.depth), c_int(self.embed_dim),
            c_int(self.num_heads), c_int(self.window_size), gidx, c_int(len(self.global_attn_indexes)), c_int(self.img_size),
            c_int(self.patch_size), c_int(self.out_chans), c_int(self.precision), mean, std, native.ptr(feats), native.ptr(interm),
            native.stream_ptr()), "vit_encode")
        return (feats, interm) if want_interm else feats

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """Upstream signature: x = preprocessed float image (B,3,img_size,img_size) (`Sam.preprocess` output) -> (B,out_chans,g,g).
        (SamPredictor uses `encode_resized_u8`, which fuses the normalisation and zero padding into the patch im2col.)"""
        if x.dim() != 4 or x.shape[1] != 3 or x.shape[2] != self.img_size or x.shape[3] != self.img_size:
            raise ValueError(f"expected a (B,3,{self.img_size},{self.img_size}) image, got {tuple(x.shape)}")
        ctx = self.native_context()
        dev = self.pos_embed.device
        x = x.to(dev, torch.float32).contiguous()
        B = x.shape[0]
        g = self.img_size // self.patch_size
        ctx.ensure_vit_workspace(self.workspace_bytes(B))
        feats = torch.empty((B, self.out_chans, g, g), device=dev, dtype=torch.float32)
        gidx = (c_int * max(1, len(self.global_attn_indexes)))(*self.global_attn_indexes)
        native.check(native.lib().sampt_vit_encode_f32(
            ctx.handle, native.ptr(x), c_int(B), c_int(self.depth), c_int(self.embed_dim), c_int(self.num_heads), c_int(self.window_size),
            gidx, c_int(len(self.global_attn_indexes)), c_int(self.img_size), c_int(self.patch_size), c_int(self.out_chans),
            c_int(self.precision), native.ptr(feats), native.ptr(None), native.stream_ptr()), "vit_encode_f32")
        return feats
