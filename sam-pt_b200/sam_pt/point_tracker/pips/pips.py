"""`Pips` with the reference's constructor / forward signature and state-dict (sam_pt/point_tracker/pips/pips.py:410-620,
SURVEY Appendix A.4) whose arithmetic runs in libsampt_b200 (csrc/pips_kernels.cu, csrc/pips_pipeline.cu)."""
from __future__ import annotations

import os
from ctypes import c_float, c_int
from typing import Dict, Tuple

import torch
from torch import nn

from sampt_b200 import native
from sampt_b200.param_tree import build_param_tree

LATENT = 128


def _pips_shapes(S: int) -> Dict[str, Tuple[int, ...]]:
    s: Dict[str, Tuple[int, ...]] = {}

    def conv(name, co, ci, k):
        s[f"{name}.weight"] = (co, ci, k, k)
        s[f"{name}.bias"] = (co,)

    conv("fnet.conv1", 64, 3, 7)
    cin = 64
    for li, (dim, stride) in enumerate(((64, 1), (96, 2), (128, 2), (128, 2)), start=1):
        for blk in (0, 1):
            conv(f"fnet.layer{li}.{blk}.conv1", dim, cin if blk == 0 else dim, 3)
            conv(f"fnet.layer{li}.{blk}.conv2", dim, dim, 3)
        if stride != 1:
            conv(f"fnet.layer{li}.0.downsample.0", dim, cin, 1)
        cin = dim
    conv("fnet.conv2", 256, 64 + 96 + 128 + 128, 3)
    conv("fnet.conv3", LATENT, 256, 1)
    p = "delta_block.to_delta."
    kitchen = 4 * 7 * 7 + LATENT + 3 * 64 + 3
    s[p + "0.weight"], s[p + "0.bias"] = (512, kitchen), (512,)
    for l in range(1, 13):
        for j, (a, b) in enumerate((((4 * S, S, 1), (S, 4 * S, 1)), ((2048, 512), (512, 2048)))):
            s[f"{p}{l}.{j}.norm.weight"] = s[f"{p}{l}.{j}.norm.bias"] = (512,)
            s[f"{p}{l}.{j}.fn.0.weight"], s[f"{p}{l}.{j}.fn.0.bias"] = a, (a[0],)
            s[f"{p}{l}.{j}.fn.3.weight"], s[f"{p}{l}.{j}.fn.3.bias"] = b, (b[0],)
    s[p + "13.weight"] = s[p + "13.bias"] = (512,)
    s[p + "15.weight"], s[p + "15.bias"] = (S * (LATENT + 2), 512), (S * (LATENT + 2),)
    s["norm.weight"] = s["norm.bias"] = (LATENT,)
    s["ffeat_updater.0.weight"], s["ffeat_updater.0.bias"] = (LATENT, LATENT), (LATENT,)
    s["vis_predictor.0.weight"], s["vis_predictor.0.bias"] = (1, LATENT), (1,)
    return s


class Pips(nn.Module):
    """Reference signature `Pips(S=8, stride=8)` (pips.py:411)."""

    def __init__(self, S=8, stride=8):
        super().__init__()
        self.S = S
        self.stride = stride
        self.hidden_dim = 256
        self.latent_dim = LATENT
        self.corr_levels = 4
        self.corr_radius = 3
        build_param_tree(self, _pips_shapes(S), seed=486124)
        self._registered_on = None
        # BasicEncoder convolutions as im2col + tensor-core GEMM with 3-pass fp16 split (~fp32); "0" = strict fp32 CUDA-core path
        self.fnet_on_tensor_cores = os.environ.get("SAMPT_PIPS_TC", "1") != "0"

    # ------------------------------------------------------------------ weights -> kernel-native layouts
    def native_context(self) -> native.Context:
        dev = self.norm.weight.device
        ctx = native.get_context(dev)
        key = (id(ctx), tuple(p._version for p in self.parameters()), dev, self.fnet_on_tensor_cores)
        if self._registered_on != key or not ctx.owns("pips", self):
            torch.cuda.synchronize(dev)  # nothing may still be reading the tensors this replaces
            sd = self.state_dict()
            # path selector read by sampt_pips_fnet (shape [1] = tensor-core convolutions, shape [2] = fp32 CUDA cores)
            ctx.set_tensor("pips.fnet.tc_flag", torch.zeros(1 if self.fnet_on_tensor_cores else 2, dtype=torch.int32,
                                                            device=self.norm.weight.device))
            for k, v in sd.items():
                v = v.detach().float()
                if k.startswith("fnet.") and k.endswith(".weight") and v.dim() == 4:
                    ctx.set_tensor(f"pips.{k}_rsck", v.permute(2, 3, 1, 0).contiguous())
                    if self.fnet_on_tensor_cores:
                        # tensor-core path: [Cout, 2*Kp] fp16 hi|lo, k = (r*S + s)*Cin + ci, K zero-padded to a multiple of 64
                        w = v.permute(0, 2, 3, 1).reshape(v.shape[0], -1)
                        kp = -(-w.shape[1] // 64) * 64
                        wp = torch.zeros((w.shape[0], kp), device=w.device)
                        wp[:, : w.shape[1]] = w
                        hi = wp.half()
                        lo = (wp - hi.float()).half()
                        ctx.set_tensor(f"pips.{k[:-len('.weight')]}.w16", torch.cat([hi, lo], dim=1).contiguous())
                elif k == "delta_block.to_delta.0.weight":
                    w = torch.zeros((v.shape[0], 520), device=v.device)
                    w[:, : v.shape[1]] = v
                    ctx.set_tensor(f"pips.{k}_kpad", w)
                else:
                    ctx.set_tensor(f"pips.{k}", v.contiguous())
            self._registered_on = key
            ctx.claim("pips", self)
        return ctx

    # ------------------------------------------------------------------ building blocks used by the tracker
    def fnet_frames(self, frames_u8: torch.Tensor) -> torch.Tensor:
        """(n,3,H,W) uint8 -> channels-last encoder features (n,H/4,W/4,128) fp32 (BasicEncoder, once per frame)."""
        assert frames_u8.dtype == torch.uint8 and frames_u8.is_cuda
        if self.stride != 4:
            raise NotImplementedError("the H100 PIPS path is built for stride 4 (configs/model/point_tracker/pips.yaml:3)")
        ctx = self.native_context()
        n, _, H, W = frames_u8.shape
        fm = torch.empty((n, H // 4, W // 4, LATENT), device=frames_u8.device, dtype=torch.float32)
        native.check(native.lib().sampt_pips_fnet(ctx.handle, native.ptr(frames_u8.contiguous()), c_int(n), c_int(H), c_int(W),
                                                  c_int(4), native.ptr(fm), native.stream_ptr()), "pips_fnet")
        return fm

    def build_pyramid(self, fmaps: torch.Tensor):
        """(T,H4,W4,128) -> [level0, /2, /4, /8] (CorrBlock.__init__ avg-pool pyramid, pips.py:355-361)."""
        ctx = self.native_context()
        T, H4, W4, _ = fmaps.shape
        pyr = [fmaps.contiguous()] + [torch.empty((T, H4 >> l, W4 >> l, LATENT), device=fmaps.device, dtype=torch.float32)
                                      for l in range(1, 4)]
        native.check(native.lib().sampt_pips_pyramid(ctx.handle, native.ptr(pyr[0]), c_int(T), c_int(H4), c_int(W4),
                                                     native.ptr(pyr[1]), native.ptr(pyr[2]), native.ptr(pyr[3]),
                                                     native.stream_ptr()), "pips_pyramid")
        return pyr

    def encode_frames(self, frames_u8: torch.Tensor):
        """(T,3,H,W) uint8 -> channels-last pyramid [(T,H/4,W/4,128), /2, /4, /8] (fnet once per frame + CorrBlock pyramid)."""
        return self.build_pyramid(self.fnet_frames(frames_u8))

    def track(self, pyr, query_points: torch.Tensor, thr0: float, iters: int = 6, flip: bool = False,
              max_windows: int = 0):
        """One direction of the linked sliding-window chain. query_points (N,3) -> traj (T,N,2), vis (T,N) sigmoid."""
        ctx = self.native_context()
        T, H4, W4, _ = pyr[0].shape
        N = query_points.shape[0]
        q = query_points.detach().float().contiguous()
        traj = torch.empty((T, N, 2), device=q.device, dtype=torch.float32)
        vis = torch.empty((T, N), device=q.device, dtype=torch.float32)
        native.check(native.lib().sampt_pips_track(
            ctx.handle, native.ptr(pyr[0]), native.ptr(pyr[1]), native.ptr(pyr[2]), native.ptr(pyr[3]), c_int(T), c_int(H4),
            c_int(W4), native.ptr(q), c_int(N), c_int(self.S), c_int(self.stride), c_float(thr0), c_int(iters),
            c_int(1 if flip else 0), c_int(max_windows), native.ptr(traj), native.ptr(vis), native.stream_ptr()), "pips_track")
        return traj, vis

    # ------------------------------------------------------------------ reference-compatible forward
    def forward(self, xys, rgbs, coords_init=None, feat_init=None, iters=3, trajs_g=None, vis_g=None, valids=None,
                sw=None, return_feat=False, is_train=False):
        """Reference `Pips.forward` (pips.py:439-620), inference: one S-frame window.
        xys (1,N,2) px, rgbs (1,S,3,H,W) 0..255, coords_init (1,S,N,2) px or None (zero-velocity init, :460-465), feat_init
        (1,N,128) or None (bilinear sample of frame 0, :469-475) -> (coord_predictions: `iters` tensors (1,S,N,2), one per
        refinement iteration (:546); coord_predictions2: the same list bracketed by two copies of the initial and two of the final
        estimate (:479-480,571-572); vis_e (1,S,N) raw logits (:568); [ffeat (1,N,128) if return_feat (:617-618);] losses=None).
        One native call (`sampt_pips_window`)."""
        if trajs_g is not None or is_train or self.training or (sw is not None and getattr(sw, "save_this", False)):
            raise NotImplementedError("H100 Pips.forward covers inference (no losses / training / summary writer)")
        B, N, D = xys.shape
        assert D == 2
        if B != 1:
            raise NotImplementedError("Batch size > 1 is not supported for PIPS yet")
        assert rgbs.shape[1] == self.S
        dev = self.norm.weight.device
        frames = rgbs[0].to(dev)
        if frames.dtype != torch.uint8:
            frames = frames.round().clamp(0, 255).to(torch.uint8)
        pyr = self.encode_frames(frames)
        ctx = self.native_context()
        S = self.S
        H4, W4 = pyr[0].shape[1:3]
        q = xys[0].detach().float().to(dev).contiguous()
        ci = coords_init[0].detach().float().to(dev).contiguous() if coords_init is not None else None
        fi = feat_init[0].detach().float().to(dev).contiguous() if feat_init is not None else None
        coords_out = torch.empty((max(iters, 1), S, N, 2), device=dev, dtype=torch.float32)
        vis_e = torch.empty((S, N), device=dev, dtype=torch.float32)
        ffeat = torch.empty((N, LATENT), device=dev, dtype=torch.float32)
        native.check(native.lib().sampt_pips_window(
            ctx.handle, native.ptr(pyr[0]), native.ptr(pyr[1]), native.ptr(pyr[2]), native.ptr(pyr[3]), c_int(H4), c_int(W4),
            native.ptr(q), native.ptr(ci), native.ptr(fi), c_int(N), c_int(S), c_int(self.stride), c_int(iters), native.ptr(coords_out),
            native.ptr(vis_e), native.ptr(ffeat), native.stream_ptr()), "pips_window")
        init = (ci if ci is not None else q[None].repeat(S, 1, 1))[None]
        preds = [coords_out[i][None] for i in range(iters)]
        last = preds[-1] if iters > 0 else init
        preds2 = [init, init] + preds + [last, last]
        if return_feat:
            return preds, preds2, vis_e[None], ffeat[None], None
        return preds, preds2, vis_e[None], None
