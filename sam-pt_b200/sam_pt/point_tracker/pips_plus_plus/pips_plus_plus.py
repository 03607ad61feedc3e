"""`PipsPlusPlus` with the reference's constructor / forward signature and state dict (sam_pt/point_tracker/pips_plus_plus/
pips_plus_plus.py:420-546) whose arithmetic runs in libsampt_b200 (csrc/pips_plus_plus.cu, the BasicEncoder of
csrc/pips_pipeline.cu at stride 8)."""
from __future__ import annotations

from ctypes import c_int
from typing import Dict, Tuple

import torch
from torch import nn

from sampt_b200 import native
from sampt_b200.gemm_weights import split_scaled
from sampt_b200.param_tree import build_param_tree

LATENT = 128
ROW = 3 * 4 * 49 + LATENT + 2          # 718 DeltaBlock input channels
BLOCK_CHANNELS = ((128, 128), (128, 128), (128, 256), (256, 256), (256, 512), (512, 512), (512, 1024), (1024, 1024))
DENSE_ROWS = 32                        # dense 1024 -> 2 runs on gemm_tc with 30 zero rows (N % 32 == 0)
PREFIX = "ppp."


def state_dict_shapes() -> Dict[str, Tuple[int, ...]]:
    """The 82 tensors of the reference's PipsPlusPlus(stride=8).state_dict()."""
    s: Dict[str, Tuple[int, ...]] = {}

    def conv(name, co, ci, k, dim=2):
        s[f"{name}.weight"] = (co, ci) + (k,) * dim
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
    conv("delta_block.first_block_conv.conv", 128, ROW, 3, dim=1)
    for i, (ci, co) in enumerate(BLOCK_CHANNELS):
        conv(f"delta_block.basicblock_list.{i}.conv1.conv", co, ci, 3, dim=1)
        conv(f"delta_block.basicblock_list.{i}.conv2.conv", co, co, 3, dim=1)
    s["delta_block.dense.weight"], s["delta_block.dense.bias"] = (2, 1024), (2,)
    s["norm.weight"] = s["norm.bias"] = (LATENT,)
    return s


def posemb_omega() -> torch.Tensor:
    """ω_k of posemb_sincos_2d_xy(C=128) as the reference computes it in float32 (utils/misc.py:18-19)."""
    omega = torch.arange(LATENT // 4) / (LATENT // 4 - 1)
    return 1.0 / (10000 ** omega)


def native_weights(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """State dict -> {name under "ppp.": tensor} in the layouts csrc/pips_plus_plus.cu and the stride-8 fnet read."""
    out: Dict[str, torch.Tensor] = {"fnet.tc_flag": torch.zeros(1, dtype=torch.int32), "omega": posemb_omega()}
    for k, v in sd.items():
        v = v.detach().float().cpu()
        if k.startswith("fnet.") and k.endswith(".weight"):
            # tensor-core encoder path (conv_by_name): [Cout, 2*Kp] fp16 hi|lo, k = (r*S + s)*Cin + ci
            w = v.permute(0, 2, 3, 1).reshape(v.shape[0], -1)
            kp = -(-w.shape[1] // 64) * 64
            wp = torch.zeros((w.shape[0], kp))
            wp[:, : w.shape[1]] = w
            hi = wp.half()
            out[k[: -len(".weight")] + ".w16"] = torch.cat([hi, (wp - hi.float()).half()], dim=1).contiguous()
        elif k.startswith("delta_block.") and k.endswith("conv.weight"):
            # Conv1d (Cout, Cin, 3) -> [Cout, 2*Kp], column tap*Cin + ci (the temporal im2col order)
            wm = v.double().permute(0, 2, 1).reshape(v.shape[0], -1)
            out[k[: -len(".weight")] + ".w16"], out[k[: -len(".weight")] + ".w16s"] = split_scaled(wm, -(-wm.shape[1] // 64) * 64)
        elif k == "delta_block.dense.weight":
            wm = torch.zeros((DENSE_ROWS, v.shape[1]), dtype=torch.float64)
            wm[:2] = v.double()
            out["delta_block.dense.w16"], out["delta_block.dense.w16s"] = split_scaled(wm, v.shape[1])
        elif k == "delta_block.dense.bias":
            b = torch.zeros(DENSE_ROWS)
            b[:2] = v
            out[k] = b
        else:
            out[k] = v.contiguous()
    return out


class PipsPlusPlus(nn.Module):
    """Reference signature `PipsPlusPlus(stride=8)` (pips_plus_plus.py:421)."""

    def __init__(self, stride=8):
        super().__init__()
        if int(stride) != 8:
            raise NotImplementedError(f"the H100 PIPS++ path is built for stride 8 (PipsPlusPlus' default), got {stride}")
        self.stride = 8
        self.hidden_dim = 256
        self.latent_dim = LATENT
        self.corr_levels = 4
        self.corr_radius = 3
        build_param_tree(self, state_dict_shapes(), seed=206)
        self._registered = None

    @property
    def device(self) -> torch.device:
        return self.norm.weight.device

    # ------------------------------------------------------------------ weights -> libsampt_b200
    def native_context(self) -> native.Context:
        dev = self.device
        ctx = native.get_context(dev)
        key = (id(ctx), tuple(p._version for p in self.parameters()), dev)
        if self._registered != key or not ctx.owns("ppp", self):
            torch.cuda.synchronize(dev)   # nothing may still be reading the tensors this replaces
            ctx.unset_prefix(PREFIX)
            for k, v in native_weights(self.state_dict()).items():
                ctx.set_tensor(PREFIX + k, v)
            self._registered = key
            ctx.claim("ppp", self)
        return ctx

    # ------------------------------------------------------------------ building blocks used by the tracker
    @staticmethod
    def check_frame_size(H: int, W: int) -> None:
        """The coarsest correlation level needs 2 rows and 2 columns: with one, bilinear_sampler divides by H-1 = 0 and the
        reference returns all-NaN trajectories (frames below 128 px)."""
        if (H // 8) >> 3 < 2 or (W // 8) >> 3 < 2:
            raise ValueError(f"PIPS++ needs frames of at least 128x128 px (the coarsest correlation level of a {H}x{W} frame "
                             f"has {(H // 8) >> 3} x {(W // 8) >> 3} cells); the reference returns NaN trajectories here")

    def encode_frames(self, frames: torch.Tensor):
        """(T,3,H,W) uint8, or float32 holding 0..255 -> channels-last pyramid [(T,H/8,W/8,128), /2, /4, /8]."""
        assert frames.is_cuda and frames.dtype in (torch.uint8, torch.float32)
        ctx = self.native_context()
        T, _, H, W = frames.shape
        self.check_frame_size(H, W)
        H8, W8 = H // 8, W // 8
        pyr = [torch.empty((T, H8 >> l, W8 >> l, LATENT), device=frames.device, dtype=torch.float32) for l in range(4)]
        native.check(native.lib().sampt_pips_plus_plus_fnet(ctx.handle, native.ptr(frames.contiguous()),
                                                            c_int(int(frames.dtype == torch.float32)), c_int(T), c_int(H), c_int(W),
                                                            native.ptr(pyr[0]), native.stream_ptr()), "pips_plus_plus_fnet")
        native.check(native.lib().sampt_pips_pyramid(ctx.handle, native.ptr(pyr[0]), c_int(T), c_int(H8), c_int(W8),
                                                     native.ptr(pyr[1]), native.ptr(pyr[2]), native.ptr(pyr[3]),
                                                     native.stream_ptr()), "pips_pyramid")
        return pyr

    def track(self, pyr, query_xy: torch.Tensor, t0: int, direction: int, n_frames: int, max_len: int, iters: int):
        """One direction of PipsPlusPlusPointTracker._forward: query_xy (N,2) px at pyramid frame t0 -> (n_frames,N,2) px for
        frames t0, t0 + direction, ... (pass order)."""
        ctx = self.native_context()
        _, H8, W8, _ = pyr[0].shape
        q = query_xy.detach().float().contiguous()
        N = q.shape[0]
        traj = torch.empty((n_frames, N, 2), device=q.device, dtype=torch.float32)
        native.check(native.lib().sampt_pips_plus_plus_track(
            ctx.handle, native.ptr(pyr[0]), native.ptr(pyr[1]), native.ptr(pyr[2]), native.ptr(pyr[3]), c_int(H8), c_int(W8),
            c_int(t0), c_int(direction), c_int(n_frames), native.ptr(q), c_int(N), c_int(max_len), c_int(self.stride),
            c_int(iters), native.ptr(traj), native.stream_ptr()), "pips_plus_plus_track")
        return traj

    # ------------------------------------------------------------------ reference-compatible forward
    def forward(self, trajs_e0, rgbs, iters=3, trajs_g=None, vis_g=None, valids=None, sw=None, feat_init=None, is_train=False,
                beautify=False):
        """Reference `PipsPlusPlus.forward` (pips_plus_plus.py:436-546), inference, one window of S >= 2 frames.
        trajs_e0 (1,S,N,2) px, rgbs (1,S,3,H,W) 0..255, feat_init None or 3 tensors (1,S,N,128) ->
        (coord_predictions1: `iters` tensors (1,S,N,2) before frame 0 is re-locked, then the final locked coords;
        coord_predictions2: the initial coords, the locked coords of every iteration, the final coords again;
        feats: (feats1, feats2, feats4), each (1,S,N,128); loss None).  One native window call after the encoder."""
        if trajs_g is not None or is_train or self.training or beautify or (sw is not None and getattr(sw, "save_this", False)):
            raise NotImplementedError("H100 PipsPlusPlus.forward covers inference (no losses / training / summaries / beautify)")
        B, S, N, D = trajs_e0.shape
        assert D == 2
        if B != 1 or rgbs.shape[0] != 1:
            raise NotImplementedError("Batch size > 1 is not supported for PIPS++ yet")
        assert rgbs.shape[1] == S
        dev = self.device
        frames = rgbs[0].to(dev)
        if frames.dtype != torch.uint8:
            frames = frames.float()
        pyr = self.encode_frames(frames)
        ctx = self.native_context()
        H8, W8 = pyr[0].shape[1:3]
        t0 = trajs_e0[0].detach().float().to(dev).contiguous()
        fi = None
        if feat_init is not None:
            fi = torch.stack([f[0].detach().float().to(dev) for f in feat_init], dim=0).contiguous()
        coords = torch.empty((iters + 1, S, N, 2), device=dev, dtype=torch.float32)
        feats = torch.empty((3, S, N, LATENT), device=dev, dtype=torch.float32)
        native.check(native.lib().sampt_pips_plus_plus_window(
            ctx.handle, native.ptr(pyr[0]), native.ptr(pyr[1]), native.ptr(pyr[2]), native.ptr(pyr[3]), c_int(H8), c_int(W8),
            native.ptr(t0), native.ptr(fi), c_int(N), c_int(S), c_int(self.stride), c_int(iters), native.ptr(coords),
            native.ptr(feats), native.stream_ptr()), "pips_plus_plus_window")
        preds1 = [coords[i][None] for i in range(iters + 1)]
        init = t0[None]
        # (trajs_e0 / 8) * 8 == trajs_e0 exactly: the locked frame 0 of every coord_predictions2 entry is the input's frame 0
        preds2 = [init] + [torch.cat([init[:, :1], p[:, 1:]], dim=1) for p in preds1[:iters]] + [preds1[-1]]
        return preds1, preds2, tuple(feats[b][None] for b in range(3)), None


def resize_frames(model: PipsPlusPlus, frames: torch.Tensor, size) -> torch.Tensor:
    """F.interpolate(rgbs / 255, size, mode="bilinear") * 255 of PipsPlusPlusPointTracker.forward (tracker.py:72-77) on uint8 or
    float32 frames (T,3,H,W) -> float32 (T,3,*size), align_corners=False."""
    assert frames.dtype in (torch.uint8, torch.float32)
    ctx = model.native_context()
    T, C, H, W = frames.shape
    Ho, Wo = size
    out = torch.empty((T, C, Ho, Wo), device=frames.device, dtype=torch.float32)
    native.check(native.lib().sampt_pips_plus_plus_resize(ctx.handle, native.ptr(frames.contiguous()),
                                                          c_int(int(frames.dtype == torch.float32)), c_int(T * C), c_int(H), c_int(W),
                                                          c_int(Ho), c_int(Wo), native.ptr(out), native.stream_ptr()), "pips_plus_plus_resize")
    return out
