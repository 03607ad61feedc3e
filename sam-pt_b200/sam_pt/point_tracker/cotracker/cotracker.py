"""`CoTracker` (cotracker_stride_4_wind_8) with upstream's state-dict key names whose arithmetic runs in libsampt_b200
(csrc/cotracker.cu).  Upstream: facebookresearch/co-tracker @ 4f297a9, cotracker/models/core/cotracker/cotracker.py
(un-vendored dependency of the reference, requirements.txt:31; SURVEY Appendix B.3).  PARITY UNPINNED: the reference
holds no golden vectors for this model, see oracle/cotracker_ref.py.

Host side = window bookkeeping of upstream `CoTracker.forward` (sorting queries by birth frame, growing the active point set,
carrying coordinates / visibilities from one window into the next); every floating-point stage is a native kernel:
encoder (shared with PIPS, tensor-core convolutions), pyramid, correlation gather, embeddings, UpdateFormer, updates."""
from __future__ import annotations

import os
from ctypes import c_int
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch
from torch import nn

from sampt_b200 import native
from sampt_b200.param_tree import build_param_tree

LATENT = 128
IN_DIM = 456
HIDDEN = 384
S_WIN = 8
STRIDE = 4


def cotracker_shapes(time_depth: int = 6, space_depth: int = 6) -> Dict[str, Tuple[int, ...]]:
    """state-dict table of upstream `CoTracker(stride=4, S=8)`: BasicEncoder + UpdateFormer(6 time / 6 space blocks, hidden
    384, 8 heads, mlp x4, LayerNorms without affine) + norm / ffeat_updater / vis_predictor."""
    s: Dict[str, Tuple[int, ...]] = {}

    def conv(name, co, ci, k):
        s[f"{name}.weight"] = (co, ci, k, k)
        s[f"{name}.bias"] = (co,)

    def lin(name, o, i):
        s[f"{name}.weight"] = (o, i)
        s[f"{name}.bias"] = (o,)

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
    lin("updateformer.input_transform", HIDDEN, IN_DIM)
    lin("updateformer.flow_head", LATENT + 2, HIDDEN)
    for kind, depth in (("time_blocks", time_depth), ("space_blocks", space_depth)):
        for i in range(depth):
            p = f"updateformer.{kind}.{i}."
            lin(p + "attn.qkv", 3 * HIDDEN, HIDDEN)
            lin(p + "attn.proj", HIDDEN, HIDDEN)
            lin(p + "mlp.fc1", 4 * HIDDEN, HIDDEN)
            lin(p + "mlp.fc2", HIDDEN, 4 * HIDDEN)
    s["norm.weight"] = s["norm.bias"] = (LATENT,)
    lin("ffeat_updater.0", LATENT, LATENT)
    lin("vis_predictor.0", 1, LATENT)
    return s


def _time_embed_table(dim: int, S: int) -> torch.Tensor:
    """upstream get_1d_sincos_pos_embed_from_grid(456, arange(S)): [sin | cos] of t * 10000^(-k/(dim/2)), float64 -> float32."""
    omega = 1.0 / 10000 ** (np.arange(dim // 2, dtype=np.float64) / (dim / 2.0))
    out = np.einsum("m,d->md", np.arange(S, dtype=np.float64), omega)
    return torch.from_numpy(np.concatenate([np.sin(out), np.cos(out)], axis=1)).float()


class CoTracker(nn.Module):
    def __init__(self, S=8, stride=4, add_space_attn=True, num_heads=8, hidden_size=384, space_depth=6, time_depth=6):
        super().__init__()
        if (S, stride, add_space_attn, num_heads, hidden_size) != (8, 4, True, 8, 384):
            raise NotImplementedError("the H100 CoTracker path is built for cotracker_stride_4_wind_8 "
                                      "(configs/model/point_tracker/cotracker.yaml:2)")
        self.S, self.stride = S, stride
        self.latent_dim = LATENT
        self.time_depth, self.space_depth = time_depth, space_depth
        build_param_tree(self, cotracker_shapes(time_depth, space_depth), seed=774411)
        self._registered_on = None
        self.fnet_on_tensor_cores = os.environ.get("SAMPT_PIPS_TC", "1") != "0"

    # ------------------------------------------------------------------ weights -> kernel-native layouts ("cot.*")
    def native_context(self) -> native.Context:
        dev = self.norm.weight.device
        ctx = native.get_context(dev)
        key = (id(ctx), tuple(p._version for p in self.parameters()), dev, self.fnet_on_tensor_cores)
        if self._registered_on != key or not ctx.owns("cot", self):
            torch.cuda.synchronize(dev)  # nothing may still be reading the tensors this replaces
            ctx.set_tensor("cot.fnet.tc_flag", torch.zeros(1 if self.fnet_on_tensor_cores else 2, dtype=torch.int32, device=dev))
            for k, v in self.state_dict().items():
                v = v.detach().float()
                if k.startswith("fnet.") and k.endswith(".weight") and v.dim() == 4:
                    ctx.set_tensor(f"cot.{k}_rsck", v.permute(2, 3, 1, 0).contiguous())
                    if self.fnet_on_tensor_cores:
                        w = v.permute(0, 2, 3, 1).reshape(v.shape[0], -1)
                        kp = -(-w.shape[1] // 64) * 64
                        wp = torch.zeros((w.shape[0], kp), device=w.device)
                        wp[:, : w.shape[1]] = w
                        hi = wp.half()
                        lo = (wp - hi.float()).half()
                        ctx.set_tensor(f"cot.{k[:-len('.weight')]}.w16", torch.cat([hi, lo], dim=1).contiguous())
                else:
                    ctx.set_tensor(f"cot.{k}", v.contiguous())
                    # UpdateFormer linear layers also as fp16 hi | lo [N, 2K] for the three-pass tensor-core GEMM (csrc/cotracker.cu: cot_tcg)
                    if k.startswith("updateformer.") and k.endswith(".weight") and ("_blocks." in k) and v.dim() == 2:
                        hi = v.half()
                        lo = (v - hi.float()).half()
                        ctx.set_tensor(f"cot.{k[:-len('.weight')]}.w16", torch.cat([hi, lo], dim=1).contiguous())
            ctx.set_tensor("cot.time_emb", _time_embed_table(IN_DIM, self.S).to(dev))
            self._time_emb = ctx._tensors["cot.time_emb"]
            self._registered_on = key
            ctx.claim("cot", self)
        return ctx

    # ------------------------------------------------------------------ per-frame work
    def fnet_frames(self, frames_f32: torch.Tensor) -> torch.Tensor:
        """(n,3,H,W) float32 0..255 -> (n,H/4,W/4,128) channels-last BasicEncoder features (once per frame)."""
        assert frames_f32.dtype == torch.float32 and frames_f32.is_cuda
        ctx = self.native_context()
        T, _, H, W = frames_f32.shape
        fm = torch.empty((T, H // 4, W // 4, LATENT), device=frames_f32.device, dtype=torch.float32)
        if T > 0:
            native.check(native.lib().sampt_cotracker_fnet(ctx.handle, native.ptr(frames_f32.contiguous()), c_int(T), c_int(H), c_int(W),
                                                           native.ptr(fm), native.stream_ptr()), "cotracker_fnet")
        return fm

    def build_pyramid(self, fm: torch.Tensor) -> List[torch.Tensor]:
        """(T,H4,W4,128) -> [level0, /2, /4, /8] (upstream CorrBlock avg-pool pyramid)."""
        ctx = self.native_context()
        T, H4, W4, _ = fm.shape
        pyr = [fm.contiguous()] + [torch.empty((T, H4 >> l, W4 >> l, LATENT), device=fm.device, dtype=torch.float32) for l in range(1, 4)]
        native.check(native.lib().sampt_pips_pyramid(ctx.handle, native.ptr(pyr[0]), c_int(T), c_int(H4), c_int(W4),
                                                     native.ptr(pyr[1]), native.ptr(pyr[2]), native.ptr(pyr[3]),
                                                     native.stream_ptr()), "pyramid")
        return pyr

    def encode_frames(self, frames_f32: torch.Tensor) -> List[torch.Tensor]:
        """(T,3,H,W) float32 0..255 -> channels-last pyramid [(T,H/4,W/4,128), /2, /4, /8]."""
        return self.build_pyramid(self.fnet_frames(frames_f32))

    # ------------------------------------------------------------------ upstream CoTracker.forward on pre-computed features
    def track(self, pyr: Sequence[torch.Tensor], queries: torch.Tensor, order: Sequence[int], iters: int = 6):
        """queries (N,3)=(t,x,y) in the pixels of the encoded clip, `t` indexing `order`; `order[i]` = index into the pyramid's
        frame axis of the clip's i-th frame (identity for the forward pass, reversed for the backward pass, tail repeated
        for clips shorter than S).  Returns traj (T,N,2) px, vis (T,N) sigmoid with T = len(order)."""
        ctx = self.native_context()
        lib = native.lib()
        dev = pyr[0].device
        S, T, N = self.S, len(order), queries.shape[0]
        H4, W4 = pyr[0].shape[1:3]
        q = queries.detach().float().to(dev)
        first = q[:, 0].long()
        sort_inds = torch.sort(first, stable=True)[1]
        inv_sort = torch.argsort(sort_inds)
        first_sorted = first[sort_inds]
        first_host = first_sorted.cpu().tolist()            # the only host read-back: window -> active point count
        order_t = torch.tensor(list(order), dtype=torch.int32, device=dev)
        coords_init = (q[sort_inds, 1:] / float(self.stride))[:, None, :].repeat(1, S, 1).contiguous()   # (N,S,2)
        vis_init = torch.full((N, S), 10.0, device=dev)
        track_mask = torch.arange(T, device=dev)[None, :] >= first_sorted[:, None]                      # (N,T)
        feat_init = torch.empty((N, S, LATENT), device=dev)
        traj_e = torch.zeros((T, N, 2), device=dev)
        vis_e = torch.zeros((T, N), device=dev)
        # frame index feeding every slot of every window, uploaded once
        starts = list(range(0, max(T - S // 2, 0), S // 2))
        win_idx = [[min(i + s, T - 1) for s in range(S)] for i in starts]
        fidx_all = torch.tensor([[0, 0] + [order[j] for j in w] for w in win_idx], dtype=torch.int32, device=dev)
        sample_frame = order_t[first_sorted]
        sample_xy = coords_init[:, 0].contiguous()
        prev_wind, coords, vis = 0, None, None
        for wi, ind in enumerate(starts):
            s_local = min(ind + S, T) - ind
            wind = sum(1 for f in first_host if f < ind + S)   # first_host is sorted ascending
            if wind == 0:
                continue
            if wind > prev_wind:
                n_new = wind - prev_wind
                native.check(lib.sampt_cotracker_sample_features(
                    ctx.handle, native.ptr(pyr[0]), c_int(H4), c_int(W4), native.ptr(sample_frame[prev_wind:wind].contiguous()),
                    native.ptr(sample_xy[prev_wind:wind].contiguous()), c_int(n_new), c_int(S), native.ptr(feat_init[prev_wind:wind]),
                    native.stream_ptr()), "cotracker_sample_features")
            if prev_wind > 0:
                coords_init[:prev_wind, : S // 2] = coords[:, S // 2:]
                coords_init[:prev_wind, S // 2:] = coords[:, -1:]
                vis_init[:prev_wind, : S // 2] = vis[:, S // 2:]
                vis_init[:prev_wind, S // 2:] = vis[:, -1:]
            coords = coords_init[:wind].clone()
            ffeats = feat_init[:wind].clone()
            tm = torch.zeros((wind, S), device=dev)
            tm[:, :s_local] = track_mask[:wind, ind:ind + S].float()
            vi = vis_init[:wind].contiguous()
            vis = torch.empty((wind, S), device=dev)
            native.check(lib.sampt_cotracker_window(
                ctx.handle, native.ptr(pyr[0]), native.ptr(pyr[1]), native.ptr(pyr[2]), native.ptr(pyr[3]), c_int(H4), c_int(W4),
                native.ptr(fidx_all[wi]), native.ptr(coords), native.ptr(ffeats), native.ptr(tm), native.ptr(vi),
                native.ptr(self._time_emb), c_int(wind), c_int(iters), c_int(self.time_depth), c_int(self.space_depth),
                native.ptr(vis), native.stream_ptr()), "cotracker_window")
            traj_e[ind:ind + s_local, :wind] = (coords[:, :s_local] * float(self.stride)).permute(1, 0, 2)
            vis_e[ind:ind + s_local, :wind] = vis[:, :s_local].t()
            track_mask[:wind, : ind + S] = False
            prev_wind = wind
        return traj_e[:, inv_sort], torch.sigmoid(vis_e[:, inv_sort])

    def forward(self, rgbs, queries, iters=4, feat_init=None, is_train=False):
        """Upstream signature; rgbs (1,T,3,H,W) float 0..255, queries (1,N,3) -> (traj (1,T,N,2), feat_init, vis (1,T,N), None)."""
        if feat_init is not None or is_train:
            raise NotImplementedError("H100 CoTracker covers inference with feat_init=None")
        if rgbs.shape[0] != 1:
            raise NotImplementedError("batch size 1 (the SAM-PT hot path tracks one clip at a time)")
        T = rgbs.shape[1]
        assert T >= self.S, "clips shorter than the window are padded by CoTrackerForShortVideosWrapper"
        pyr = self.encode_frames(rgbs[0].float().to(self.norm.weight.device))
        traj, vis = self.track(pyr, queries[0], list(range(T)), iters=iters)
        return traj[None], None, vis[None], None
