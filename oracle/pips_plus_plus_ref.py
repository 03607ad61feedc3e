"""ORACLE (test infrastructure, NOT product code): CPU restatement of PIPS++ and PipsPlusPlusPointTracker.

Restates, as pure functions over the PipsPlusPlus state dict, in the dtype and on the device of the inputs (float32 or
float64):

* ``PipsPlusPlus.forward``   /root/reference/sam_pt/point_tracker/pips_plus_plus/pips_plus_plus.py:436-546
* ``DeltaBlock`` / ``ResidualBlock1d`` / ``Conv1dPad``  pips_plus_plus.py:12-105,262-337
* ``CorrBlock``              pips_plus_plus.py:363-417 (dense formulation, as the reference executes it)
* ``posemb_sincos_2d_xy``    utils/misc.py:10-27
* ``PipsPlusPlusPointTracker``  pips_plus_plus/tracker.py:25-134; ``intent=True`` replaces the reference's two failure
  modes (IndexError with two or more query timesteps, T-1 frames for a query on the last frame) by each point's own stitched
  trajectory, as the drop-in does.  With ``intent=False`` the T-1 frames are reproduced, but the IndexError is SIMULATED: it
  is raised by hand whenever there are two or more query timesteps, not by restating the reference's indexing (the reference's
  own failure is pinned by the golden's recorded error).

The BasicEncoder and ``bilinear_sample2d`` are PIPS's (oracle/pips_ref.py), at stride 8.

PINNED: ``tests/golden/make_golden_pips_plus_plus.py`` runs the UNMODIFIED reference on CPU on seeded inputs and stores the
outputs under ``tests/golden/``; ``tests/test_oracle_pips_plus_plus.py`` checks this restatement against them.
"""
from __future__ import annotations

from collections import defaultdict
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

from oracle.pips_ref import bilinear_sample2d, build_pyramid, fnet

SD = Dict[str, torch.Tensor]
LATENT = 128
BLOCK_CHANNELS = ((128, 128), (128, 128), (128, 256), (256, 256), (256, 512), (512, 512), (512, 1024), (1024, 1024))


def posemb_sincos_2d_xy(xy, C: int = LATENT, temperature: float = 10000):
    """utils/misc.py:10-27 with cat_coords=True: xy (B,S,2) -> (B,S,C+2)."""
    B, S, _ = xy.shape
    omega = torch.arange(C // 4, device=xy.device) / (C // 4 - 1)
    omega = (1.0 / (temperature ** omega)).to(xy.dtype)
    y = xy[:, :, 1].flatten()[:, None] * omega[None, :]
    x = xy[:, :, 0].flatten()[:, None] * omega[None, :]
    pe = torch.cat((x.sin(), x.cos(), y.sin(), y.cos()), dim=1).reshape(B, S, C)
    return torch.cat([pe, xy], dim=2)


def _conv1d(sd: SD, name: str, x):
    return F.conv1d(F.pad(x, (1, 1)), sd[name + ".conv.weight"].to(x.dtype), sd[name + ".conv.bias"].to(x.dtype))


def _inorm1d(x):
    return F.instance_norm(x, eps=1e-5)


def residual_block(sd: SD, i: int, x):
    """ResidualBlock1d i on x (B, Cin, S) (pips_plus_plus.py:77-105)."""
    ci, co = BLOCK_CHANNELS[i]
    p = f"delta_block.basicblock_list.{i}."
    out = x if i == 0 else F.relu(_inorm1d(x))
    out = _conv1d(sd, p + "conv1", out)
    out = _conv1d(sd, p + "conv2", F.relu(_inorm1d(out)))
    identity = x
    if co != ci:
        ch1 = (co - ci) // 2
        identity = F.pad(x, (0, 0, ch1, co - ci - ch1))
    return out + identity


def delta_block_rows(sd: SD, rows):
    """DeltaBlock after the input concat: rows (B*N, S, 718) -> delta (B*N, S, 2) (pips_plus_plus.py:326-337)."""
    out = F.relu(_conv1d(sd, "delta_block.first_block_conv", rows.permute(0, 2, 1)))
    for i in range(len(BLOCK_CHANNELS)):
        out = residual_block(sd, i, out)
    out = F.relu(out).permute(0, 2, 1)
    return F.linear(out, sd["delta_block.dense.weight"].to(rows.dtype), sd["delta_block.dense.bias"].to(rows.dtype))


def corr_sample(pyr: List[torch.Tensor], targets, coords, radius: int = 3):
    """CorrBlock.corr(targets) + CorrBlock.sample(coords) (pips_plus_plus.py:378-417): targets (B,S,N,C), coords (B,S,N,2) ->
    (B,S,N,4*49); the 7x7 window is TRANSPOSED (x takes the row offset)."""
    B, S, N, C = targets.shape
    r = radius
    dt, dev = targets.dtype, targets.device
    out = []
    for i, fm in enumerate(pyr):
        H, W = fm.shape[-2:]
        corrs = torch.matmul(targets, fm.reshape(B, S, C, H * W)).view(B, S, N, H, W)
        corrs = corrs / torch.sqrt(torch.tensor(C, dtype=dt, device=dev))
        d = torch.linspace(-r, r, 2 * r + 1, dtype=dt, device=dev)
        delta = torch.stack(torch.meshgrid(d, d, indexing="ij"), dim=-1)
        cl = coords.reshape(B * S * N, 1, 1, 2) / 2 ** i + delta.view(1, 2 * r + 1, 2 * r + 1, 2)
        xg = 2 * cl[..., 0:1] / (W - 1) - 1
        yg = 2 * cl[..., 1:2] / (H - 1) - 1
        samp = F.grid_sample(corrs.reshape(B * S * N, 1, H, W), torch.cat([xg, yg], dim=-1), align_corners=True)
        out.append(samp.view(B, S, N, -1))
    return torch.cat(out, dim=-1)


def input_rows(pyr, feats1, feats2, feats4, coords):
    """The 718-column DeltaBlock input (B*N, S, 718): [corr1 | corr2 | corr4 | posemb(flow) | flow]."""
    B, S, N, _ = coords.shape
    fc = [corr_sample(pyr, f, coords).permute(0, 2, 1, 3).reshape(B * N, S, -1) for f in (feats1, feats2, feats4)]
    flows = (coords[:, 1:] - coords[:, :-1]).permute(0, 2, 1, 3).reshape(B * N, S - 1, 2)
    flows = torch.cat([flows, flows[:, -1:]], dim=1)
    return torch.cat(fc + [posemb_sincos_2d_xy(flows)], dim=2)


def sample_targets(fmaps, coords, inds):
    """feats (B,S,N,C) = bilinear_sample2d of frame inds[s] at coords[:, inds[s]] (pips_plus_plus.py:490-504)."""
    B, S, N, _ = coords.shape
    C, H8, W8 = fmaps.shape[2:]
    c_ = coords[:, inds].reshape(B * S, N, 2)
    f_ = fmaps[:, inds].reshape(B * S, C, H8, W8)
    return bilinear_sample2d(f_, c_[:, :, 0], c_[:, :, 1]).permute(0, 2, 1).reshape(B, S, N, C)


@torch.no_grad()
def pips_plus_plus_forward(sd: SD, trajs_e0, rgbs=None, iters: int = 3, feat_init=None, stride: int = 8, fmaps=None,
                           taps: Optional[dict] = None):
    """trajs_e0 (B,S,N,2) px, rgbs (B,S,3,H,W) 0..255 (or fmaps (B,S,128,H/8,W/8)) -> (coord_predictions1, coord_predictions2,
    (feats1, feats2, feats4)) exactly as the reference returns them (pips_plus_plus.py:483-546)."""
    dt = trajs_e0.dtype
    B, S, N, _ = trajs_e0.shape
    if fmaps is None:
        _, _, C, H, W = rgbs.shape
        x = 2 * (rgbs.to(dt) / 255.0) - 1.0
        fmaps = fnet(sd, x.reshape(B * S, C, H, W), stride).reshape(B, S, LATENT, H // stride, W // stride)
    coords = trajs_e0.clone() / float(stride)
    pyr = build_pyramid(fmaps)
    if feat_init is not None:
        feats1, feats2, feats4 = feat_init
    else:
        feat1 = bilinear_sample2d(fmaps[:, 0], coords[:, 0, :, 0], coords[:, 0, :, 1]).permute(0, 2, 1)
        feats1 = feats2 = feats4 = feat1.unsqueeze(1).repeat(1, S, 1, 1)
    coords_bak = coords.clone()
    preds1, preds2 = [], [coords * stride]
    for itr in range(iters):
        if itr >= 1:
            feats2 = sample_targets(fmaps, coords, (torch.arange(S) - 2).clip(min=0))
            feats4 = sample_targets(fmaps, coords, (torch.arange(S) - 4).clip(min=0))
        rows = input_rows(pyr, feats1, feats2, feats4, coords)
        delta = delta_block_rows(sd, rows)
        if taps is not None:
            taps.setdefault("rows", []).append(rows.clone())
            taps.setdefault("delta", []).append(delta.clone())
        coords = coords + delta.reshape(B, N, S, 2).permute(0, 2, 1, 3)
        preds1.append(coords * stride)
        coords[:, 0] = coords_bak[:, 0]
        preds2.append(coords * stride)
    preds2.append(coords * stride)
    preds1.append(coords * stride)
    return preds1, preds2, (feats1, feats2, feats4)


@torch.no_grad()
def track_one_direction(sd: SD, fmaps, query_xy, max_len: int = 128, iters: int = 16, stride: int = 8):
    """PipsPlusPlusPointTracker._forward (tracker.py:25-65) on per-frame features fmaps (1,T,128,H/8,W/8) of the pass (already
    in pass order); query_xy (N,2) -> (1,T,N,2)."""
    T = fmaps.shape[1]
    trajs = query_xy[None, None].repeat(1, T, 1, 1).clone()
    cur, feat_init = 0, None
    while True:
        end = cur + max_len
        if end > T:
            diff = end - T
            end -= diff
            cur = max(cur - diff, 0)
        S_local = end - cur
        if feat_init is not None:
            feat_init = [fi[:, :S_local] for fi in feat_init]
        preds, _, feat_init = pips_plus_plus_forward(sd, trajs[:, cur:end], None, iters, feat_init, stride,
                                                     fmaps=fmaps[:, cur:end])
        trajs[:, cur:end] = preds[-1][:, :S_local]
        trajs[:, end:] = trajs[:, end - 1:end]
        if end >= T:
            return trajs
        cur = cur + max_len - 1


@torch.no_grad()
def pips_plus_plus_tracker_forward(sd: SD, rgbs, query_points, max_len: int = 128, iters: int = 16, image_size=None,
                                   intent: bool = True, stride: int = 8):
    """PipsPlusPlusPointTracker.forward (tracker.py:67-134), computed in the dtype of `query_points`.  rgbs (1,T,3,H,W) 0..255.
    The encoder runs once per frame (each image is independent).  intent=False reproduces the reference's failures."""
    dt = query_points.dtype
    B, T, C, H, W = rgbs.shape
    query_points = query_points.clone()
    rgbs = rgbs.to(dt)
    if image_size is not None:
        r = F.interpolate(rgbs.reshape(B * T, C, H, W) / 255.0, size=tuple(image_size), mode="bilinear") * 255.0
        rgbs = r.reshape(B, T, C, *image_size)
        query_points[:, :, 1] *= image_size[0] / H
        query_points[:, :, 2] *= image_size[1] / W
    x = 2 * (rgbs[0] / 255.0) - 1.0
    fm = torch.cat([fnet(sd, x[i:i + 1], stride) for i in range(T)], dim=0)[None]
    groups = defaultdict(list)
    for idx, point in enumerate(query_points[0]):
        groups[int(point[0].item())].append(idx)
    N = query_points.shape[1]
    out = {}
    for t, idx in groups.items():
        q = query_points[0, idx, 1:]
        if t == T - 1:
            left = q[None, None] if intent else q[None, None][:, :0]
        else:
            left = track_one_direction(sd, fm[:, t:], q, max_len, iters, stride)
        if t == 0:
            right = q[None, None][:, :0]
        else:
            right = track_one_direction(sd, fm[:, :t + 1].flip(1), q, max_len, iters, stride).flip(1)
        traj = torch.cat([right[:, :-1], left], dim=1)
        for j, i in enumerate(idx):
            if not intent and len(groups) > 1:   # simulated, see the module docstring
                raise IndexError("reference tracker.py:120-122 indexes the group's trajectories with the global point index")
            out[i] = traj[:, :, j]
    traj = torch.stack([out[i] for i in range(N)], dim=2)
    if image_size is not None:
        traj[:, :, :, 0] *= H / image_size[0]
        traj[:, :, :, 1] *= W / image_size[1]
    return traj, torch.ones_like(traj[:, :, :, 0])
