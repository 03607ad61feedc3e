"""ORACLE (test infrastructure, NOT product code): CPU restatement of CoTracker v1 + the reference's wrapper.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl reference`` leg may import this.

PARITY STATUS: **parity unpinned.**  The model is the un-vendored third-party package ``co-tracker @ 4f297a9``
(``/root/reference/requirements.txt:31``); its source is not in /root/reference, nothing in this image re-implements it
(no cross-check exists, unlike SAM), and the reference holds no golden vectors for it.  This file restates the published
algorithm (CoTracker v1, ``cotracker_stride_4_wind_8``: ``CoTracker(stride=4, S=8, add_space_attn=True, space_depth=6,
time_depth=6)``; SURVEY.md Appendix B.3) from the upstream code as of that commit, to the best of the author's knowledge;
details that could not be verified are marked [unverified].  The in-tree pieces ARE anchored:

* ``CoTrackerPointTracker.forward``           /root/reference/sam_pt/point_tracker/cotracker/tracker.py:72-152
* ``_compute_backward_tracks``                 tracker.py:154-170
* ``CoTrackerForShortVideosWrapper.__call__``  tracker.py:12-24
* encoder / correlation pyramid / lookup      identical to PIPS (``oracle/pips_ref.py``, pinned to the reference)
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from . import pips_ref

SD = Dict[str, torch.Tensor]
LATENT, HID, HEADS = 128, 384, 8
IN_DIM = 456  # 130 (flow emb) + 196 (corr) + 128 (feat) + 2 (track mask, vis)


# ----------------------------------------------------------------------------- embeddings (upstream models/core/embeddings.py)
def get_2d_embedding(xy, C=64):
    """(B,N,2) -> (B,N,2C+2) = [xy | sincos(x) | sincos(y)]  ([unverified]: coordinate columns first), in xy's dtype."""
    div = (torch.arange(0, C, 2, dtype=xy.dtype, device=xy.device) * (1000.0 / C)).reshape(1, 1, C // 2)
    out = [xy]
    for d in range(2):
        v = xy[:, :, d:d + 1]
        pe = torch.zeros(xy.shape[0], xy.shape[1], C, dtype=xy.dtype, device=xy.device)
        pe[:, :, 0::2] = torch.sin(v * div)
        pe[:, :, 1::2] = torch.cos(v * div)
        out.append(pe)
    return torch.cat(out, dim=2)


def _sincos_1d(embed_dim: int, pos: np.ndarray) -> np.ndarray:
    omega = np.arange(embed_dim // 2, dtype=np.float64)
    omega /= embed_dim / 2.0
    omega = 1.0 / 10000 ** omega
    out = np.einsum("m,d->md", pos.reshape(-1).astype(np.float64), omega)
    return np.concatenate([np.sin(out), np.cos(out)], axis=1)


def get_2d_sincos_pos_embed(embed_dim: int, grid_hw: Tuple[int, int]) -> np.ndarray:
    """MAE-style table (H*W, D): first half from the x (w) coordinate, second half from y (h)."""
    gh, gw = grid_hw
    grid = np.stack(np.meshgrid(np.arange(gw, dtype=np.float32), np.arange(gh, dtype=np.float32)), axis=0)  # (2,H,W): [x, y]
    emb_a = _sincos_1d(embed_dim // 2, grid[0])
    emb_b = _sincos_1d(embed_dim // 2, grid[1])
    return np.concatenate([emb_a, emb_b], axis=1)


def sample_pos_embed(grid_hw, embed_dim, coords0):
    """bilinear sample of the 2-D table (float64, rounded to coords0's dtype) at the window's first-frame coords: (B,N,2) -> (B,N,D)."""
    tab = torch.from_numpy(get_2d_sincos_pos_embed(embed_dim, grid_hw)).to(dtype=coords0.dtype, device=coords0.device)
    tab = tab.reshape(1, grid_hw[0], grid_hw[1], embed_dim)
    s = pips_ref.bilinear_sample2d(tab.permute(0, 3, 1, 2), coords0[:, :, 0], coords0[:, :, 1])
    return s.permute(0, 2, 1)


def time_embed(embed_dim: int, S: int, dtype=torch.float32, device=None):
    return torch.from_numpy(_sincos_1d(embed_dim, np.linspace(0, S - 1, S))).to(dtype=dtype, device=device)  # (S, D)


# ----------------------------------------------------------------------------- UpdateFormer
def _attn_block(sd: SD, p: str, x):
    """x (B, L, 384): pre-LN (no affine, eps 1e-6) -> timm Attention (qkv bias) ; pre-LN -> MLP with tanh-GELU."""
    B, L, C = x.shape
    h = F.layer_norm(x, (C,), None, None, 1e-6)
    qkv = F.linear(h, sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"]).reshape(B, L, 3, HEADS, C // HEADS).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    a = (q @ k.transpose(-2, -1)) * ((C // HEADS) ** -0.5)
    a = a.softmax(dim=-1)
    o = (a @ v).transpose(1, 2).reshape(B, L, C)
    x = x + F.linear(o, sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"])
    h = F.layer_norm(x, (C,), None, None, 1e-6)
    h = F.gelu(F.linear(h, sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"]), approximate="tanh")
    return x + F.linear(h, sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"])


def update_former(sd: SD, x, time_depth=6, space_depth=6, prefix="updateformer."):
    """x (B, N, T, 456) -> (B, N, T, 130): time attention over the T frames of each point interleaved with space attention
    over the N points of each frame."""
    p = prefix
    x = F.linear(x, sd[p + "input_transform.weight"], sd[p + "input_transform.bias"])
    B, N, T, C = x.shape
    j = 0
    for i in range(time_depth):
        xt = _attn_block(sd, f"{p}time_blocks.{i}.", x.reshape(B * N, T, C))
        x = xt.reshape(B, N, T, C)
        if i % (time_depth // space_depth) == 0:
            xs = _attn_block(sd, f"{p}space_blocks.{j}.", x.permute(0, 2, 1, 3).reshape(B * T, N, C))
            x = xs.reshape(B, T, N, C).permute(0, 2, 1, 3)
            j += 1
    return F.linear(x, sd[p + "flow_head.weight"], sd[p + "flow_head.bias"])


# ----------------------------------------------------------------------------- one window (upstream forward_iteration)
def forward_iteration(sd: SD, fmaps, coords_init, feat_init, vis_init, track_mask, iters=6, stride=4, S=8):
    """fmaps (1,S,128,H4,W4); coords_init (1,S,N,2) feature px; feat_init (1,S,N,128); vis_init (1,S,N,1); track_mask (1,<=S,N,1)."""
    B, _, N, _ = coords_init.shape
    H4, W4 = fmaps.shape[-2:]
    coords = coords_init.clone()
    pyr = pips_ref.build_pyramid(fmaps)
    ffeats = feat_init.clone()
    pos = sample_pos_embed((H4, W4), IN_DIM, coords[:, 0])           # (1,N,456)
    pos = pos.reshape(B * N, 1, IN_DIM)
    tim = time_embed(IN_DIM, S, coords.dtype, coords.device)[None]   # (1,S,456)
    if track_mask.shape[1] < S:
        track_mask = torch.cat([track_mask, torch.zeros_like(track_mask[:, :1]).repeat(1, S - track_mask.shape[1], 1, 1)], dim=1)
    preds = []
    for _ in range(iters):
        fcorrs = pips_ref.corr_lookup(pyr, ffeats, coords)            # (1,S,N,196)
        fcorrs_ = fcorrs.permute(0, 2, 1, 3).reshape(B * N, S, -1)
        flows_ = (coords - coords[:, 0:1]).permute(0, 2, 1, 3).reshape(B * N, S, 2)
        flows_cat = get_2d_embedding(flows_, 64)                      # (BN,S,130)
        ffeats_ = ffeats.permute(0, 2, 1, 3).reshape(B * N, S, LATENT)
        concat = torch.cat([track_mask.to(vis_init.dtype), vis_init], dim=3).permute(0, 2, 1, 3).reshape(B * N, S, 2)
        x = torch.cat([flows_cat, fcorrs_, ffeats_, concat], dim=2) + pos + tim
        delta = update_former(sd, x.reshape(B, N, S, IN_DIM)).reshape(B * N, S, LATENT + 2)
        dcoords, dfeats = delta[:, :, :2], delta[:, :, 2:].reshape(B * N * S, LATENT)
        ffeats_ = ffeats_.reshape(B * N * S, LATENT)
        upd = F.gelu(F.linear(F.group_norm(dfeats, 1, sd["norm.weight"], sd["norm.bias"], 1e-5), sd["ffeat_updater.0.weight"],
                              sd["ffeat_updater.0.bias"]))
        ffeats = (upd + ffeats_).reshape(B, N, S, LATENT).permute(0, 2, 1, 3)
        coords = coords + dcoords.reshape(B, N, S, 2).permute(0, 2, 1, 3)
        preds.append(coords * stride)
    vis_e = F.linear(ffeats.reshape(B * S * N, LATENT), sd["vis_predictor.0.weight"], sd["vis_predictor.0.bias"]).reshape(B, S, N)
    return preds, vis_e


# ----------------------------------------------------------------------------- CoTracker.forward (sliding windows, step S/2)
@torch.no_grad()
def cotracker_forward(sd: SD, rgbs, queries, iters=6, stride=4, S=8, fmaps_all: Optional[torch.Tensor] = None):
    """rgbs (1,T,3,H,W) float 0..255 at the interp resolution; queries (1,N,3)=(t,x,y) -> traj (1,T,N,2) px, vis (1,T,N) sigmoid,
    in the dtype and on the device of `queries`.
    `fmaps_all` (T,128,H/4,W/4): encoder output computed once per frame (results-neutral; upstream re-encodes S/2 frames per window)."""
    B, T, C, H, W = rgbs.shape
    N = queries.shape[1]
    assert B == 1
    first = queries[:, :, 0].long()
    sort_inds = torch.sort(first[0], dim=0, descending=False, stable=True)[1]
    inv_sort = torch.argsort(sort_inds, dim=0)
    first_sorted = first[0][sort_inds]
    coords_init = queries[:, :, 1:].reshape(B, 1, N, 2).repeat(1, S, 1, 1) / float(stride)
    if fmaps_all is None:
        x = 2 * (rgbs[0] / 255.0) - 1.0
        fmaps_all = torch.cat([pips_ref.fnet(sd, x[i:i + 1], stride) for i in range(T)], dim=0)
    dt, dev = queries.dtype, queries.device
    traj_e = torch.zeros((B, T, N, 2), dtype=dt, device=dev)
    vis_e = torch.zeros((B, T, N), dtype=dt, device=dev)
    ind_array = torch.arange(T, device=dev).repeat(B, 1)
    track_mask = (ind_array[:, :, None] >= first[:, None, :]).unsqueeze(-1)
    vis_init = torch.ones((B, S, N, 1), dtype=dt, device=dev) * 10
    track_mask_ = track_mask[:, :, sort_inds].clone()
    coords_init_ = coords_init[:, :, sort_inds].clone()
    vis_init_ = vis_init[:, :, sort_inds].clone()
    feat_init = None
    prev_wind_idx = 0
    coords, vis = None, None
    ind = 0
    while ind < T - S // 2:
        idx = list(range(ind, min(ind + S, T)))
        S_local = len(idx)
        idx = idx + [idx[-1]] * (S - S_local)
        fmaps = fmaps_all[idx][None]
        curr = torch.nonzero(first_sorted < ind + S)
        if curr.shape[0] == 0:
            ind += S // 2
            continue
        wind_idx = int(curr[-1]) + 1
        if wind_idx - prev_wind_idx > 0:
            fsel = fmaps[:, first_sorted[prev_wind_idx:wind_idx] - ind]            # (1, n_new, 128, H4, W4)
            c0 = coords_init_[:, 0, prev_wind_idx:wind_idx]
            feats = []
            for j in range(fsel.shape[1]):
                feats.append(pips_ref.bilinear_sample2d(fsel[:, j], c0[:, j:j + 1, 0], c0[:, j:j + 1, 1]).permute(0, 2, 1))
            f_new = torch.cat(feats, dim=1).unsqueeze(1).repeat(1, S, 1, 1)         # (1,S,n_new,128)
            feat_init = f_new if feat_init is None else torch.cat([feat_init, f_new], dim=2)
        if prev_wind_idx > 0:
            new_coords = coords[-1][:, S // 2:] / float(stride)
            coords_init_[:, : S // 2, :prev_wind_idx] = new_coords
            coords_init_[:, S // 2:, :prev_wind_idx] = new_coords[:, -1].repeat(1, S // 2, 1, 1)
            new_vis = vis[:, S // 2:].unsqueeze(-1)
            vis_init_[:, : S // 2, :prev_wind_idx] = new_vis
            vis_init_[:, S // 2:, :prev_wind_idx] = new_vis[:, -1].repeat(1, S // 2, 1, 1)
        coords, vis = forward_iteration(sd, fmaps, coords_init_[:, :, :wind_idx], feat_init[:, :, :wind_idx],
                                        vis_init_[:, :, :wind_idx], track_mask_[:, ind:ind + S, :wind_idx], iters, stride, S)
        traj_e[:, ind:ind + S, :wind_idx] = coords[-1][:, :S_local]
        vis_e[:, ind:ind + S, :wind_idx] = vis[:, :S_local]
        track_mask_[:, : ind + S, :wind_idx] = False
        ind += S // 2
        prev_wind_idx = wind_idx
    traj_e = traj_e[:, :, inv_sort]
    vis_e = torch.sigmoid(vis_e[:, :, inv_sort])
    return traj_e, vis_e


# ----------------------------------------------------------------------------- the reference's wrapper (in-tree, anchored)
def get_points_on_a_grid(grid_size: int, interp_shape: Tuple[int, int]):
    """upstream helper used at cotracker/tracker.py:100: regular grid with a margin of W//64 px; (1, g*g, 2) xy."""
    if grid_size == 1:
        return torch.tensor([interp_shape[1] / 2, interp_shape[0] / 2])[None, None]
    gy, gx = torch.meshgrid(torch.linspace(0, grid_size - 1, grid_size), torch.linspace(0, grid_size - 1, grid_size), indexing="ij")
    step = interp_shape[1] // 64
    gy = step + gy.reshape(1, -1) / float(grid_size - 1) * (interp_shape[0] - step * 2)
    gx = step + gx.reshape(1, -1) / float(grid_size - 1) * (interp_shape[1] - step * 2)
    return torch.stack([gx, gy], dim=-1)


@torch.no_grad()
def cotracker_point_tracker_forward(sd: SD, rgbs_u8, query_points, interp_shape=(384, 512), visibility_threshold=0.7,
                                    support_grid_size=2, support_grid_every_n_frames=12, raw: Optional[dict] = None):
    """CoTrackerPointTracker.forward (cotracker/tracker.py:72-152) incl. the short-clip wrapper and the backward pass."""
    query_points = query_points.float()
    rgbs = rgbs_u8.float()
    B, T, C, H, W = rgbs.shape
    n_points = query_points.shape[1]
    rgbs = F.interpolate(rgbs.reshape(B * T, C, H, W), tuple(interp_shape), mode="bilinear").reshape(B, T, C, *interp_shape)
    q = query_points.clone()
    q[:, :, 1] *= interp_shape[1] / W
    q[:, :, 2] *= interp_shape[0] / H
    if support_grid_size > 0:
        for i in range(0, T, support_grid_every_n_frames):
            g = get_points_on_a_grid(support_grid_size, interp_shape)
            g = torch.cat([i * torch.ones_like(g[:, :, :1]), g], dim=2)
            q = torch.cat([q, g], dim=1)

    def model(r, qq):  # CoTrackerForShortVideosWrapper: pad short clips by repeating the last frame
        n = r.shape[1]
        if n < 8:
            r = torch.cat([r, r[:, -1:].repeat(1, 8 - n, 1, 1, 1)], dim=1)
        t, v = cotracker_forward(sd, r, qq, iters=6)
        return t[:, :n], v[:, :n]

    traj, vis = model(rgbs, q)
    # _compute_backward_tracks (tracker.py:154-170)
    qf = q.clone()
    qf[:, :, 0] = T - qf[:, :, 0] - 1
    traj_f, vis_f = model(rgbs.flip(1).clone(), qf)
    traj_f, vis_f = traj_f.flip(1), vis_f.flip(1)
    mask = traj == 0
    traj[mask] = traj_f[mask]
    vis[mask[:, :, :, 0]] = vis_f[mask[:, :, :, 0]]
    traj = traj[:, :, :n_points].clone()
    if raw is not None:   # the sigmoid values the threshold is applied to (tests: how close to the decision boundary?)
        raw["vis_sigmoid"] = vis[:, :, :n_points].clone()
    vis = vis[:, :, :n_points].clone() > visibility_threshold
    traj[:, :, :, 0] *= W / float(interp_shape[1])
    traj[:, :, :, 1] *= H / float(interp_shape[0])
    return traj, vis


# ----------------------------------------------------------------------------- state-dict shapes
def cotracker_state_dict_shapes(time_depth=6, space_depth=6) -> Dict[str, Tuple[int, ...]]:
    s = {k: v for k, v in pips_ref.pips_state_dict_shapes().items() if k.startswith("fnet.")}
    p = "updateformer."
    s[p + "input_transform.weight"], s[p + "input_transform.bias"] = (HID, IN_DIM), (HID,)
    s[p + "flow_head.weight"], s[p + "flow_head.bias"] = (LATENT + 2, HID), (LATENT + 2,)
    for grp, n in (("time_blocks", time_depth), ("space_blocks", space_depth)):
        for i in range(n):
            b = f"{p}{grp}.{i}."
            s[b + "attn.qkv.weight"], s[b + "attn.qkv.bias"] = (3 * HID, HID), (3 * HID,)
            s[b + "attn.proj.weight"], s[b + "attn.proj.bias"] = (HID, HID), (HID,)
            s[b + "mlp.fc1.weight"], s[b + "mlp.fc1.bias"] = (4 * HID, HID), (4 * HID,)
            s[b + "mlp.fc2.weight"], s[b + "mlp.fc2.bias"] = (HID, 4 * HID), (HID,)
    s["norm.weight"] = s["norm.bias"] = (LATENT,)
    s["ffeat_updater.0.weight"], s["ffeat_updater.0.bias"] = (LATENT, LATENT), (LATENT,)
    s["vis_predictor.0.weight"], s["vis_predictor.0.bias"] = (1, LATENT), (1,)
    return s
