"""The CoTracker oracle follows the dtype and device of its inputs: float64 serves as the reference of the window's kernel tests
(tests/test_gpu_cotracker_kernels.py), and the float32 path, the one the C3 / C5s full-clip goldens were made with, is
bit-identical to the float32-only restatement it replaced (kept below verbatim)."""
from typing import Optional

import numpy as np
import torch
import torch.nn.functional as F

from oracle import cotracker_ref as R
from oracle import pips_ref
from sampt_b200 import synth


def _f32_get_2d_embedding(xy, C=64):
    div = (torch.arange(0, C, 2, dtype=torch.float32) * (1000.0 / C)).reshape(1, 1, C // 2)
    out = [xy]
    for d in range(2):
        v = xy[:, :, d:d + 1]
        pe = torch.zeros(xy.shape[0], xy.shape[1], C)
        pe[:, :, 0::2] = torch.sin(v * div)
        pe[:, :, 1::2] = torch.cos(v * div)
        out.append(pe)
    return torch.cat(out, dim=2)


def _f32_sample_pos_embed(grid_hw, embed_dim, coords0):
    tab = torch.from_numpy(R.get_2d_sincos_pos_embed(embed_dim, grid_hw)).float().reshape(1, grid_hw[0], grid_hw[1], embed_dim)
    s = pips_ref.bilinear_sample2d(tab.permute(0, 3, 1, 2), coords0[:, :, 0], coords0[:, :, 1])
    return s.permute(0, 2, 1)


def _f32_time_embed(embed_dim: int, S: int):
    return torch.from_numpy(R._sincos_1d(embed_dim, np.linspace(0, S - 1, S))).float()  # (S, D)


# ----------------------------------------------------------------------------- one window (upstream forward_iteration)
def _f32_forward_iteration(sd, fmaps, coords_init, feat_init, vis_init, track_mask, iters=6, stride=4, S=8):
    """fmaps (1,S,128,H4,W4); coords_init (1,S,N,2) feature px; feat_init (1,S,N,128); vis_init (1,S,N,1); track_mask (1,<=S,N,1)."""
    B, _, N, _ = coords_init.shape
    H4, W4 = fmaps.shape[-2:]
    coords = coords_init.clone()
    pyr = pips_ref.build_pyramid(fmaps)
    ffeats = feat_init.clone()
    pos = _f32_sample_pos_embed((H4, W4), R.IN_DIM, coords[:, 0])           # (1,N,456)
    pos = pos.reshape(B * N, 1, R.IN_DIM)
    tim = _f32_time_embed(R.IN_DIM, S)[None]                                # (1,S,456)
    if track_mask.shape[1] < S:
        track_mask = torch.cat([track_mask, torch.zeros_like(track_mask[:, :1]).repeat(1, S - track_mask.shape[1], 1, 1)], dim=1)
    preds = []
    for _ in range(iters):
        fcorrs = pips_ref.corr_lookup(pyr, ffeats, coords)            # (1,S,N,196)
        fcorrs_ = fcorrs.permute(0, 2, 1, 3).reshape(B * N, S, -1)
        flows_ = (coords - coords[:, 0:1]).permute(0, 2, 1, 3).reshape(B * N, S, 2)
        flows_cat = _f32_get_2d_embedding(flows_, 64)                      # (BN,S,130)
        ffeats_ = ffeats.permute(0, 2, 1, 3).reshape(B * N, S, R.LATENT)
        concat = torch.cat([track_mask.float(), vis_init], dim=3).permute(0, 2, 1, 3).reshape(B * N, S, 2)
        x = torch.cat([flows_cat, fcorrs_, ffeats_, concat], dim=2) + pos + tim
        delta = R.update_former(sd, x.reshape(B, N, S, R.IN_DIM)).reshape(B * N, S, R.LATENT + 2)
        dcoords, dfeats = delta[:, :, :2], delta[:, :, 2:].reshape(B * N * S, R.LATENT)
        ffeats_ = ffeats_.reshape(B * N * S, R.LATENT)
        upd = F.gelu(F.linear(F.group_norm(dfeats, 1, sd["norm.weight"], sd["norm.bias"], 1e-5), sd["ffeat_updater.0.weight"],
                              sd["ffeat_updater.0.bias"]))
        ffeats = (upd + ffeats_).reshape(B, N, S, R.LATENT).permute(0, 2, 1, 3)
        coords = coords + dcoords.reshape(B, N, S, 2).permute(0, 2, 1, 3)
        preds.append(coords * stride)
    vis_e = F.linear(ffeats.reshape(B * S * N, R.LATENT), sd["vis_predictor.0.weight"], sd["vis_predictor.0.bias"]).reshape(B, S, N)
    return preds, vis_e


# ----------------------------------------------------------------------------- CoTracker.forward (sliding windows, step S/2)
@torch.no_grad()
def _f32_cotracker_forward(sd, rgbs, queries, iters=6, stride=4, S=8, fmaps_all: Optional[torch.Tensor] = None):
    """rgbs (1,T,3,H,W) float 0..255 at the interp resolution; queries (1,N,3)=(t,x,y) -> traj (1,T,N,2) px, vis (1,T,N) sigmoid.
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
    traj_e = torch.zeros((B, T, N, 2))
    vis_e = torch.zeros((B, T, N))
    ind_array = torch.arange(T).repeat(B, 1)
    track_mask = (ind_array[:, :, None] >= first[:, None, :]).unsqueeze(-1)
    vis_init = torch.ones((B, S, N, 1)) * 10
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
        coords, vis = _f32_forward_iteration(sd, fmaps, coords_init_[:, :, :wind_idx], feat_init[:, :, :wind_idx],
                                        vis_init_[:, :, :wind_idx], track_mask_[:, ind:ind + S, :wind_idx], iters, stride, S)
        traj_e[:, ind:ind + S, :wind_idx] = coords[-1][:, :S_local]
        vis_e[:, ind:ind + S, :wind_idx] = vis[:, :S_local]
        track_mask_[:, : ind + S, :wind_idx] = False
        ind += S // 2
        prev_wind_idx = wind_idx
    traj_e = traj_e[:, :, inv_sort]
    vis_e = torch.sigmoid(vis_e[:, :, inv_sort])
    return traj_e, vis_e


def _inputs():
    sd = synth.condition_cotracker(synth.make_state_dict(R.cotracker_state_dict_shapes(), seed=31))
    g = torch.Generator().manual_seed(5)
    T, H4, W4 = 14, 24, 32
    fm = torch.randn((T, 128, H4, W4), generator=g) * 0.5
    q = torch.tensor([[0.0, 20.0, 14.0], [0.0, 41.5, 30.25], [3.0, 2.0, 44.0], [6.0, 60.0, 3.0], [9.0, -3.0, 20.0]])[None]
    return sd, fm, q


def _window(fm, q, S=8):
    N = q.shape[1]
    co = (q[0, :, 1:] / 4.0)[None, None].repeat(1, S, 1, 1)
    co = co + torch.linspace(0, 3, S)[None, :, None, None]            # non-zero flows
    ff = torch.randn((1, 1, N, 128), generator=torch.Generator().manual_seed(2)).repeat(1, S, 1, 1)
    vis = torch.ones((1, S, N, 1)) * 10
    tm = torch.ones((1, 5, N, 1), dtype=torch.bool)                    # short track mask: the zero padding path
    return fm[:S][None], co, ff, vis, tm


def test_cotracker_oracle_float32_bit_identical():
    sd, fm, q = _inputs()
    fw, co, ff, vis, tm = _window(fm, q)
    new = R.forward_iteration(sd, fw, co, ff, vis, tm, iters=2)
    old = _f32_forward_iteration(sd, fw, co, ff, vis, tm, iters=2)
    for a, o in zip(new[0] + [new[1]], old[0] + [old[1]]):
        assert a.dtype == torch.float32 and torch.equal(a, o)
    rgbs = torch.zeros((1, fm.shape[0], 3, 4, 4))                      # only the time axis is read when fmaps_all is given
    new = R.cotracker_forward(sd, rgbs, q, iters=2, fmaps_all=fm)
    old = _f32_cotracker_forward(sd, rgbs, q, iters=2, fmaps_all=fm)
    for a, o in zip(new, old):
        assert a.dtype == torch.float32 and torch.equal(a, o)
    flow = torch.randn((4, 8, 2), generator=torch.Generator().manual_seed(1)) * 100
    assert torch.equal(R.get_2d_embedding(flow), _f32_get_2d_embedding(flow))
    c0 = torch.rand((1, 6, 2), generator=torch.Generator().manual_seed(3)) * 20 - 2
    assert torch.equal(R.sample_pos_embed((12, 16), R.IN_DIM, c0), _f32_sample_pos_embed((12, 16), R.IN_DIM, c0))
    assert torch.equal(R.time_embed(R.IN_DIM, 8), _f32_time_embed(R.IN_DIM, 8))


def test_cotracker_oracle_float64_is_float64(monkeypatch):
    """every intermediate of the float64 path is float64, and the path differs from float32 by a small non-zero amount"""
    seen = []

    def spy(mod, name):
        f = getattr(mod, name)

        def wrapped(*a, **k):
            out = f(*a, **k)
            for t in (out if isinstance(out, (tuple, list)) else [out]):
                for u in (t if isinstance(t, list) else [t]):
                    seen.append((name, u.dtype))
            return out
        monkeypatch.setattr(mod, name, wrapped)

    for mod, name in ((R, "get_2d_embedding"), (R, "sample_pos_embed"), (R, "time_embed"), (R, "_attn_block"), (R, "update_former"),
                      (R, "forward_iteration"), (pips_ref, "corr_lookup"), (pips_ref, "bilinear_sample2d"), (pips_ref, "build_pyramid"),
                      (F, "linear"), (F, "layer_norm"), (F, "group_norm"), (F, "gelu")):
        spy(mod, name)
    sd, fm, q = _inputs()
    sd64 = {k: v.double() for k, v in sd.items()}
    fw, co, ff, vis, tm = _window(fm, q)
    p64, v64 = R.forward_iteration(sd64, fw.double(), co.double(), ff.double(), vis.double(), tm, iters=2)
    rgbs = torch.zeros((1, fm.shape[0], 3, 4, 4), dtype=torch.float64)
    t64, vi64 = R.cotracker_forward(sd64, rgbs, q.double(), iters=2, fmaps_all=fm.double())
    names = {n for n, _ in seen}
    assert {"get_2d_embedding", "sample_pos_embed", "time_embed", "_attn_block", "update_former", "corr_lookup",
            "bilinear_sample2d", "linear", "layer_norm", "group_norm", "gelu"} <= names, names
    bad = [(n, d) for n, d in seen if d != torch.float64]
    assert not bad, bad[:5]
    assert all(t.dtype == torch.float64 for t in p64 + [v64, t64, vi64])
    monkeypatch.undo()
    p32, v32 = R.forward_iteration(sd, fw, co, ff, vis, tm, iters=2)
    t32, vi32 = R.cotracker_forward(sd, rgbs.float(), q, iters=2, fmaps_all=fm)
    for a, b in ((p64[-1], p32[-1]), (v64, v32), (t64, t32), (vi64, vi32)):
        d = (a - b.double()).abs().max().item()
        assert 0 < d <= 1e-3 * max(1.0, a.abs().max().item()), d
