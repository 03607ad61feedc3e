"""ORACLE (test infrastructure, NOT product code): CPU restatement of PIPS + PipsPointTracker.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline /
``--impl reference`` leg may import this module.

Restates, as pure functions over the PIPS state-dict (SURVEY.md Appendix A.4):

* ``Pips.forward``            /root/reference/sam_pt/point_tracker/pips/pips.py:439-620
* ``BasicEncoder.forward``    pips.py:254-287, ``ResidualBlock`` pips.py:180-188
* ``CorrBlock``               pips.py:344-407 (dense formulation, exactly as the reference executes it)
* ``DeltaBlock``/``MLPMixer`` pips.py:96-128,290-317; ``get_3d_embedding`` utils/misc.py:30-55
* ``bilinear_sample2d``       utils/samp.py:6-80
* ``PipsPointTracker``        pips/tracker.py:42-201 (trajectory linking + bidirectional merge)

PINNED: ``tests/golden/make_golden_pips.py`` imports the UNMODIFIED reference from /root/reference in the
build container, runs it on seeded inputs and stores the outputs under ``tests/golden/``;
``tests/test_oracle_pips.py`` checks this restatement against those vectors (CPU, no GPU needed).
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

SD = Dict[str, torch.Tensor]
LATENT = 128


# ----------------------------------------------------------------------------- fnet (pips.py:191-287)
def _inorm(x):
    return F.instance_norm(x, eps=1e-5)


def _res_block(sd: SD, p: str, x, stride: int):
    y = F.relu(_inorm(F.conv2d(x, sd[p + "conv1.weight"], sd[p + "conv1.bias"], stride=stride, padding=1)))
    y = F.relu(_inorm(F.conv2d(y, sd[p + "conv2.weight"], sd[p + "conv2.bias"], padding=1)))
    if stride != 1:
        x = _inorm(F.conv2d(x, sd[p + "downsample.0.weight"], sd[p + "downsample.0.bias"], stride=stride))
    return F.relu(x + y)


def fnet(sd: SD, x, stride: int = 4, prefix: str = "fnet."):
    """x (B,3,H,W) in [-1,1] -> (B,128,H//stride,W//stride).  pips.py:254-287."""
    p = prefix
    _, _, H, W = x.shape
    x = F.relu(_inorm(F.conv2d(x, sd[p + "conv1.weight"], sd[p + "conv1.bias"], stride=2, padding=3)))
    a = _res_block(sd, p + "layer1.1.", _res_block(sd, p + "layer1.0.", x, 1), 1)
    b = _res_block(sd, p + "layer2.1.", _res_block(sd, p + "layer2.0.", a, 2), 1)
    c = _res_block(sd, p + "layer3.1.", _res_block(sd, p + "layer3.0.", b, 2), 1)
    d = _res_block(sd, p + "layer4.1.", _res_block(sd, p + "layer4.0.", c, 2), 1)
    size = (H // stride, W // stride)
    a, b, c, d = [F.interpolate(t, size, mode="bilinear", align_corners=True) for t in (a, b, c, d)]
    x = F.conv2d(torch.cat([a, b, c, d], dim=1), sd[p + "conv2.weight"], sd[p + "conv2.bias"], padding=1)
    x = F.relu(_inorm(x))
    return F.conv2d(x, sd[p + "conv3.weight"], sd[p + "conv3.bias"])


# ----------------------------------------------------------------------------- sampling helpers
def bilinear_sample2d(im, x, y):
    """utils/samp.py:6-66: clamp the four indices, weights from the UNCLAMPED floats.  im (B,C,H,W); x,y (B,N) -> (B,C,N)."""
    B, C, H, W = im.shape
    x0 = torch.floor(x).int(); x1 = x0 + 1
    y0 = torch.floor(y).int(); y1 = y0 + 1
    x0c, x1c = x0.clamp(0, W - 1), x1.clamp(0, W - 1)
    y0c, y1c = y0.clamp(0, H - 1), y1.clamp(0, H - 1)
    flat = im.permute(0, 2, 3, 1).reshape(B, H * W, C)

    def g(yy, xx):
        idx = (yy * W + xx).long()
        return torch.gather(flat, 1, idx[:, :, None].expand(-1, -1, C))

    x0f, x1f, y0f, y1f = (t.to(x.dtype) for t in (x0, x1, y0, y1))
    w00 = ((x1f - x) * (y1f - y)).unsqueeze(2)
    w01 = ((x - x0f) * (y1f - y)).unsqueeze(2)
    w10 = ((x1f - x) * (y - y0f)).unsqueeze(2)
    w11 = ((x - x0f) * (y - y0f)).unsqueeze(2)
    out = w00 * g(y0c, x0c) + w01 * g(y0c, x1c) + w10 * g(y1c, x0c) + w11 * g(y1c, x1c)
    return out.permute(0, 2, 1)


def build_pyramid(fmaps, levels: int = 4):
    """pips.py:355-361: level l+1 = avg_pool2d(level l, 2, 2).  fmaps (B,S,C,H,W)."""
    B, S, C, H, W = fmaps.shape
    pyr = [fmaps]
    for _ in range(levels - 1):
        f = F.avg_pool2d(pyr[-1].reshape(B * S, C, *pyr[-1].shape[-2:]), 2, stride=2)
        pyr.append(f.reshape(B, S, C, *f.shape[-2:]))
    return pyr


def corr_lookup(pyr: List[torch.Tensor], ffeats, coords, radius: int = 3):
    """CorrBlock.corr + CorrBlock.sample (pips.py:364-407), dense formulation.
    ffeats (B,S,N,C), coords (B,S,N,2) in level-0 pixels -> (B,S,N,L*(2r+1)^2).
    NB the window is TRANSPOSED (pips.py:378-384): x takes the `dy` grid."""
    B, S, N, C = ffeats.shape
    r = radius
    dt, dev = ffeats.dtype, ffeats.device
    out = []
    for i, fm in enumerate(pyr):
        H, W = fm.shape[-2:]
        corrs = torch.matmul(ffeats, fm.reshape(B, S, C, H * W)).view(B, S, N, H, W)
        corrs = corrs / torch.sqrt(torch.tensor(float(C), dtype=dt, device=dev))
        dx = torch.linspace(-r, r, 2 * r + 1, dtype=dt, device=dev)
        dy = torch.linspace(-r, r, 2 * r + 1, dtype=dt, device=dev)
        delta = torch.stack(torch.meshgrid(dy, dx, indexing="ij"), dim=-1)
        cl = coords.reshape(B * S * N, 1, 1, 2) / 2 ** i + delta.view(1, 2 * r + 1, 2 * r + 1, 2)
        xg = 2 * cl[..., 0:1] / (W - 1) - 1
        yg = 2 * cl[..., 1:2] / (H - 1) - 1
        samp = F.grid_sample(corrs.reshape(B * S * N, 1, H, W), torch.cat([xg, yg], dim=-1), align_corners=True)
        out.append(samp.view(B, S, N, -1))
    return torch.cat(out, dim=-1).contiguous()


def get_3d_embedding(xyz, C: int = 64):
    """utils/misc.py:30-55 with cat_coords=True. xyz (B,N,3) -> (B,N,3C+3)."""
    div = (torch.arange(0, C, 2, dtype=xyz.dtype, device=xyz.device) * (1000.0 / C)).reshape(1, 1, C // 2)
    pes = []
    for d in range(3):
        v = xyz[:, :, d:d + 1]
        pe = torch.zeros(xyz.shape[0], xyz.shape[1], C, dtype=xyz.dtype, device=xyz.device)
        pe[:, :, 0::2] = torch.sin(v * div)
        pe[:, :, 1::2] = torch.cos(v * div)
        pes.append(pe)
    return torch.cat(pes + [xyz], dim=2)


# ----------------------------------------------------------------------------- delta block (pips.py:96-128,290-317)
def mixer(sd: SD, x, prefix: str = "delta_block.to_delta.", depth: int = 12):
    p = prefix
    x = F.linear(x, sd[p + "0.weight"], sd[p + "0.bias"])
    for l in range(1, depth + 1):
        y = F.layer_norm(x, (512,), sd[f"{p}{l}.0.norm.weight"], sd[f"{p}{l}.0.norm.bias"], 1e-5)
        y = F.conv1d(y, sd[f"{p}{l}.0.fn.0.weight"], sd[f"{p}{l}.0.fn.0.bias"])
        y = F.conv1d(F.gelu(y), sd[f"{p}{l}.0.fn.3.weight"], sd[f"{p}{l}.0.fn.3.bias"])
        x = x + y
        y = F.layer_norm(x, (512,), sd[f"{p}{l}.1.norm.weight"], sd[f"{p}{l}.1.norm.bias"], 1e-5)
        y = F.linear(y, sd[f"{p}{l}.1.fn.0.weight"], sd[f"{p}{l}.1.fn.0.bias"])
        y = F.linear(F.gelu(y), sd[f"{p}{l}.1.fn.3.weight"], sd[f"{p}{l}.1.fn.3.bias"])
        x = x + y
    x = F.layer_norm(x, (512,), sd[f"{p}{depth + 1}.weight"], sd[f"{p}{depth + 1}.bias"], 1e-5)
    x = x.mean(dim=1)
    return F.linear(x, sd[f"{p}{depth + 3}.weight"], sd[f"{p}{depth + 3}.bias"])


def delta_block(sd: SD, fhid, fcorr, flow, S: int = 8):
    x = torch.cat([fhid, fcorr, get_3d_embedding(flow, 64)], dim=2)
    return mixer(sd, x).reshape(flow.shape[0], S, LATENT + 2)


# ----------------------------------------------------------------------------- Pips.forward (pips.py:439-620)
@torch.no_grad()
def pips_forward(sd: SD, xys, rgbs, feat_init=None, iters: int = 6, stride: int = 4, S: int = 8,
                 fmaps: Optional[torch.Tensor] = None, taps: Optional[dict] = None):
    """xys (B,N,2) px; rgbs (B,S,3,H,W) float 0..255 -> (list of `iters` coords (B,S,N,2) px, vis_e (B,S,N), ffeat (B,N,128)).
    `fmaps` may be supplied (B,S,128,H/stride,W/stride) to skip the encoder (results-neutral, SURVEY §0.7-i)."""
    B, N, _ = xys.shape
    if fmaps is None:
        _, S_, C, H, W = rgbs.shape
        x = 2 * (rgbs / 255.0) - 1.0
        fmaps = fnet(sd, x.reshape(B * S_, C, H, W), stride).reshape(B, S_, LATENT, H // stride, W // stride)
    coords = (xys.clone() / float(stride)).reshape(B, 1, N, 2).repeat(1, S, 1, 1)
    pyr = build_pyramid(fmaps)
    if feat_init is None:
        ffeat = bilinear_sample2d(fmaps[:, 0], coords[:, 0, :, 0], coords[:, 0, :, 1]).permute(0, 2, 1)
    else:
        ffeat = feat_init
    ffeats = ffeat.unsqueeze(1).repeat(1, S, 1, 1)
    coords_bak = coords.clone()
    preds = []
    for itr in range(iters):
        fcorrs = corr_lookup(pyr, ffeats, coords)
        LRR = fcorrs.shape[3]
        fcorrs_ = fcorrs.permute(0, 2, 1, 3).reshape(B * N, S, LRR)
        flows_ = (coords - coords[:, 0:1]).permute(0, 2, 1, 3).reshape(B * N, S, 2)
        times_ = torch.linspace(0, S, S, dtype=coords.dtype, device=coords.device).reshape(1, S, 1).repeat(B * N, 1, 1)
        flows_ = torch.cat([flows_, times_], dim=2)
        ffeats_ = ffeats.permute(0, 2, 1, 3).reshape(B * N, S, LATENT)
        delta = delta_block(sd, ffeats_, fcorrs_, flows_, S)
        dcoords, dfeats = delta[:, :, :2], delta[:, :, 2:]
        if taps is not None:
            taps.setdefault("fcorrs", []).append(fcorrs.clone())
            taps.setdefault("delta", []).append(delta.clone())
        ffeats_ = ffeats_.reshape(B * N * S, LATENT)
        dfeats = dfeats.reshape(B * N * S, LATENT)
        upd = F.group_norm(dfeats, 1, sd["norm.weight"], sd["norm.bias"], 1e-5)
        upd = F.gelu(F.linear(upd, sd["ffeat_updater.0.weight"], sd["ffeat_updater.0.bias"]))
        ffeats_ = upd + ffeats_
        ffeats = ffeats_.reshape(B, N, S, LATENT).permute(0, 2, 1, 3)
        coords = coords + dcoords.reshape(B, N, S, 2).permute(0, 2, 1, 3)
        coords[:, 0] = coords_bak[:, 0]
        preds.append(coords * stride)
    vis_e = F.linear(ffeats.reshape(B * S * N, LATENT), sd["vis_predictor.0.weight"], sd["vis_predictor.0.bias"])
    return preds, vis_e.reshape(B, S, N), ffeat


# ----------------------------------------------------------------------------- tracker (pips/tracker.py:42-201)
@torch.no_grad()
def track_one_direction(sd: SD, rgbs, query_points, s: int = 8, stride: int = 4, thr0: float = 0.9,
                        fmaps_all: Optional[torch.Tensor] = None, log: Optional[list] = None):
    """pips/tracker.py:42-153.  rgbs (1,T,3,H,W) any dtype; query_points (1,N,3).
    `fmaps_all` (T,128,H/4,W/4): per-frame encoder features computed once (results-neutral shortcut).
    Runs in the dtype and on the device of `query_points`."""
    B, T = rgbs.shape[:2]
    N = query_points.shape[1]
    if B != 1:
        raise NotImplementedError("Batch size > 1 is not supported for PIPS yet")
    dt, dev = query_points.dtype, query_points.device
    traj = torch.zeros((T, N, 2), dtype=dt, device=dev)
    vis = torch.zeros((T, N), dtype=dt, device=dev)
    start = query_points[0, :, 0].long()
    ar = torch.arange(N, device=dev)
    vis[start, ar] = 1.0
    traj[start, ar, :] = query_points[0, :, 1:]
    feat_init = torch.zeros((1, N, LATENT), dtype=dt, device=dev)
    cur = start.clone()
    for f in range(T - 1):
        if (cur == f).sum() == 0:
            continue
        n_missing = max(0, f + s - T)
        idx = list(range(f, min(f + s, T))) + [T - 1] * n_missing
        if fmaps_all is not None:
            fm = fmaps_all[idx][None]
            rg = None
        else:
            fm = None
            rg = rgbs[:, idx].to(dt)
        born = start == f
        if born.any():
            _, _, ff = pips_forward(sd, traj[None, f, born, :], rg, None, 6, stride, s, fmaps=fm)
            feat_init[:, born, :] = ff
        act = cur == f
        preds, vis_e, _ = pips_forward(sd, traj[None, f, act, :], rg, feat_init[:, act, :], 6, stride, s, fmaps=fm)
        out_vis = torch.sigmoid(vis_e)
        out_traj = preds[-1]
        if log is not None:
            log.append({"frame": f, "active": act.clone(), "traj": out_traj.clone(), "vis": out_vis.clone()})
        osl = slice(1, s - n_missing)
        psl = slice(1 + f, f + s - n_missing)
        vis[psl, act] = out_vis[0, osl, :]
        traj[psl, act, :] = out_traj[0, osl, :, :]
        thr = torch.where(act, torch.ones(N, dtype=dt, device=dev) * thr0, torch.zeros(N, dtype=dt, device=dev))
        earliest = torch.where(act, cur + 1, cur)
        last = torch.where(act, cur + s - n_missing - 1, cur)
        nxt = last
        while (vis[nxt, ar] <= thr).any():
            nxt = torch.where(vis[nxt, ar] <= thr, nxt - 1, nxt)
            thr = torch.where(nxt < earliest, thr - 0.02, thr)
            nxt = torch.where(nxt < earliest, last, nxt)
        cur = torch.where(act, nxt, cur)
    return traj[None], (vis > 0.5)[None]


@torch.no_grad()
def pips_tracker_forward(sd: SD, rgbs, query_points, s: int = 8, stride: int = 4, thr0: float = 0.9,
                         share_fnet: bool = True):
    """PipsPointTracker.forward (pips/tracker.py:155-201): L->R, flipped R->L, per-point stitch."""
    query_points = query_points.float()
    T = rgbs.shape[1]
    fm = fm_flip = None
    if share_fnet:
        x = 2 * (rgbs[0].float() / 255.0) - 1.0
        fm = torch.cat([fnet(sd, x[i:i + 1], stride) for i in range(T)], dim=0)
        fm_flip = fm.flip(0)
    tr_r, vi_r = track_one_direction(sd, rgbs, query_points, s, stride, thr0, fm)
    qf = query_points.clone()
    qf[:, :, 0] = T - qf[:, :, 0] - 1
    tr_l, vi_l = track_one_direction(sd, rgbs.flip(1), qf, s, stride, thr0, fm_flip)
    tr_l, vi_l = tr_l.flip(1), vi_l.flip(1)
    N = query_points.shape[1]
    trs, vis = [], []
    for n in range(N):
        t0 = int(query_points[0, n, 0].item())
        trs.append(torch.cat([tr_l[0, :t0, n, :], tr_r[0, t0:, n, :]]))
        vis.append(torch.cat([vi_l[0, :t0, n], vi_r[0, t0:, n]]))
    return torch.stack(trs, dim=1).unsqueeze(0), torch.stack(vis, dim=1).unsqueeze(0)


# ----------------------------------------------------------------------------- state-dict shapes (Appendix A.4)
def pips_state_dict_shapes(S: int = 8) -> Dict[str, Tuple[int, ...]]:
    s: Dict[str, Tuple[int, ...]] = {}

    def conv(name, co, ci, k, bias=True):
        s[name + ".weight"] = (co, ci, k, k)
        if bias:
            s[name + ".bias"] = (co,)

    conv("fnet.conv1", 64, 3, 7)
    cin = 64
    for li, (dim, stride) in enumerate([(64, 1), (96, 2), (128, 2), (128, 2)], start=1):
        conv(f"fnet.layer{li}.0.conv1", dim, cin, 3)
        conv(f"fnet.layer{li}.0.conv2", dim, dim, 3)
        if stride != 1:
            conv(f"fnet.layer{li}.0.downsample.0", dim, cin, 1)
        conv(f"fnet.layer{li}.1.conv1", dim, dim, 3)
        conv(f"fnet.layer{li}.1.conv2", dim, dim, 3)
        cin = dim
    conv("fnet.conv2", 256, 416, 3)
    conv("fnet.conv3", 128, 256, 1)
    p = "delta_block.to_delta."
    kitchen = 4 * 49 + 128 + 64 * 3 + 3
    s[p + "0.weight"] = (512, kitchen); s[p + "0.bias"] = (512,)
    for l in range(1, 13):
        s[f"{p}{l}.0.norm.weight"] = (512,); s[f"{p}{l}.0.norm.bias"] = (512,)
        s[f"{p}{l}.0.fn.0.weight"] = (4 * S, S, 1); s[f"{p}{l}.0.fn.0.bias"] = (4 * S,)
        s[f"{p}{l}.0.fn.3.weight"] = (S, 4 * S, 1); s[f"{p}{l}.0.fn.3.bias"] = (S,)
        s[f"{p}{l}.1.norm.weight"] = (512,); s[f"{p}{l}.1.norm.bias"] = (512,)
        s[f"{p}{l}.1.fn.0.weight"] = (2048, 512); s[f"{p}{l}.1.fn.0.bias"] = (2048,)
        s[f"{p}{l}.1.fn.3.weight"] = (512, 2048); s[f"{p}{l}.1.fn.3.bias"] = (512,)
    s[p + "13.weight"] = (512,); s[p + "13.bias"] = (512,)
    s[p + "15.weight"] = (S * 130, 512); s[p + "15.bias"] = (S * 130,)
    s["norm.weight"] = (128,); s["norm.bias"] = (128,)
    s["ffeat_updater.0.weight"] = (128, 128); s["ffeat_updater.0.bias"] = (128,)
    s["vis_predictor.0.weight"] = (1, 128); s["vis_predictor.0.bias"] = (1,)
    return s
