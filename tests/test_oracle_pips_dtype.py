"""The PIPS oracle follows the dtype and device of its inputs: float64 serves as the reference of the tracker's kernel tests
(tests/test_gpu_pips_kernels.py), and the float32 path, the one pinned against the reference's golden vectors, is bit-identical to
the float32-only restatement it replaced (kept below verbatim)."""
import torch
import torch.nn.functional as F

from oracle import pips_ref
from sampt_b200 import synth

LATENT = 128


def _f32_bilinear_sample2d(im, x, y):
    B, C, H, W = im.shape
    x0 = torch.floor(x).int(); x1 = x0 + 1
    y0 = torch.floor(y).int(); y1 = y0 + 1
    x0c, x1c = x0.clamp(0, W - 1), x1.clamp(0, W - 1)
    y0c, y1c = y0.clamp(0, H - 1), y1.clamp(0, H - 1)
    flat = im.permute(0, 2, 3, 1).reshape(B, H * W, C)

    def g(yy, xx):
        idx = (yy * W + xx).long()
        return torch.gather(flat, 1, idx[:, :, None].expand(-1, -1, C))

    w00 = ((x1.float() - x) * (y1.float() - y)).unsqueeze(2)
    w01 = ((x - x0.float()) * (y1.float() - y)).unsqueeze(2)
    w10 = ((x1.float() - x) * (y - y0.float())).unsqueeze(2)
    w11 = ((x - x0.float()) * (y - y0.float())).unsqueeze(2)
    out = w00 * g(y0c, x0c) + w01 * g(y0c, x1c) + w10 * g(y1c, x0c) + w11 * g(y1c, x1c)
    return out.permute(0, 2, 1)


def _f32_corr_lookup(pyr, ffeats, coords, radius=3):
    B, S, N, C = ffeats.shape
    r = radius
    out = []
    for i, fm in enumerate(pyr):
        H, W = fm.shape[-2:]
        corrs = torch.matmul(ffeats, fm.reshape(B, S, C, H * W)).view(B, S, N, H, W)
        corrs = corrs / torch.sqrt(torch.tensor(C).float())
        dx = torch.linspace(-r, r, 2 * r + 1)
        dy = torch.linspace(-r, r, 2 * r + 1)
        delta = torch.stack(torch.meshgrid(dy, dx, indexing="ij"), dim=-1)
        cl = coords.reshape(B * S * N, 1, 1, 2) / 2 ** i + delta.view(1, 2 * r + 1, 2 * r + 1, 2)
        xg = 2 * cl[..., 0:1] / (W - 1) - 1
        yg = 2 * cl[..., 1:2] / (H - 1) - 1
        samp = F.grid_sample(corrs.reshape(B * S * N, 1, H, W), torch.cat([xg, yg], dim=-1), align_corners=True)
        out.append(samp.view(B, S, N, -1))
    return torch.cat(out, dim=-1).contiguous().float()


def _f32_get_3d_embedding(xyz, C=64):
    div = (torch.arange(0, C, 2, dtype=torch.float32) * (1000.0 / C)).reshape(1, 1, C // 2)
    pes = []
    for d in range(3):
        v = xyz[:, :, d:d + 1]
        pe = torch.zeros(xyz.shape[0], xyz.shape[1], C)
        pe[:, :, 0::2] = torch.sin(v * div)
        pe[:, :, 1::2] = torch.cos(v * div)
        pes.append(pe)
    return torch.cat(pes + [xyz], dim=2)


@torch.no_grad()
def _f32_pips_forward(sd, xys, fmaps, feat_init=None, iters=6, stride=4, S=8):
    B, N, _ = xys.shape
    coords = (xys.clone() / float(stride)).reshape(B, 1, N, 2).repeat(1, S, 1, 1)
    pyr = pips_ref.build_pyramid(fmaps)
    if feat_init is None:
        ffeat = _f32_bilinear_sample2d(fmaps[:, 0], coords[:, 0, :, 0], coords[:, 0, :, 1]).permute(0, 2, 1)
    else:
        ffeat = feat_init
    ffeats = ffeat.unsqueeze(1).repeat(1, S, 1, 1)
    coords_bak = coords.clone()
    preds = []
    for itr in range(iters):
        fcorrs = _f32_corr_lookup(pyr, ffeats, coords)
        LRR = fcorrs.shape[3]
        fcorrs_ = fcorrs.permute(0, 2, 1, 3).reshape(B * N, S, LRR)
        flows_ = (coords - coords[:, 0:1]).permute(0, 2, 1, 3).reshape(B * N, S, 2)
        times_ = torch.linspace(0, S, S).reshape(1, S, 1).repeat(B * N, 1, 1)
        flows_ = torch.cat([flows_, times_], dim=2)
        ffeats_ = ffeats.permute(0, 2, 1, 3).reshape(B * N, S, LATENT)
        x = torch.cat([ffeats_, fcorrs_, _f32_get_3d_embedding(flows_, 64)], dim=2)
        delta = pips_ref.mixer(sd, x).reshape(flows_.shape[0], S, LATENT + 2)
        dcoords, dfeats = delta[:, :, :2], delta[:, :, 2:]
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


@torch.no_grad()
def _f32_track_one_direction(sd, T, query_points, fmaps_all, s=8, stride=4, thr0=0.9):
    N = query_points.shape[1]
    traj = torch.zeros((T, N, 2))
    vis = torch.zeros((T, N))
    start = query_points[0, :, 0].long()
    ar = torch.arange(N)
    vis[start, ar] = 1.0
    traj[start, ar, :] = query_points[0, :, 1:]
    feat_init = torch.zeros((1, N, LATENT))
    cur = start.clone()
    for f in range(T - 1):
        if (cur == f).sum() == 0:
            continue
        n_missing = max(0, f + s - T)
        idx = list(range(f, min(f + s, T))) + [T - 1] * n_missing
        fm = fmaps_all[idx][None]
        born = start == f
        if born.any():
            _, _, ff = _f32_pips_forward(sd, traj[None, f, born, :], fm, None, 6, stride, s)
            feat_init[:, born, :] = ff
        act = cur == f
        preds, vis_e, _ = _f32_pips_forward(sd, traj[None, f, act, :], fm, feat_init[:, act, :], 6, stride, s)
        out_vis = torch.sigmoid(vis_e).float()
        out_traj = preds[-1].float()
        osl = slice(1, s - n_missing)
        psl = slice(1 + f, f + s - n_missing)
        vis[psl, act] = out_vis[0, osl, :]
        traj[psl, act, :] = out_traj[0, osl, :, :]
        thr = torch.where(act, torch.ones(N) * thr0, torch.zeros(N))
        earliest = torch.where(act, cur + 1, cur)
        last = torch.where(act, cur + s - n_missing - 1, cur)
        nxt = last
        while (vis[nxt, ar] <= thr).any():
            nxt = torch.where(vis[nxt, ar] <= thr, nxt - 1, nxt)
            thr = torch.where(nxt < earliest, thr - 0.02, thr)
            nxt = torch.where(nxt < earliest, last, nxt)
        cur = torch.where(act, nxt, cur)
    return traj[None], (vis > 0.5)[None]


def _inputs():
    sd = synth.condition_pips(synth.make_state_dict(pips_ref.pips_state_dict_shapes(), 7201))
    clip = synth.make_clip(11, 64, 96, seed=3)
    fm = pips_ref.fnet(sd, 2 * (clip["frames"].float() / 255.0) - 1.0)     # (T, 128, 16, 24)
    q = synth.make_query_points(clip, 4, seed=3)
    q[0, :, 0] = torch.tensor([0.0, 0.0, 5.0, 9.0])
    q[0, 1, 1:] = torch.tensor([-3.0, 66.0])       # off the map: clamped gathers, out-of-map correlation samples
    return sd, fm, q


def test_pips_oracle_float32_bit_identical_and_float64_runs():
    sd, fm, q = _inputs()
    T = fm.shape[0]
    rgbs = torch.zeros((1, T, 3, 4, 4), dtype=torch.uint8)     # only the time axis is read when fmaps_all is given
    new = pips_ref.track_one_direction(sd, rgbs, q, fmaps_all=fm)
    old = _f32_track_one_direction(sd, T, q, fm)
    for a, o in zip(new, old):
        assert a.dtype == o.dtype and torch.equal(a, o)
    xys = q[:, :, 1:]
    win = fm[:8][None]
    new = pips_ref.pips_forward(sd, xys, None, None, 3, fmaps=win)
    old = _f32_pips_forward(sd, xys, win, None, 3)
    for a, o in zip(new[0] + list(new[1:]), old[0] + list(old[1:])):
        assert a.dtype == torch.float32 and torch.equal(a, o)
    pyr = pips_ref.build_pyramid(win)
    ff = torch.randn((1, 8, 4, 128))
    co = torch.rand((1, 8, 4, 2)) * 30 - 5
    assert torch.equal(pips_ref.corr_lookup(pyr, ff, co), _f32_corr_lookup(pyr, ff, co))
    flow = torch.randn((4, 8, 3)) * 300
    assert torch.equal(pips_ref.get_3d_embedding(flow), _f32_get_3d_embedding(flow))

    sd64 = {k: v.double() for k, v in sd.items()}
    new64 = pips_ref.pips_forward(sd64, xys.double(), None, None, 3, fmaps=win.double())
    for a, o in zip(new64[0] + list(new64[1:]), new[0] + list(new[1:])):
        assert a.dtype == torch.float64
        assert (a - o.double()).abs().max() <= 1e-3 * max(1.0, o.abs().max().item())
    tr64, vi64 = pips_ref.track_one_direction(sd64, rgbs, q.double(), fmaps_all=fm.double())
    assert tr64.dtype == torch.float64 and vi64.shape == (1, T, q.shape[1])
    x = torch.rand((1, 3, 36, 52), generator=torch.Generator().manual_seed(4)) * 2 - 1
    f64 = pips_ref.fnet(sd64, x.double())
    assert f64.dtype == torch.float64
    assert (f64 - pips_ref.fnet(sd, x).double()).abs().max() <= 1e-3 * max(1.0, f64.abs().max().item())
