"""GPU parity of the CoTracker path (SURVEY §8 row a15; configs C3/C5 use it) against oracle/cotracker_ref.py.
PARITY UNPINNED: the oracle restates the un-vendored upstream model from its published description (no golden vectors in the
reference), so these tests prove kernel == restatement, not restatement == upstream checkpoint behaviour."""
import pytest
import torch

from sampt_b200 import synth

pytestmark = pytest.mark.gpu

INTERP = (96, 128)


def _weights():
    # conditioned random weights: an UNconditioned random CoTracker is chaotic (see synth.condition_cotracker), which would turn
    # any comparison into a coin flip; the conditioned one is contractive like the trained checkpoint
    from sam_pt.point_tracker.cotracker.cotracker import cotracker_shapes
    return synth.condition_cotracker(synth.make_state_dict(cotracker_shapes(), seed=31))


def _clip(T, H, W, seed=5):
    return synth.make_clip(T, H, W, seed=seed)["frames"]  # (T,3,H,W) uint8


def _queries(H, W, T):
    # (t, x, y): different birth frames, one point born late, one near the border
    q = torch.tensor([[0.0, 0.30 * W, 0.40 * H], [0.0, 0.72 * W, 0.25 * H], [3.0, 0.55 * W, 0.66 * H],
                      [min(6, T - 1) * 1.0, 0.18 * W, 0.80 * H], [min(9, T - 1) * 1.0, 0.97 * W, 0.52 * H]])
    return q[None]


def _tracker(sd, **kw):
    from sam_pt.point_tracker import CoTrackerPointTracker
    args = dict(checkpoint_path=None, interp_shape=list(INTERP), visibility_threshold=0.7, support_grid_size=2,
                support_grid_every_n_frames=12, add_debug_visualisations=False)
    args.update(kw)
    trk = CoTrackerPointTracker(**args)
    trk.model.load_state_dict(sd)
    trk.model.fnet_on_tensor_cores = False  # strict fp32 encoder for the tight comparison
    return trk.cuda()


def test_resize_matches_aten_bilinear():
    import torch.nn.functional as F
    frames = _clip(3, 80, 112)
    trk = _tracker(_weights())
    got = trk.resize_clip(frames.cuda()).cpu()
    ref = F.interpolate(frames.float(), INTERP, mode="bilinear")
    assert (got - ref).abs().max().item() < 1e-3


@pytest.mark.parametrize("tc", [False, True])
def test_encoder_on_float_frames(tc):
    from oracle import pips_ref
    import torch.nn.functional as F
    sd = _weights()
    frames = F.interpolate(_clip(2, 80, 112).float(), INTERP, mode="bilinear")
    trk = _tracker(sd)
    trk.model.fnet_on_tensor_cores = tc
    pyr = trk.model.encode_frames(frames.cuda())
    ref = torch.cat([pips_ref.fnet(sd, 2 * (frames[i:i + 1] / 255.0) - 1.0, 4) for i in range(2)]).permute(0, 2, 3, 1)
    err = (pyr[0].cpu() - ref).abs().max().item() / ref.abs().max().item()
    assert err < (2e-4 if tc else 2e-5), err


def test_model_windows_vs_oracle():
    """upstream CoTracker.forward: 14 frames -> 3 overlapping windows, points entering at windows 0, 0/1 and 2."""
    from oracle import cotracker_ref as R
    import torch.nn.functional as F
    sd = _weights()
    T, H, W = 14, 96, 128
    frames = _clip(T, H, W).float()
    q = _queries(H, W, T)
    traj_ref, vis_ref = R.cotracker_forward(sd, frames[None], q, iters=6)
    trk = _tracker(sd)
    pyr = trk.model.encode_frames(frames.cuda())
    traj, vis = trk.model.track(pyr, q[0].cuda(), list(range(T)), iters=6)
    d = (traj.cpu() - traj_ref[0]).abs().max().item()
    dv = (vis.cpu() - vis_ref[0]).abs().max().item()
    print(f"cotracker model: max |traj - oracle| = {d:.2e} px, max |vis - oracle| = {dv:.2e}")
    assert d < 2e-3 and dv < 2e-3
    # frames before the first window that contains a point stay exactly zero in the one-directional pass (the wrapper's
    # `traj == 0` merge relies on it): the point born at t=9 enters with the window starting at frame 4
    assert (traj[:4, 4] == 0).all() and (traj[4:, 4] != 0).all()


@pytest.mark.parametrize("T", [14, 5])
def test_tracker_wrapper_vs_oracle(T):
    """CoTrackerPointTracker.forward: resize to interp_shape, support grid, backward pass, short-clip padding (T=5 < 8)."""
    from oracle import cotracker_ref as R
    sd = _weights()
    H, W = 80, 112
    frames = _clip(T, H, W)
    q = _queries(H, W, T)
    traj_ref, vis_ref = R.cotracker_point_tracker_forward(sd, frames[None], q, interp_shape=INTERP, visibility_threshold=0.7,
                                                          support_grid_size=2, support_grid_every_n_frames=12)
    trk = _tracker(sd)
    traj, vis = trk(frames[None].cuda(), q.cuda())
    assert traj.shape == (1, T, 5, 2) and vis.shape == (1, T, 5) and vis.dtype == torch.bool
    d = (traj.cpu() - traj_ref).abs().max().item()
    agree = (vis.cpu() == vis_ref).float().mean().item()
    print(f"cotracker wrapper T={T}: max |traj - oracle| = {d:.2e} px, visibility agreement {agree:.3f}, visible {vis_ref.float().mean():.2f}")
    assert d < 1e-3          # north-star bar (measured ~3e-5 px)
    assert agree >= 0.97


def test_tensor_core_encoder_end_to_end():
    """default configuration (encoder convolutions on tensor cores with the 3-pass split): trajectories within 1e-3 px of the oracle."""
    from oracle import cotracker_ref as R
    sd = _weights()
    T, H, W = 12, 96, 128
    frames = _clip(T, H, W, seed=9)
    q = _queries(H, W, T)
    traj_ref, _ = R.cotracker_point_tracker_forward(sd, frames[None], q, interp_shape=INTERP)
    trk = _tracker(sd)
    trk.model.fnet_on_tensor_cores = True
    traj, _ = trk(frames[None].cuda(), q.cuda())
    d = (traj.cpu() - traj_ref).abs().max().item()
    print(f"cotracker wrapper (TC encoder): max |traj - oracle| = {d:.2e} px")
    assert d < 1e-3


@pytest.mark.parametrize("hq", [False, True])
def test_sampt_with_cotracker_end_to_end(tmp_path, hq):
    """BASELINE configs[2] / configs[4] in miniature: SamPt.forward with the CoTracker tracker (+ HQ-SAM), 2 masks x 4 points (mask
    batching, other objects' positives as negatives, out-of-frame relabel), against the oracle of the whole path."""
    from oracle import cotracker_ref as R, sam_ref, sampt_ref
    from sampt_b200 import factory
    cfg = sam_ref.VIT_TEST
    sam_sd = synth.condition_sam(synth.make_state_dict(sam_ref.sam_state_dict_shapes(cfg, hq=hq), 47))
    cot_sd = _weights()
    video = synth.make_video_dict(10, 96, 128, 4, seed=13)   # seed chosen so that no sigmoid(vis) lies within 3e-3 of the threshold
    q0 = video["query_points"]
    q1 = q0.clone()
    q1[..., 1] = (q1[..., 1] + 37.0) % 120.0 + 4.0
    q1[..., 2] = (q1[..., 2] + 23.0) % 88.0 + 4.0
    q1[..., 0] = 3.0                                  # second object annotated on frame 3 -> exercises the backward pass
    video["query_points"] = torch.cat([q0, q1], dim=0)

    def oracle_tracker(images, queries):
        return R.cotracker_point_tracker_forward(cot_sd, images, queries, interp_shape=INTERP)

    ref = sampt_ref.sampt_forward(None, sam_ref.RefSamPredictor(sam_sd, cfg, hq=hq), video, positive_points_per_mask=4,
                                  sam_iou_threshold=-1e9, tracker=oracle_tracker)
    model = factory.build_sam_pt("vit_test", sam_sd, None, positive_points_per_mask=4, sam_iou_threshold=-1e9, hq=hq,
                                 cotracker_state_dict=cot_sd, cotracker_interp_shape=INTERP)
    out = model(video)
    terr = (out["trajectories"].cpu() - ref["trajectories"]).abs().max().item()
    assert torch.equal(out["visibilities"].cpu(), ref["visibilities"])
    print_rows = []
    assert terr < 1e-3
    for m in range(2):
        for f in range(10):
            a, b = out["logits"][m][f].cpu(), ref["logits"][m][f]
            diff = (a > 0) != (b > 0)
            iou, flipped, area = _iou(a, b), int(diff.sum()), int((b > 0).sum())
            print_rows.append((iou, flipped, area))
            # north-star bar: IoU >= 0.999.  Logit-margin criterion for the tiny (~180 px) masks of the random-weight HQ branch,
            # where one pixel is 0.0056 IoU: a disagreeing pixel is tolerated only if the ORACLE itself is undecided there
            # (|logit| < 1e-2 of a field whose typical magnitude is O(1)), and at most 2 of them per mask (DESIGN.md §2)
            margin_ok = flipped <= 2 and (flipped == 0 or float(b[diff].abs().max()) < 1e-2)
            assert iou >= 0.999 or margin_ok, (m, f, iou, flipped, area)
    print(f"SamPt + CoTracker (hq={hq}): max |dcoord| = {terr:.2e} px, min mask IoU = {min(r[0] for r in print_rows):.5f}, "
          f"flipped pixels = {sum(r[1] for r in print_rows)}, mask areas {min(r[2] for r in print_rows)}..{max(r[2] for r in print_rows)} px")


def _iou(a, b):
    a, b = a > 0, b > 0
    u = (a | b).sum().item()
    return ((a & b).sum().item() / u) if u else 1.0
