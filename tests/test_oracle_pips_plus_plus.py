"""CPU: the PIPS++ oracle (oracle/pips_plus_plus_ref.py) against vectors from the unmodified reference
(tests/golden/make_golden_pips_plus_plus.py), the structural pins, the reference YAML and the reference's edge behaviour."""
import os

import pytest
import torch

from oracle import pips_plus_plus_ref as ref
from sampt_b200 import synth

REF_CFG = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_configs")
H, W = 128, 160


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(os.path.join(golden_dir, "pips_plus_plus_golden.pt"))


@pytest.fixture(scope="module")
def sd():
    return synth.make_pips_plus_plus_state_dict()


def _window_inputs(cfg):
    clip = synth.make_clip(cfg["S"], H, W, seed=cfg["seed"])
    q = synth.make_query_points(clip, cfg["N"], seed=cfg["seed"])[0, :, 1:]
    return clip["frames"][None].float(), q[None, None].repeat(1, cfg["S"], 1, 1)


def _clip_q(cfg):
    clip = synth.make_clip(cfg["T"], H, W, seed=cfg["seed"])
    return clip["frames"][None], synth.make_query_points(clip, cfg["N"], seed=cfg["seed"], t=cfg.get("t", 0))


def test_structure(golden):
    from sam_pt.point_tracker.pips_plus_plus import PipsPlusPlus
    m = PipsPlusPlus(stride=8)
    sd = m.state_dict()
    assert (len(sd), sum(v.numel() for v in sd.values())) == (82, 17_565_410)
    assert golden["structure"] == {"tensors": 82, "params": 17_565_410}
    assert sum(v.numel() for k, v in sd.items() if k.startswith("delta_block")) == 14_932_866


@pytest.mark.parametrize("key", ["window_S8", "window_S128"])
def test_window_matches_reference(golden, sd, key):
    g = golden[key]
    rgbs, tr = _window_inputs(g["cfg"])
    p1, p2, feats = ref.pips_plus_plus_forward(sd, tr, rgbs, g["cfg"]["iters"])
    assert (torch.stack(p1)[:, 0] - g["preds1"]).abs().max().item() <= 1e-4
    assert (torch.stack(p2)[:, 0] - g["preds2"]).abs().max().item() <= 1e-4
    assert (torch.stack(feats)[:, 0] - g["feats"]).abs().max().item() <= 1e-5
    if "feat_init_preds1" in g:
        q1, _, f2 = ref.pips_plus_plus_forward(sd, tr + 1.5, rgbs, 4, feat_init=feats)
        assert (torch.stack(q1)[:, 0] - g["feat_init_preds1"]).abs().max().item() <= 1e-4
        assert (torch.stack(f2)[:, 0] - g["feat_init_feats"]).abs().max().item() <= 1e-5


def test_float32_drift(sd):
    """float32 vs float64 oracle on the 16-iteration S=8 window: 5.6e-5 px, so the GPU end-to-end bar of 1e-3 px is above 10x it"""
    rgbs, tr = _window_inputs({"S": 8, "N": 5, "seed": 72})
    p32, _, _ = ref.pips_plus_plus_forward(sd, tr, rgbs, 16)
    p64, _, _ = ref.pips_plus_plus_forward({k: v.double() for k, v in sd.items()}, tr.double(), rgbs.double(), 16)
    drift = (torch.stack(p32) - torch.stack(p64)).abs().max().item()
    print(f"PIPS++ window, 16 iterations: float32 vs float64 {drift:.3g} px")
    assert drift * 10 <= 1e-3


@pytest.mark.parametrize("name", ["t0", "t5", "image_size", "long140"])
def test_tracker_matches_reference(golden, sd, name):
    g = golden["tracker"][name]
    frames, q = _clip_q(g["cfg"])
    assert torch.equal(q, g["query_points"])
    traj, vis = ref.pips_plus_plus_tracker_forward(sd, frames, q, iters=g["cfg"]["iters"], image_size=g["cfg"]["image_size"])
    assert traj.shape == g["trajectories"].shape
    assert (traj - g["trajectories"]).abs().max().item() <= 1e-3
    assert torch.equal(vis, g["visibilities"])


def test_last_frame_query(golden, sd):
    """The reference returns T-1 frames for a query on the last frame; the drop-in returns T with frame T-1 = the query."""
    g = golden["tracker"]["last"]
    frames, q = _clip_q(g["cfg"])
    quirk, _ = ref.pips_plus_plus_tracker_forward(sd, frames, q, iters=4, intent=False)
    assert quirk.shape[1] == g["cfg"]["T"] - 1 == g["trajectories"].shape[1]
    assert (quirk - g["trajectories"]).abs().max().item() <= 1e-3
    fixed, _ = ref.pips_plus_plus_tracker_forward(sd, frames, q, iters=4)
    assert fixed.shape[1] == g["cfg"]["T"]
    assert torch.equal(fixed[0, -1], q[0, :, 1:]) and torch.equal(fixed[:, :-1], quirk)


def test_mixed_timesteps(golden, sd):
    """The reference raises IndexError for two or more query timesteps; the drop-in gives every point its group's trajectory."""
    g = golden["tracker"]["mixed"]
    assert g["error"].startswith("IndexError")
    frames, q = _clip_q(g["cfg"])
    q[0, 2:, 0] = 6.0
    assert torch.equal(q, g["query_points"])
    with pytest.raises(IndexError):
        ref.pips_plus_plus_tracker_forward(sd, frames, q, iters=2, intent=False)
    traj, _ = ref.pips_plus_plus_tracker_forward(sd, frames, q, iters=2)
    for sel in (slice(0, 2), slice(2, 4)):
        alone, _ = ref.pips_plus_plus_tracker_forward(sd, frames, q[:, sel], iters=2)
        assert torch.equal(traj[:, :, sel], alone)


def test_small_frames_raise(golden):
    """Below 128 px the coarsest level has one row and the reference returns NaN; the drop-in raises before any launch."""
    from sam_pt.point_tracker.pips_plus_plus import PipsPlusPlus
    assert golden["nan_96x128"]
    with pytest.raises(ValueError):
        PipsPlusPlus.check_frame_size(96, 128)
    with pytest.raises(ValueError):
        PipsPlusPlus.check_frame_size(128, 120)
    PipsPlusPlus.check_frame_size(128, 160)


def test_batch_size_raises():
    from sam_pt.point_tracker.pips_plus_plus import PipsPlusPlusPointTracker
    trk = PipsPlusPlusPointTracker(checkpoint_path=None, image_size=None)
    with pytest.raises(NotImplementedError):
        trk(torch.zeros((2, 4, 3, 128, 128), dtype=torch.uint8), torch.zeros((2, 1, 3)))


def test_reference_yaml_instantiates(tmp_path):
    from sampt_b200 import hydra_lite
    ckpt = synth.write_pips_checkpoint_dir(synth.make_pips_plus_plus_state_dict(),
                                           str(tmp_path / "models" / "pips_plus_plus_ckpts" / "reference_model"))
    cfg = hydra_lite.compose_model(REF_CFG, {"point_tracker": "pips_plus_plus", "sam@sam_predictor.sam_model": "sam_vit_base",
                                             "sam_predictor._target_": "segment_anything.predictor.SamPredictor",
                                             "sam_predictor.sam_model.checkpoint": None}, cwd=str(tmp_path))
    pt = cfg["point_tracker"]
    assert pt["_target_"] == "sam_pt.point_tracker.pips_plus_plus.PipsPlusPlusPointTracker"
    assert pt["checkpoint_path"] == ckpt and pt["image_size"] is None
    trk = hydra_lite.instantiate(pt)
    from sam_pt.point_tracker.pips_plus_plus import PipsPlusPlusPointTracker
    assert type(trk) is PipsPlusPlusPointTracker
    assert (trk.stride, trk.max_sequence_length, trk.iters, trk.image_size) == (8, 128, 16, None)
    want = synth.make_pips_plus_plus_state_dict()
    assert all(torch.equal(v.cpu(), want[k]) for k, v in trk.model.state_dict().items())
