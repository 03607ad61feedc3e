"""CPU: the interactive point-correction oracle (oracle/interactive_ref.py) and the SamPtInteractive config boundary.

* the restated J&F (cv2.dilate with skimage's disk) equals a second, independent dilation (scipy.ndimage) on random masks
  and masks touching the border;
* the oracle's extract_largest_cluster_points reproduces the unmodified reference on the golden cases
  (tests/golden/interactive_cluster_cases.json, made by tests/golden/make_golden_interactive.py);
* the host half of the product's J&F (counts -> float64 J, F) equals the oracle's numpy code;
* the reference YAML with the documented interactive overrides instantiates SamPtInteractive; the visualisation flags raise."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import interactive_ref as R
from tests.golden.cluster_cases import CASES, make_mask

HERE = os.path.dirname(os.path.abspath(__file__))
REF_CFG = os.path.join(HERE, "golden", "reference_configs")


def _dilate_scipy(b, r):
    from scipy import ndimage
    return ndimage.binary_dilation(b.astype(bool), structure=R.disk(r).astype(bool)).astype(np.uint8)


def _masks(h, w, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[:h, :w]
    m = np.zeros((h, w), bool)
    for _ in range(3):
        cy, cx = rng.uniform(-0.1, 1.1) * h, rng.uniform(-0.1, 1.1) * w
        m |= ((yy - cy) / (rng.uniform(0.05, 0.5) * h)) ** 2 + ((xx - cx) / (rng.uniform(0.05, 0.5) * w)) ** 2 <= 1
    return m ^ (rng.random((h, w)) < 0.003)


@pytest.mark.parametrize("h,w,seed", [(97, 131, 0), (120, 160, 1), (480, 854, 2), (1, 9, 3), (13, 1, 4)])
def test_jf_restatement_matches_scipy_dilation(h, w, seed):
    P, G = _masks(h, w, seed), _masks(h, w, seed + 100)
    for a, b in ((P, G), (P, np.zeros_like(G)), (np.ones_like(P), G), (P, P)):
        assert np.array_equal(R.jf_counts(a, b), R.jf_counts(a, b, dilate=_dilate_scipy))
        assert R.db_eval_boundary(a, b) == R.db_eval_boundary(a, b, dilate=_dilate_scipy)


def test_seg2bmap_edges():
    m = np.zeros((5, 6), bool)
    m[-1, 2:4] = True            # last row: S ^ E
    m[1:3, -1] = True            # last column: S ^ S
    b = R.seg2bmap(m)
    assert b[-1].tolist() == [False, True, False, True, False, False]
    assert b[:, -1].tolist() == [True, False, True, False, False]
    assert R.bound_pix((480, 854)) == 8 and R.bound_pix((1080, 1920)) == 18


def test_jf_from_counts_matches_numpy_code():
    from sam_pt.modeling.sam_pt_interactive import jf_from_counts
    z = np.zeros((20, 30), bool)
    px = z.copy(); px[5, 5] = True
    cases = [(z, z), (z, ~z), (~z, z), (px, z), (z, px), (px, px), (_masks(20, 30, 7), _masks(20, 30, 8))]
    for a, b in cases:
        j, f = jf_from_counts(R.jf_counts(a, b))
        rj, rf = R.davis_jf(a, b)
        assert j == rj and isinstance(j, int) == isinstance(rj, int)
        assert f == rf and isinstance(f, int) == isinstance(rf, int)


def test_extract_largest_cluster_points_matches_reference_golden():
    with open(os.path.join(HERE, "golden", "interactive_cluster_cases.json")) as f:
        golden = {c["name"]: c for c in json.load(f)["cases"]}
    assert set(golden) == {c["name"] for c in CASES}
    for case in CASES:
        g = golden[case["name"]]
        torch.manual_seed(case["seed"])
        got = R.extract_largest_cluster_points(torch.from_numpy(make_mask(case)), g["n_points_to_select"])
        assert got.tolist() == g["all"], case["name"]


def _cfg(tmp_path, **extra):
    from oracle import pips_ref
    from sampt_b200 import hydra_lite, synth
    pips_sd = synth.condition_pips(synth.make_state_dict(pips_ref.pips_state_dict_shapes(), 1))
    synth.write_pips_checkpoint_dir(pips_sd, str(tmp_path / "models" / "pips_ckpts" / "reference_model"))
    # docs/04-running-experiments.md, "Running Interactive Point-Based Video Segmentation"
    return hydra_lite.compose_model(REF_CFG, {
        "point_tracker": "pips", "sam@sam_predictor.sam_model": "sam_vit_base",
        "sam_predictor._target_": "segment_anything.predictor.SamPredictor", "sam_predictor.sam_model.checkpoint": None,
        "_target_": "sam_pt.modeling.sam_pt_interactive.SamPtInteractive",
        "interactions_max": 200, "interactions_max_per_frame": 2, "online_interactive_iou_threshold": 0.95,
        "online": True, "disable_point_tracking": False, **extra}, cwd=str(tmp_path))


def test_reference_yaml_instantiates_sam_pt_interactive(tmp_path):
    from sampt_b200 import hydra_lite
    from sam_pt.modeling.sam_pt_interactive import SamPtInteractive
    model = hydra_lite.instantiate(_cfg(tmp_path))
    assert type(model) is SamPtInteractive
    assert (model.interactions_max, model.interactions_max_per_frame, model.online_interactive_iou_threshold) == (200, 2, 0.95)
    assert model.online and not model.disable_point_tracking
    assert model.positive_points_per_mask == 16 and model.iterative_refinement_iterations == 12
    assert model.offline_interactive_iou_thresholds[0] == 0.10 and model.offline_interactive_iou_thresholds[-1] == 0.95


@pytest.mark.parametrize("flag", ["visualize_all_interactions_separately", "visualize_all_interactions_as_mp4"])
def test_visualisation_flags_raise(tmp_path, flag):
    from sampt_b200 import hydra_lite
    with pytest.raises(NotImplementedError):
        hydra_lite.instantiate(_cfg(tmp_path, **{flag: True}))


def _golden_forward(name):
    z = np.load(os.path.join(HERE, "golden", "interactive_forward.npz"))
    return {k.split("__", 1)[1]: z[k] for k in z.files if k.startswith(name + "__")}


@pytest.mark.parametrize("name", ["online", "offline", "no_tracking"])
def test_restated_loop_reproduces_reference_forward(tmp_path, name):
    """The restated loop, driven by the CPU oracles (SAM predictor, PIPS, cv2 J&F, sklearn DBSCAN, k-medoids), equals the
    UNMODIFIED reference forward (tests/golden/interactive_forward.npz) exactly: files, history, points, masks."""
    import pickle
    from oracle import sam_ref, sampt_ref
    from tests.golden import interactive_scenarios as S
    g = _golden_forward(name)
    video = S.video()
    pips_sd = S.pips_state_dict()
    decode = R.sam_decoder(sam_ref.RefSamPredictor(S.sam_state_dict(), sam_ref.VIT_TEST), torch.stack(video["image"]),
                           S.REFINEMENTS)
    track = lambda images, q: sampt_ref.track_points(pips_sd, images, q.float())
    torch.manual_seed(S.TORCH_SEED)
    out = R.interactive_forward(video, decode=decode, track=track, positive_points_per_mask=S.P, out_root=str(tmp_path),
                                **S.SCENARIOS[name])
    d = tmp_path / "interactions" / "synthetic"
    assert (d / "history.json").read_text() == str(g["history"])
    assert (d / "overall_iou_history.json").read_text() == str(g["overall"])
    with open(d / "final.pkl", "rb") as f:
        final = pickle.load(f)
    for k in ("trajectories", "visibilities", "point_labels", "scores_per_frame"):
        assert np.array_equal(final[k].numpy(), g[k]), k
    assert np.array_equal(np.packbits((final["logits"] > 0).numpy()), g["final_masks"])
    assert np.array_equal(np.packbits(torch.stack(out["logits"]).numpy() > 0), g["returned_masks"])
    with open(d / "achieved_iou_thresholds_cache.pkl", "rb") as f:
        cache = pickle.load(f)
    ref_cache = json.loads(str(g["cache"]))
    assert len(cache) == len(ref_cache)
    for a, b in zip(cache, ref_cache):
        assert a["current_threshold"] == b["current_threshold"] and a["interactions_left"] == b["interactions_left"]
        assert float(a["average_iou"]) == b["average_iou"] and float(a["average_boundary_score"]) == b["average_boundary_score"]
        assert [float(v) for v in a["current_pass_ious"]] == b["current_pass_ious"]
        assert json.loads(json.dumps(a["interaction_history"])) == b["interaction_history"]
