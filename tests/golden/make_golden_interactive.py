"""Goldens of the UNMODIFIED reference `sam_pt/modeling/sam_pt_interactive.py` (build container only: needs /root/reference).

* tests/golden/interactive_cluster_cases.json: `extract_largest_cluster_points` on the masks of cluster_cases.py (torch seed,
  n_points_to_select, the selected points (x, y)).
* tests/golden/interactive_forward.npz: `SamPtInteractive.forward` on the inputs of interactive_scenarios.py, for each of its
  configurations (online PIPS, offline thresholds, disable_point_tracking): the written history.json /
  overall_iou_history.json, the cache pickle's entries, final.pkl's trajectories / visibilities / point_labels /
  scores_per_frame and bit-packed `logits > 0`, the returned masks, the per-frame J and F of the first full pass and the
  lengths of every `torch.randperm` draw.

The reference module imports wandb / matplotlib / imageio / tqdm / sklearn_extra, davis2017 and `sam_pt.modeling.sam_pt.SamPt`,
which are absent here; they are replaced by stub modules before the import (same approach as _refimport.py):
`sklearn_extra.cluster.KMedoids` is oracle/query_points_ref.py's restatement, `davis2017.metrics` is oracle/interactive_ref.py's
J&F restatement, and `SamPt` is a thin base class giving the attributes forward() uses: `sam_predictor` =
oracle/sam_ref.RefSamPredictor (assignable `.features`; `transform.apply_coords_torch` added), `_track_points` =
oracle/sampt_ref.track_points with the PIPS restatement (pinned to the reference PIPS), `extract_query_masks` returning a
mask of the asserted shape.  DBSCAN is scikit-learn's own.

    python tests/golden/make_golden_interactive.py
"""
import importlib
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "sam-pt_b200")]
REF = "/root/reference"

from oracle import interactive_ref, query_points_ref, sam_ref, sampt_ref  # noqa: E402
from tests.golden import interactive_scenarios as S  # noqa: E402
from tests.golden.cluster_cases import CASES, make_mask  # noqa: E402


class _KMedoids:
    def __init__(self, n_clusters=8, **kw):
        self.n_clusters = n_clusters

    def fit(self, X):
        self.cluster_centers_ = query_points_ref.kmedoids_alternate(np.asarray(X, dtype=np.float32), self.n_clusters)
        return self


JF_LOG = []


def _jf_log(kind, fn):
    def f(a, b):
        v = fn(a, b)
        JF_LOG.append((kind, v))
        return v
    return f


class _StubSamPt(torch.nn.Module):
    device = torch.device("cpu")

    def __init__(self, sam_predictor, pips_sd, positive_points_per_mask, iterative_refinement_iterations):
        super().__init__()
        self.sam_predictor = sam_predictor
        self.pips_sd = pips_sd
        self.positive_points_per_mask = positive_points_per_mask
        self.iterative_refinement_iterations = iterative_refinement_iterations

    def extract_query_masks(self, images, query_points):
        return torch.zeros((query_points.shape[0],) + tuple(images.shape[-2:]), dtype=torch.bool)

    def _track_points(self, images, query_points):
        return sampt_ref.track_points(self.pips_sd, images, query_points.float())


def predictor():
    pred = sam_ref.RefSamPredictor(S.sam_state_dict(), sam_ref.VIT_TEST)
    pred.transform.apply_coords_torch = lambda coords, original_size: interactive_ref.apply_coords_torch(
        coords, original_size, sam_ref.VIT_TEST.img_size)
    return pred


def run_reference_forward(ref, name, cwd):
    import pickle
    video = S.video()
    model = ref.SamPtInteractive(sam_predictor=predictor(), pips_sd=S.pips_state_dict(), positive_points_per_mask=S.P,
                                 iterative_refinement_iterations=S.REFINEMENTS, **S.SCENARIOS[name]).eval()
    draws = []
    randperm = torch.randperm

    def logged(n, *a, **k):
        draws.append(int(n))
        return randperm(n, *a, **k)

    JF_LOG.clear()
    old = os.getcwd()
    os.chdir(cwd)
    torch.randperm = logged
    try:
        torch.manual_seed(S.TORCH_SEED)
        out = model(video)
    finally:
        torch.randperm = randperm
        os.chdir(old)
    d = os.path.join(cwd, "interactions", video["video_id"])
    with open(os.path.join(d, "final.pkl"), "rb") as f:
        final = pickle.load(f)
    with open(os.path.join(d, "achieved_iou_thresholds_cache.pkl"), "rb") as f:
        cache = pickle.load(f)
    ious = [float(v) for k, v in JF_LOG if k == "iou"][:S.T]
    bnds = [float(v) for k, v in JF_LOG if k == "boundary"][:S.T]
    return {
        "history": open(os.path.join(d, "history.json")).read(),
        "overall": open(os.path.join(d, "overall_iou_history.json")).read(),
        "cache": json.dumps([{"current_threshold": c["current_threshold"], "interactions_left": c["interactions_left"],
                              "average_iou": float(c["average_iou"]), "average_boundary_score": float(c["average_boundary_score"]),
                              "current_pass_ious": [float(v) for v in c["current_pass_ious"]],
                              "interaction_history": c["interaction_history"]} for c in cache]),
        "trajectories": final["trajectories"].numpy(), "visibilities": final["visibilities"].numpy(),
        "point_labels": final["point_labels"].numpy(), "scores_per_frame": final["scores_per_frame"].numpy(),
        "final_masks": np.packbits((final["logits"] > 0).numpy()),
        "returned_masks": np.packbits(torch.stack(out["logits"]).numpy() > 0),
        "first_pass_iou": np.array(ious), "first_pass_boundary": np.array(bnds), "draws": np.array(draws, dtype=np.int64),
    }


def import_reference_interactive():
    stubs = {}
    for name in ("wandb", "imageio", "matplotlib", "matplotlib.pyplot", "tqdm", "sklearn_extra", "sklearn_extra.cluster",
                 "davis2017", "davis2017.metrics"):
        stubs[name] = types.ModuleType(name)
    stubs["davis2017.metrics"].db_eval_iou = _jf_log("iou", interactive_ref.db_eval_iou)
    stubs["davis2017.metrics"].db_eval_boundary = _jf_log("boundary", interactive_ref.db_eval_boundary)
    stubs["matplotlib"].pyplot = stubs["matplotlib.pyplot"]
    stubs["matplotlib.pyplot"].__getattr__ = lambda name: (lambda *a, **k: None)     # the IoU-history plot draws only
    stubs["tqdm"].tqdm = lambda x, *a, **k: x
    stubs["sklearn_extra.cluster"].KMedoids = _KMedoids
    saved = {k: v for k, v in sys.modules.items() if k == "sam_pt" or k.startswith("sam_pt.")}
    for k in saved:
        del sys.modules[k]
    for name, path in (("sam_pt", f"{REF}/sam_pt"), ("sam_pt.modeling", f"{REF}/sam_pt/modeling")):
        m = types.ModuleType(name)
        m.__path__ = [path]
        sys.modules[name] = m
    base = types.ModuleType("sam_pt.modeling.sam_pt")
    base.SamPt = _StubSamPt
    sys.modules["sam_pt.modeling.sam_pt"] = base
    for k, v in stubs.items():
        sys.modules.setdefault(k, v)
    mod = importlib.import_module("sam_pt.modeling.sam_pt_interactive")
    for k in [k for k in sys.modules if k == "sam_pt" or k.startswith("sam_pt.")]:
        del sys.modules[k]
    sys.modules.update(saved)
    return mod


def main():
    ref = import_reference_interactive()
    out = []
    for case in CASES:
        mask = torch.from_numpy(make_mask(case))
        k = min(3, int(mask.sum()))
        torch.manual_seed(case["seed"])
        xy = ref.extract_largest_cluster_points(mask, n_points_to_select=k)
        out.append({"name": case["name"], "n_points_to_select": k, "xy": xy[0].tolist(), "all": xy.tolist()})
        print(case["name"], out[-1]["xy"])
    with open(os.path.join(HERE, "interactive_cluster_cases.json"), "w") as f:
        json.dump({"source": "reference sam_pt/modeling/sam_pt_interactive.py:678-729, unmodified", "cases": out}, f, indent=1)
    import tempfile
    arrays = {}
    for name in S.SCENARIOS:
        with tempfile.TemporaryDirectory() as d:
            res = run_reference_forward(ref, name, d)
        print(name, len(json.loads(res["history"])), "interactions, draws", res["draws"].tolist())
        for k, v in res.items():
            arrays[f"{name}__{k}"] = np.array(v) if isinstance(v, str) else v
    np.savez_compressed(os.path.join(HERE, "interactive_forward.npz"), **arrays)


if __name__ == "__main__":
    main()
