"""GPU: interactive point correction (sam_pt/modeling/sam_pt_interactive.py, csrc/interactive.cu).

* the J&F counts are bit-equal to the numpy + cv2 restatement of davis2017-evaluation, J and F equal in float64;
* DBSCAN labels are those of sklearn.cluster.DBSCAN, and the chosen largest cluster is the same;
* extract_largest_cluster_points picks the oracle's point under the same torch seed;
* SamPtInteractive.forward equals the restated reference loop driven by the product's own primitives one call at a time
  (no batching, no decode reuse), with the per-frame decode cache on and off."""
import json
import os
import pickle
from collections import Counter

import numpy as np
import pytest
import torch

from oracle import interactive_ref as R
from sam_pt.modeling import sam_pt_interactive as I

pytestmark = pytest.mark.gpu


def _ellipse(h, w, cy, cx, ry, rx):
    yy, xx = np.mgrid[:h, :w]
    return ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1.0


def _random_masks(T, h, w, seed):
    rng = np.random.default_rng(seed)
    out = np.zeros((T, h, w), dtype=bool)
    for t in range(T):
        for _ in range(rng.integers(1, 4)):
            out[t] |= _ellipse(h, w, rng.uniform(-0.1, 1.1) * h, rng.uniform(-0.1, 1.1) * w, rng.uniform(0.05, 0.5) * h,
                               rng.uniform(0.05, 0.5) * w)
        out[t] ^= rng.random((h, w)) < 0.002        # isolated pixels and holes
    return out


def _check_counts(P, G):
    logits = torch.from_numpy(np.where(P, 1.5, -1.5).astype(np.float32)).cuda()
    counts = I.jf_counts(logits, torch.from_numpy(G.astype(np.uint8)).cuda()).cpu().numpy()
    for t in range(P.shape[0]):
        ref = R.jf_counts(P[t], G[t])
        assert np.array_equal(counts[t], ref), (t, counts[t], ref)
        j, f = I.jf_from_counts(counts[t])
        rj, rf = R.davis_jf(P[t], G[t])
        assert j == rj and isinstance(j, int) == isinstance(rj, int)
        assert f == rf and isinstance(f, int) == isinstance(rf, int)


@pytest.mark.parametrize("h,w,T", [(480, 854, 1), (1080, 1920, 2), (97, 131, 50), (1, 7, 3), (9, 1, 3)])
def test_jf_counts_random_masks(h, w, T):
    _check_counts(_random_masks(T, h, w, 1000 + h), _random_masks(T, h, w, 2000 + w))


def test_jf_counts_degenerate_masks():
    h, w = 97, 131
    z, o = np.zeros((h, w), bool), np.ones((h, w), bool)
    px = z.copy(); px[40, 50] = True
    corner = z.copy(); corner[-1, -1] = True
    border = z.copy(); border[0, :] = True; border[:, -1] = True
    edge_blob = _ellipse(h, w, 0, 0, 30, 40)
    cases = [(z, z), (z, o), (o, z), (o, o), (px, z), (z, px), (px, px), (corner, px), (border, edge_blob), (edge_blob, border),
             (edge_blob, edge_blob)]
    _check_counts(np.stack([a for a, _ in cases]), np.stack([b for _, b in cases]))


def _points(seed, kind):
    rng = np.random.default_rng(seed)
    if kind == "blobs":
        c = [rng.normal((100, 200), 12, (3000, 2)), rng.normal((300, 600), 25, (5000, 2)), rng.uniform(0, (480, 854), (400, 2))]
        p = np.concatenate(c)
    elif kind == "bridge":      # two dense blobs joined by a sparse line of border points
        a = rng.normal((100, 100), 6, (400, 2))
        b = rng.normal((100, 190), 6, (400, 2))
        line = np.stack([np.full(30, 100.0), np.linspace(120, 170, 30)], 1)
        p = np.concatenate([a, line, b])
    elif kind == "tied":
        p = np.concatenate([rng.normal((50, 50), 4, (300, 2)), rng.normal((50, 300), 4, (300, 2))])
    p = np.unique(np.round(p).astype(np.int64), axis=0)
    return p[rng.permutation(len(p))].astype(np.float32)


@pytest.mark.parametrize("kind,eps", [("blobs", 2.4 * 480 * 854 / 18000), ("blobs", 6.0), ("bridge", 7.0), ("tied", 5.0),
                                      ("tied", 2.4 * 1080 * 1920 / 18000)])
def test_dbscan_matches_sklearn(kind, eps):
    pts = _points(7, kind)
    ref = R.dbscan_sklearn(pts, eps, 10)
    got = I.dbscan_labels(torch.from_numpy(pts).cuda(), eps, 10).cpu().numpy()
    assert np.array_equal(got, ref)
    count = Counter(ref.tolist())
    count.pop(-1, None)
    assert I.largest_cluster_label(got) == (count.most_common(1)[0][0] if count else None)


@pytest.mark.parametrize("h,w,n", [(480, 854, 18000), (1080, 1920, 18000), (20, 20, 1), (20, 20, 9)])
def test_dbscan_mask_pixels(h, w, n):
    m = torch.from_numpy(_random_masks(1, h, w, 5)[0] | _ellipse(h, w, h / 2, w / 2, h / 3, w / 3))
    g = torch.Generator().manual_seed(3)
    px = m.nonzero().float()
    px = px[torch.randperm(len(px), generator=g)[:n]]
    eps = 2.4 * h * w / 18000
    ref = R.dbscan_sklearn(px.numpy(), eps, 10)
    got = I.dbscan_labels(px.cuda(), eps, 10).cpu().numpy()
    assert np.array_equal(got, ref)


def test_dbscan_tie_goes_to_the_first_label_in_labels_order():
    """Two clusters of 50 points.  Point 0 is a border point of the cluster numbered 1, so Counter's insertion order puts
    label 1 first: the tie is decided for label 1, not for the smaller label 0."""
    grid = lambda y0, x0: [(y0 + i, x0 + j) for i in range(7) for j in range(7)]
    border = [(100, 211)]                              # 5 px from (100, 206) only: 2 neighbours with itself, not core
    a = grid(50, 50) + [(50, 57)]                      # 50 points, smallest core index 1 -> label 0
    b = grid(100, 200)                                 # 49 core points + the border point -> label 1
    pts = np.array(border + a + b, dtype=np.float32)
    ref = R.dbscan_sklearn(pts, 5.0, 10)
    got = I.dbscan_labels(torch.from_numpy(pts).cuda(), 5.0, 10).cpu().numpy()
    assert np.array_equal(got, ref)
    assert ref[0] == 1 and (ref == 0).sum() == (ref == 1).sum() == 50
    assert I.largest_cluster_label(got) == Counter(ref.tolist()).most_common(1)[0][0] == 1


def test_extract_largest_cluster_points_matches_reference_golden():
    """Every case of tests/golden/interactive_cluster_cases.json (the unmodified reference): same seed, same points."""
    from tests.golden.cluster_cases import CASES, make_mask
    with open(os.path.join(os.path.dirname(__file__), "golden", "interactive_cluster_cases.json")) as f:
        golden = {c["name"]: c for c in json.load(f)["cases"]}
    for case in CASES:
        g = golden[case["name"]]
        torch.manual_seed(case["seed"])
        got = I.extract_largest_cluster_points(torch.from_numpy(make_mask(case)).cuda(), g["n_points_to_select"])
        assert got.cpu().tolist() == g["all"], case["name"]


# ------------------------------------------------------------------------------------------------ the loop
def _model(tmp_path, tracker="pips", hq=False, **kw):
    from oracle import cotracker_ref
    from sam_pt.modeling.sam_pt_interactive import SamPtInteractive
    from sampt_b200 import factory, synth
    from tests.golden import interactive_scenarios as S
    ckpt = synth.write_pips_checkpoint_dir(S.pips_state_dict(), str(tmp_path / "pips"))
    cot = None
    if tracker == "cotracker":
        cot = synth.condition_cotracker(synth.make_state_dict(cotracker_ref.cotracker_state_dict_shapes(), 31))
    base = factory.build_sam_pt("vit_test", S.sam_state_dict(hq=hq), ckpt, positive_points_per_mask=S.P, hq=hq,
                                iterative_refinement_iterations=S.REFINEMENTS, cotracker_state_dict=cot,
                                cotracker_interp_shape=(S.H, S.W))
    args = {k: getattr(base, k) for k in (
        "point_tracker", "sam_predictor", "sam_iou_threshold", "positive_point_selection_method", "negative_point_selection_method",
        "positive_points_per_mask", "negative_points_per_mask", "add_other_objects_positive_points_as_negative_points",
        "max_other_objects_positive_points", "point_tracker_mask_batch_size", "iterative_refinement_iterations",
        "use_patch_matching_filtering", "patch_size", "patch_similarity_threshold", "use_point_reinit",
        "reinit_point_tracker_horizon", "reinit_horizon", "reinit_variant")}
    return SamPtInteractive(**args, **kw).cuda().eval()


def _product_primitives(model, video):
    """The product's pieces called one at a time.  Every frame is encoded once; with HQ-SAM every decode uses the LAST frame's
    intermediate embeddings, as the reference's encoder cache does."""
    pred = model.sam_predictor
    images = torch.stack(video["image"]).cuda()
    H, W = images.shape[-2:]
    B = model.encoder_batch
    want_interm = pred._uses_interm()
    enc = [pred.encode_frames(images[f0:f0 + B], want_interm=want_interm) for f0 in range(0, images.shape[0], B)]
    feats = torch.cat([e[0] for e in enc]) if want_interm else torch.cat(enc)
    interm = torch.cat([e[1] for e in enc])[-1:] if want_interm else None
    n_ref = int(model.iterative_refinement_iterations)

    def decode(f, coords, labels):
        pred.set_frames_features((H, W), (feats[f:f + 1], interm) if want_interm else feats[f:f + 1])
        c = pred.transform.apply_coords_torch(coords, pred.original_size).cuda()
        has_neg = bool((labels == 0).any())
        out = torch.empty((H, W), device="cuda")
        iou, _, _ = pred.predict_refine(c, labels.cuda().int(), 1 if has_neg else 0, n_ref, out, slot=0,
                                        positive_index=(labels == 1).nonzero()[:, 0].tolist() if has_neg else None)
        return out.cpu(), iou[0].cpu()

    def track(imgs, q):
        t, v = model._track_points(imgs.cuda(), q.float())
        return t.cpu(), v.cpu()

    def jf(m, g):
        c = I.jf_counts(torch.from_numpy(m.astype(np.float32))[None].cuda(), torch.from_numpy(g.astype(np.uint8))[None].cuda())
        return I.jf_from_counts(c[0].cpu().numpy())

    dbscan = lambda p, eps, ms: I.dbscan_labels(torch.from_numpy(p).cuda(), eps, ms).cpu().numpy()
    from sam_pt.utils.query_points import kmedoids_gpu
    kmed = lambda p, k: kmedoids_gpu(torch.from_numpy(p).cuda(), k).cpu().numpy()
    return dict(decode=decode, track=track, jf=jf, dbscan=dbscan, kmedoids=kmed)


def _files(root):
    d = os.path.join(root, "interactions", "synthetic")
    with open(os.path.join(d, "history.json")) as f:
        hist = json.load(f)
    with open(os.path.join(d, "overall_iou_history.json")) as f:
        overall = json.load(f)
    with open(os.path.join(d, "final.pkl"), "rb") as f:
        final = pickle.load(f)
    with open(os.path.join(d, "achieved_iou_thresholds_cache.pkl"), "rb") as f:
        cache = pickle.load(f)
    return hist, overall, final, cache


def _same_tensors(a, b):
    return all(torch.equal(a[k].cpu(), b[k].cpu()) for k in a if isinstance(a[k], torch.Tensor))


_ONLINE = dict(online=True, online_interactive_iou_threshold=0.95, interactions_max=14)


@pytest.mark.parametrize("setup,kw", [(dict(), _ONLINE),
                                      (dict(), dict(online=False, interactions_max=16)),
                                      (dict(), dict(disable_point_tracking=True, interactions_max_per_frame=2)),
                                      (dict(tracker="cotracker"), _ONLINE),
                                      (dict(hq=True), _ONLINE),
                                      (dict(hq=True), dict(online=False, interactions_max=12))],
                         ids=["online", "offline", "no_tracking", "cotracker_online", "hq_online", "hq_offline"])
def test_forward_equals_reference_loop_on_product_primitives(tmp_path, monkeypatch, setup, kw):
    from tests.golden import interactive_scenarios as S
    model = _model(tmp_path, **setup, **kw)
    video = S.video()
    runs = {}
    for name, reuse in (("cached", True), ("uncached", False)):
        d = tmp_path / name
        d.mkdir()
        monkeypatch.chdir(d)
        model._reuse_decodes = reuse
        torch.manual_seed(S.TORCH_SEED)
        runs[name] = (model(video), _files(str(d)))
    d = tmp_path / "oracle"
    d.mkdir()
    taps = {}
    torch.manual_seed(S.TORCH_SEED)
    ref = R.interactive_forward(video, positive_points_per_mask=model.positive_points_per_mask, out_root=str(d), taps=taps,
                                **kw, **_product_primitives(model, video))
    ref_files = _files(str(d))
    print(f"{len(taps['history'])} interactions: {[(h.action, h.type, h.frame_idx) for h in taps['history']]}")
    for name, (out, files) in runs.items():
        assert torch.equal(out["logits"][0], ref["logits"][0]), name
        assert files[0] == ref_files[0], name                      # history.json
        assert files[1] == ref_files[1], name                      # overall_iou_history.json
        assert _same_tensors(files[2], ref_files[2]), name         # final.pkl
        assert len(files[3]) == len(ref_files[3])
        for a, b in zip(files[3], ref_files[3]):
            assert _same_tensors(a, b) and a["interaction_history"] == b["interaction_history"]
            assert a["average_iou"] == b["average_iou"] and a["current_threshold"] == b["current_threshold"]
    assert len(taps["history"]) > 0


@pytest.mark.parametrize("name", ["online", "offline", "no_tracking"])
def test_forward_against_reference_golden(tmp_path, monkeypatch, name):
    """The product against the UNMODIFIED reference forward on CPU (tests/golden/interactive_forward.npz).  The decoders differ
    in the last bits (GPU vs CPU float32), so a mask can differ by a pixel, which changes the random draws' lengths and every
    later click: interactions are compared in order up to the first difference; the first must match."""
    from tests.golden import interactive_scenarios as S
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "interactive_forward.npz"))
    g = {k.split("__", 1)[1]: z[k] for k in z.files if k.startswith(name + "__")}
    model = _model(tmp_path, **S.SCENARIOS[name])
    draws = []
    randperm = torch.randperm

    def logged(n, *a, **k):
        draws.append(int(n))
        return randperm(n, *a, **k)

    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(torch, "randperm", logged)
    torch.manual_seed(S.TORCH_SEED)
    model(S.video())
    monkeypatch.setattr(torch, "randperm", randperm)
    hist, _, _, _ = _files(str(tmp_path))
    ref_hist = json.loads(str(g["history"]))
    ref_draws = g["draws"].tolist()
    # the first full pass: mean J of every frame (entry 0's overall_iou_before) within the decoders' difference
    assert abs(hist[0][8] - float(np.mean(g["first_pass_iou"]))) < 1e-3
    matched, di = 0, 0
    for a, b in zip(hist, ref_hist):
        if a[:4] != b[:4] or abs(a[4] - b[4]) > 1e-3:      # action, type, frame_idx, point_idx; iou_before
            break
        n_draws = 2 if a[0] == "add" else 0
        if draws[di:di + n_draws] != ref_draws[di:di + n_draws]:
            break
        di += n_draws
        matched += 1
    print(f"{name}: {matched} of {len(ref_hist)} interactions match the reference")
    assert matched >= 1
