"""ORACLE (test infrastructure, NOT product code): CPU restatement of the reference's interactive point correction.

Only ``tests/`` and ``tools/`` may import this.

Restates /root/reference/sam_pt/modeling/sam_pt_interactive.py:
* ``SamPtInteractive.forward``          :56-675 (query_points branch; visualisation branches omitted: they draw only)
* ``extract_largest_cluster_points``    :678-729
parameterised by its primitives, so the same loop can be driven by CPU oracles or by the product's GPU pieces one call at a
time:
* ``decode(frame_idx, coords (K,2) float32, labels (K,) int) -> (logits (H,W) float32, score 0-d float32)`` for a prompt with at
  least one point and one positive label (predict_mask :133-188 without its zero return, which stays in the loop);
* ``track(images_from_frame, query (1,1,3) int) -> (traj (T',1,1,2), vis (T',1,1))`` (SamPt._track_points);
* ``jf(m (H,W) bool np, gt (H,W) bool np) -> (J, F)`` with davis2017's value types (``davis_jf`` below);
* ``dbscan(points (n,2) float32 np, eps, min_samples) -> labels`` (``sklearn.cluster.DBSCAN`` by default);
* ``kmedoids(points (n,2) float32 np, k) -> cluster_centers_`` (``query_points_ref.kmedoids_alternate`` by default).

DAVIS J&F (davis2017-evaluation ``db_eval_iou`` / ``db_eval_boundary`` / ``f_measure`` / ``_seg2bmap``) is restated from the
published code: that package is not installed here, so its parity is unpinned against the package itself; the dilation is
the real ``cv2.dilate`` with skimage's ``disk(r)`` footprint (``dx^2 + dy^2 <= r^2``), and ``tests/test_oracle_interactive.py``
checks it against an independent ``scipy.ndimage.binary_dilation``.
"""
from __future__ import annotations

import json
import os
import pickle
from collections import Counter, namedtuple
from typing import Callable, List

import numpy as np
import torch
import torch.nn.functional as F

from . import query_points_ref

HistoryEntry = namedtuple('HistoryEntry',
                          'action type '
                          'frame_idx point_idx '
                          'iou_before iou_after '
                          'interaction_idx current_iou_threshold '
                          'overall_iou_before overall_iou_after '
                          'boundary_score_before boundary_score_after '
                          'overall_boundary_score_before overall_boundary_score_after '
                          'jf_score_before jf_score_after')

OFFLINE_THRESHOLDS = [0.10, 0.20, 0.30, 0.40, 0.50, 0.60, 0.65, 0.70, 0.75, 0.80, 0.85, 0.88, 0.90, 0.92, 0.95]


# ----------------------------------------------------------------------------------------------------------- DAVIS J&F
def seg2bmap(seg: np.ndarray) -> np.ndarray:
    """davis2017 _seg2bmap with the mask's own size."""
    seg = seg.astype(bool)
    e = np.zeros_like(seg)
    s = np.zeros_like(seg)
    se = np.zeros_like(seg)
    e[:, :-1] = seg[:, 1:]
    s[:-1, :] = seg[1:, :]
    se[:-1, :-1] = seg[1:, 1:]
    b = seg ^ e | seg ^ s | seg ^ se
    b[-1, :] = seg[-1, :] ^ e[-1, :]
    b[:, -1] = seg[:, -1] ^ s[:, -1]
    b[-1, -1] = 0
    return b


def disk(r: int) -> np.ndarray:
    """skimage.morphology.disk(r) as uint8."""
    L = np.arange(-r, r + 1)
    X, Y = np.meshgrid(L, L)
    return (X ** 2 + Y ** 2 <= r ** 2).astype(np.uint8)


def bound_pix(shape) -> float:
    return np.ceil(0.008 * np.linalg.norm(shape))


def dilate_cv2(b: np.ndarray, r: int) -> np.ndarray:
    import cv2
    return cv2.dilate(b.astype(np.uint8), disk(r))


def db_eval_iou(annotation, segmentation):
    inters = np.sum(segmentation & annotation, axis=(-2, -1))
    union = np.sum(segmentation | annotation, axis=(-2, -1))
    j = inters / union if union != 0 else 0.0
    return 1 if np.isclose(union, 0) else j


def f_measure(foreground_mask, gt_mask, dilate=dilate_cv2):
    r = int(bound_pix(foreground_mask.shape))
    fg_boundary = seg2bmap(foreground_mask)
    gt_boundary = seg2bmap(gt_mask)
    fg_dil = dilate(fg_boundary, r)
    gt_dil = dilate(gt_boundary, r)
    gt_match = gt_boundary * fg_dil
    fg_match = fg_boundary * gt_dil
    n_fg = np.sum(fg_boundary)
    n_gt = np.sum(gt_boundary)
    if n_fg == 0 and n_gt > 0:
        precision, recall = 1, 0
    elif n_fg > 0 and n_gt == 0:
        precision, recall = 0, 1
    elif n_fg == 0 and n_gt == 0:
        precision, recall = 1, 1
    else:
        precision = np.sum(fg_match) / float(n_fg)
        recall = np.sum(gt_match) / float(n_gt)
    if precision + recall == 0:
        return 0
    return 2 * precision * recall / (precision + recall)


def db_eval_boundary(annotation, segmentation, dilate=dilate_cv2):
    return f_measure(segmentation, annotation, dilate=dilate)


def davis_jf(m: np.ndarray, gt_m: np.ndarray):
    """(db_eval_iou(m, gt), db_eval_boundary(m, gt)) as the reference calls them (sam_pt_interactive.py:214-218)."""
    return db_eval_iou(m, gt_m), db_eval_boundary(m, gt_m)


def jf_counts(m: np.ndarray, gt_m: np.ndarray, dilate=dilate_cv2) -> np.ndarray:
    """The 8 counts of sampt_jf_counts: |P&G|, |P|G|, |P|, |G|, |dP|, |dG|, |dP & dil(dG)|, |dG & dil(dP)|."""
    m, gt_m = m.astype(bool), gt_m.astype(bool)
    r = int(bound_pix(m.shape))
    bp, bg = seg2bmap(m), seg2bmap(gt_m)
    return np.array([(m & gt_m).sum(), (m | gt_m).sum(), m.sum(), gt_m.sum(), bp.sum(), bg.sum(),
                     (bp & (dilate(bg, r) > 0)).sum(), (bg & (dilate(bp, r) > 0)).sum()], dtype=np.int64)


# ----------------------------------------------------------------------------------------------------------- decode
def apply_coords_torch(coords, original_size, long_side: int = 1024):
    """segment_anything ResizeLongestSide.apply_coords_torch."""
    from .sam_ref import get_preprocess_shape
    old_h, old_w = original_size
    new_h, new_w = get_preprocess_shape(old_h, old_w, long_side)
    coords = coords.clone().to(torch.float)
    coords[..., 0] = coords[..., 0] * (new_w / old_w)
    coords[..., 1] = coords[..., 1] * (new_h / old_h)
    return coords


def sam_decoder(predictor, images_u8, iterative_refinement_iterations: int):
    """`decode` primitive over a ``sam_ref.RefSamPredictor``: every frame encoded once (sam_pt_interactive.py:113-131; the
    predictor keeps the LAST frame's intermediate embeddings, which HQ-SAM then uses for every frame), then predict_mask
    :133-188 with the frame's features assigned."""
    feats = []
    for f in range(images_u8.shape[0]):
        predictor.set_image(images_u8[f].permute(1, 2, 0).cpu().numpy())
        feats.append(predictor.features)

    @torch.no_grad()
    def decode(frame_idx, coords, labels):
        predictor.features = feats[frame_idx]
        pc = apply_coords_torch(coords, predictor.original_size, predictor.cfg.img_size)
        pos = labels == 1
        ml, iou, low = predictor.predict_torch(pc[pos][None], labels[pos][None], None, None, False, True)
        if bool((labels == 0).any()):
            ml, iou, low = predictor.predict_torch(pc[None], labels[None], None, low, False, True)
        for _ in range(iterative_refinement_iterations):
            m = ml[0, 0] > 0
            if m.sum() < 2:
                break
            yx = m.nonzero()
            box = torch.tensor([yx[:, 1].min(), yx[:, 0].min(), yx[:, 1].max(), yx[:, 0].max()], dtype=torch.float)
            ml, iou, low = predictor.predict_torch(pc[None], labels[None], box[None, None, :], low, False, True)
        return ml[0, 0], iou[0, 0]

    return decode


# ----------------------------------------------------------------------------------------------------------- clicks
def dbscan_sklearn(points, eps, min_samples):
    from sklearn.cluster import DBSCAN
    return DBSCAN(eps=eps, min_samples=min_samples).fit(points).labels_


def extract_largest_cluster_points(mask, n_points_to_select, dbscan_points=18000, db_largest_cluster_min_points=180,
                                   kmedian_points=720, dbscan=dbscan_sklearn, kmedoids=query_points_ref.kmedoids_alternate,
                                   info=None):
    """sam_pt_interactive.py:678-729 on CPU tensors; `info` receives the lengths of the two random draws."""
    mask = mask.cpu()
    mask_pixels = mask.nonzero().float()
    perm1 = torch.randperm(len(mask_pixels))
    mask_pixels = mask_pixels[perm1[:dbscan_points]]
    assert len(mask_pixels) > 0
    dbscan_eps = 2.4 * (mask.shape[0] * mask.shape[1]) / dbscan_points
    labels = np.asarray(dbscan(mask_pixels.numpy(), dbscan_eps, 10))
    cluster_count = Counter(labels.tolist())
    cluster_count.pop(-1, None)
    if len(cluster_count) == 0:
        largest_cluster_points = mask.nonzero().float()
    else:
        largest_cluster_id = cluster_count.most_common(1)[0][0]
        largest_cluster_points = mask_pixels[torch.from_numpy(labels == largest_cluster_id)]
        if len(largest_cluster_points) < db_largest_cluster_min_points:
            largest_cluster_points = mask.nonzero().float()
    perm2 = torch.randperm(len(largest_cluster_points))
    largest_cluster_points = largest_cluster_points[perm2[:kmedian_points]]
    selected = torch.from_numpy(np.asarray(kmedoids(largest_cluster_points.numpy(), n_points_to_select))).type(torch.float32)
    if info is not None:
        info["draws"] = (len(perm1), len(perm2))
        info["labels"] = labels
    return selected.flip(1)


# ----------------------------------------------------------------------------------------------------------- the loop
def interactive_forward(video, *, decode: Callable, track: Callable, jf: Callable = davis_jf,
                        dbscan: Callable = dbscan_sklearn, kmedoids: Callable = query_points_ref.kmedoids_alternate,
                        positive_points_per_mask: int, interactions_max=300, interactions_max_per_frame=3,
                        online_interactive_iou_threshold=0.9, disable_point_tracking=False, online=False,
                        out_root: str = ".", taps: dict | None = None):
    """SamPtInteractive.forward (query_points branch).  Writes the reference's files under `out_root`/interactions/<video_id>/;
    `taps` receives per-interaction decision margins (|iou - threshold|, fn - fp, random-draw lengths)."""
    images = torch.stack(video["image"], dim=0)
    n_frames, _, height, width = images.shape
    query_points = video["query_points"]
    n_masks, n_points_per_mask, _ = query_points.shape
    thresholds = [online_interactive_iou_threshold] if online else list(OFFLINE_THRESHOLDS)
    interactions_left = interactions_max
    if disable_point_tracking:
        thresholds = [1.0]
        interactions_max = interactions_max_per_frame * n_frames
    assert n_masks == 1
    gt_masks = torch.stack(video["gt_masks"]).squeeze(1).bool()
    margins = [] if taps is None else taps.setdefault("margins", [])

    def predict_mask(frame_idx, coords, labels):
        if len(coords) == 0 or labels.sum() == 0:
            return torch.zeros((height, width), dtype=torch.float32), torch.tensor(0, dtype=torch.float32)
        return decode(frame_idx, coords, labels)

    def against_gt(frame_idx, trajectories, visibilities, point_labels):
        vis = visibilities[frame_idx, 0, :]
        coords = trajectories[frame_idx, 0, :, :][vis == 1]
        labels = point_labels[vis == 1]
        logits, score = predict_mask(frame_idx, coords, labels)
        m = logits > 0
        gt_m = gt_masks[frame_idx]
        j, f = jf(m.numpy(), gt_m.numpy())
        return m, gt_m, torch.tensor(j), torch.tensor(f), logits, score

    def full_pass(trajectories, visibilities, point_labels):
        logits = torch.zeros((n_masks, n_frames, height, width), dtype=torch.float32)
        spf = torch.zeros((n_frames, n_masks), dtype=torch.float32)
        ious, bs = [], []
        for f in range(n_frames):
            _, _, j, b, lg, s = against_gt(f, trajectories, visibilities, point_labels)
            logits[:, f] = lg
            spf[f] = s
            ious += [j]
            bs += [b]
        return logits, spf.mean(dim=0), spf, ious, bs

    if disable_point_tracking:
        trajectories = torch.zeros((n_frames, 1, 1, 2), dtype=torch.float32)
        visibilities = torch.zeros((n_frames, 1, 1), dtype=torch.float32)
        point_labels = torch.ones((1,), dtype=torch.int)
        interactions_left = interactions_max
    else:
        trajectories, visibilities = track(images, query_points)
        point_labels = torch.ones((n_points_per_mask,), dtype=torch.int)
        point_labels[positive_points_per_mask:] = 0
        interactions_left -= len(query_points[0])

    cache = []
    current_threshold = thresholds.pop(0)
    history: List[HistoryEntry] = []
    pass_ious, pass_bs = [], []
    frame_idx = 0
    frame_interactions = 0
    _, _, _, prev_iou, prev_b = full_pass(trajectories, visibilities, point_labels)
    prev_iou, prev_b = np.mean(prev_iou), np.mean(prev_b)
    while interactions_left > 0:
        if frame_idx == n_frames:
            cache += [{"current_threshold": current_threshold, "trajectories": trajectories.clone(),
                       "visibilities": visibilities.clone(), "point_labels": point_labels.clone(),
                       "interaction_history": history.copy(), "interactions_left": interactions_left,
                       "average_iou": np.mean(pass_ious), "average_boundary_score": np.mean(pass_bs),
                       "current_pass_ious": pass_ious, "current_pass_boundary_scores": pass_bs}]
            if len(thresholds) == 0:
                break
            current_threshold = thresholds.pop(0)
            frame_idx = 0
            frame_interactions = 0
            pass_ious, pass_bs = [], []
        m, gt_m, iou, b, _, _ = against_gt(frame_idx, trajectories, visibilities, point_labels)
        if iou >= current_threshold:
            frame_idx += 1
            frame_interactions = 0
            pass_ious += [iou]
            pass_bs += [b]
            continue
        tp_mask, tn_mask, fp_mask, fn_mask = m & gt_m, ~m & ~gt_m, m & ~gt_m, ~m & gt_m
        incorrect_neg, incorrect_pos = [], []
        for pi in range(trajectories.shape[2]):
            if visibilities[frame_idx, 0, pi].item() != 1:
                incorrect_neg.append(False)
                incorrect_pos.append(False)
                continue
            positive = point_labels[pi].item() == 1
            x, y = trajectories[frame_idx, 0, pi, :].round().int().tolist()
            correct = (positive and (tp_mask[y, x].item() or fn_mask[y, x].item())) or \
                      (not positive and (tn_mask[y, x].item() or fp_mask[y, x].item()))
            incorrect_neg.append(not positive and not correct)
            incorrect_pos.append(positive and not correct)
        margin = {"iou_margin": abs(float(iou) - current_threshold),
                  "fn_minus_fp": int(fn_mask.sum()) - int(fp_mask.sum()), "draws": None}
        if any(incorrect_neg):
            action_point_idx = incorrect_neg.index(True)
            visibilities[frame_idx:, 0, action_point_idx] = 0
            action_name, action_type = "remove", "negative"
        elif any(incorrect_pos):
            action_point_idx = incorrect_pos.index(True)
            visibilities[frame_idx:, 0, action_point_idx] = 0
            action_name, action_type = "remove", "positive"
        else:
            action_name = "add"
            action_point_idx = trajectories.shape[2]
            if fn_mask.sum() > fp_mask.sum():
                mask, label, action_type = fn_mask, 1, "positive"
            else:
                mask, label, action_type = fp_mask, 0, "negative"
            mask_sum = mask.sum().item()
            assert mask_sum > 0
            info = {}
            x, y = extract_largest_cluster_points(mask, min(3, mask_sum), dbscan=dbscan, kmedoids=kmedoids,
                                                  info=info)[0, :].tolist()
            margin["draws"] = info["draws"]
            if disable_point_tracking:
                ct = torch.zeros((n_frames, 1, 1, 2), dtype=torch.float32)
                cv = torch.zeros((n_frames, 1, 1), dtype=torch.float32)
                ct[frame_idx, 0, 0, :] = torch.tensor([x, y], dtype=torch.float32)
                cv[frame_idx, 0, 0] = 1
            else:
                ct, cv = track(images[frame_idx:], torch.tensor([0, x, y], dtype=torch.int)[None, None, :])
                ct[0, 0, 0, :] = torch.tensor([x, y], dtype=torch.float32)
                cv[0, 0, 0] = 1
                ct = torch.cat([torch.zeros((frame_idx, 1, 1, 2), dtype=torch.float32), ct])
                cv = torch.cat([torch.zeros((frame_idx, 1, 1), dtype=torch.float32), cv])
            trajectories = torch.cat([trajectories, ct], dim=2)
            visibilities = torch.cat([visibilities, cv], dim=2)
            point_labels = torch.cat([point_labels, torch.tensor([label], dtype=torch.int)], dim=0)
        margins.append(margin)
        _, _, iou_after, b_after, _, _ = against_gt(frame_idx, trajectories, visibilities, point_labels)
        if disable_point_tracking:
            next_iou, next_b = prev_iou, prev_b
        else:
            _, _, _, next_iou, next_b = full_pass(trajectories, visibilities, point_labels)
            next_iou, next_b = np.mean(next_iou), np.mean(next_b)
        entry = HistoryEntry(
            action=action_name, type=action_type, frame_idx=frame_idx, point_idx=action_point_idx,
            iou_before=iou.item(), iou_after=iou_after.item(), interaction_idx=interactions_left,
            current_iou_threshold=current_threshold, overall_iou_before=prev_iou.item(), overall_iou_after=next_iou.item(),
            boundary_score_before=b.item(), boundary_score_after=b_after.item(),
            overall_boundary_score_before=prev_b.item(), overall_boundary_score_after=next_b.item(),
            jf_score_before=(prev_iou.item() + prev_b.item()) / 2, jf_score_after=(next_iou.item() + next_b.item()) / 2)
        history += [entry]
        interactions_left -= 1
        frame_interactions += 1
        prev_iou, prev_b = next_iou, next_b
        if iou_after >= current_threshold or frame_interactions >= interactions_max_per_frame:
            frame_idx += 1
            frame_interactions = 0
            pass_ious += [iou_after]
            pass_bs += [b_after]

    logits, scores, spf, final_ious, final_bs = full_pass(trajectories, visibilities, point_labels)
    final_iou = np.mean(final_ious)
    root = os.path.join(out_root, f"interactions/{video['video_id']}/")
    os.makedirs(root, exist_ok=True)
    with open(f"{root}history.json", "w") as f:
        json.dump(history, f, indent=4)
    with open(f"{root}achieved_iou_thresholds_cache.pkl", "wb") as f:
        for x in cache:
            x["interaction_history"] = [he._asdict() for he in x["interaction_history"]]
        pickle.dump(cache, f)
    with open(f"{root}final.pkl", "wb") as f:
        pickle.dump({"trajectories": trajectories, "visibilities": visibilities, "point_labels": point_labels,
                     "logits": logits, "scores": scores, "scores_per_frame": spf}, f)
    thr = [h.current_iou_threshold for h in history]
    achieved = [max([0] + [t for t in thr[:i + 1] if t < thr[i]]) for i in range(len(thr))]
    with open(f"{root}overall_iou_history.json", "w") as f:
        json.dump({"threshold": thr, "achieved_threshold": achieved, "before": [h.overall_iou_before for h in history],
                   "after": [h.overall_iou_after for h in history]}, f, indent=4)
    if len(cache) > 0:
        best = cache[int(np.argmax([x["average_iou"] for x in cache]))]
        if best["average_iou"] > final_iou:
            trajectories, visibilities, point_labels = best["trajectories"], best["visibilities"], best["point_labels"]
            logits, scores, spf, final_ious, final_bs = full_pass(trajectories, visibilities, point_labels)
    target_hw = tuple(int(v) for v in video["target_hw"])
    if tuple(logits.shape[-2:]) != target_hw:
        logits = F.interpolate(logits, size=target_hw, mode="bilinear", align_corners=False)
    if taps is not None:
        taps.update(history=history, trajectories=trajectories, visibilities=visibilities, point_labels=point_labels,
                    final_ious=final_ious, final_boundary_scores=final_bs)
    return {"logits": [m for m in logits], "scores": None, "scores_per_frame": None, "trajectories": None, "visibilities": None}
