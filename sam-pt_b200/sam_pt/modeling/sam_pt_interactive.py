"""`SamPtInteractive` drop-in (reference sam_pt/modeling/sam_pt_interactive.py): interactive point-based video segmentation,
simulated against ground-truth masks.  Same constructor kwargs, `forward(video)` contract, returned dict and files under
`interactions/<video_id>/` (relative to the working directory).

The control loop is the reference's.  What runs where:

* every frame is encoded once, in batches, through `encode_frames`; frames are switched by installing their features on the
  predictor, as the reference does by assigning `sam_predictor.features`.  With HQ-SAM the reference never re-assigns
  `interm_features`, so every frame is decoded with the LAST encoded frame's intermediate embeddings: reproduced;
* `predict_mask` (1-2 + `iterative_refinement_iterations` predict_torch calls) is one `predict_refine` call; a full pass decodes
  its frames concurrently on the decoder's graph slots;
* DAVIS J and F are exact integer counts from one native launch over the frames (csrc/interactive.cu), J and F themselves
  are formed in float64 on the host exactly as davis2017-evaluation's numpy code does;
* a frame's (logits, score) depends only on its features and its visible prompt set, so a frame is decoded again only when
  that set changed since its last decode (decodes are bitwise deterministic across slots and graph replays);
* the corrective click: DBSCAN and point categories are native kernels, k-medoids is `kmedoids_gpu`; the two `torch.randperm`
  draws stay on the CPU default generator in the reference's order, so `torch.manual_seed` reproduces its clicks.

Not built: `visualize_all_interactions_separately` / `visualize_all_interactions_as_mp4` (drawings, mp4 and wandb uploads, no
computation) raise NotImplementedError; `font_path` is accepted and unused; the matplotlib plot of the IoU history is not
drawn (its data is written to overall_iou_history.json).
"""
from __future__ import annotations

import json
import os
import pickle
from collections import namedtuple
from ctypes import c_double, c_int
from typing import List

import numpy as np
import torch
from torch.nn import functional as F

from sam_pt.modeling.sam_pt import SamPt
from sam_pt.utils.query_points import kmedoids_gpu
from sampt_b200 import native

HistoryEntry = namedtuple('HistoryEntry',
                          'action type '
                          'frame_idx point_idx '
                          'iou_before iou_after '
                          'interaction_idx current_iou_threshold '
                          'overall_iou_before overall_iou_after '
                          'boundary_score_before boundary_score_after '
                          'overall_boundary_score_before overall_boundary_score_after '
                          'jf_score_before jf_score_after')

# bits of sampt_point_categories' output
_TP, _TN, _FP, _FN, _CORRECT = 1, 2, 4, 8, 16


# ------------------------------------------------------------------------------------------------------------ native calls
def boundary_radius(h: int, w: int) -> int:
    """davis2017 f_measure: bound_pix = ceil(0.008 * ||(H, W)||), in float64 as numpy computes it."""
    return int(np.ceil(0.008 * np.linalg.norm((h, w))))


def jf_counts(logits: torch.Tensor, gt_u8: torch.Tensor) -> torch.Tensor:
    """logits (T,H,W) float32, gt (T,H,W) uint8 on the GPU -> (T,8) int64 on the GPU: |P&G|, |P|G|, |P|, |G|, |dP|, |dG|,
    |dP & dil(dG)|, |dG & dil(dP)| (P = logits > 0, G = gt != 0)."""
    T, H, W = logits.shape
    assert gt_u8.shape == (T, H, W) and gt_u8.dtype == torch.uint8 and logits.dtype == torch.float32
    dev = logits.device
    scratch = torch.empty((3 * T * H * W + 2,), dtype=torch.uint8, device=dev)
    counts = torch.empty((T, 8), dtype=torch.int64, device=dev)
    logits, gt_u8 = logits.contiguous(), gt_u8.contiguous()
    ctx = native.get_context(dev)
    native.check(native.lib().sampt_jf_counts(ctx.handle, native.ptr(logits), native.ptr(gt_u8), c_int(T),
                                              c_int(H), c_int(W), c_int(boundary_radius(H, W)), native.ptr(scratch),
                                              native.ptr(counts), native.stream_ptr()), "jf_counts")
    return counts


def jf_from_counts(c):
    """(J, F) of one frame from its 8 counts, with the value types of davis2017's db_eval_iou(pred, gt) /
    db_eval_boundary(pred, gt): an int where numpy's code yields a Python int, np.float64 otherwise."""
    inter, union, _, _, n_p, n_g, p_match, g_match = (int(v) for v in c)
    j = 1 if union == 0 else np.int64(inter) / np.int64(union)
    # db_eval_boundary(annotation=pred, segmentation=gt) calls f_measure(foreground=gt, gt=pred)
    n_fg, n_gt = n_g, n_p
    if n_fg == 0 and n_gt > 0:
        precision, recall = 1, 0
    elif n_fg > 0 and n_gt == 0:
        precision, recall = 0, 1
    elif n_fg == 0 and n_gt == 0:
        precision, recall = 1, 1
    else:
        precision = np.uint64(g_match) / float(n_fg)
        recall = np.uint64(p_match) / float(n_gt)
    f = 0 if precision + recall == 0 else 2 * precision * recall / (precision + recall)
    return j, f


def point_categories(logits: torch.Tensor, gt_u8: torch.Tensor, xy: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
    """logits (H,W), gt (H,W) uint8 on the GPU, xy (n,2) float32 (x,y), labels (n,) -> (n,) int32 category bits on the host."""
    H, W = logits.shape
    xy = xy.float().contiguous()
    r = xy.round().int()
    bad = (r[:, 0] < -W) | (r[:, 0] >= W) | (r[:, 1] < -H) | (r[:, 1] >= H)
    if bool(bad.any()):
        i = int(bad.nonzero()[0, 0])
        raise IndexError(f"point {i} at (x, y) = {tuple(r[i].tolist())} is outside the {H}x{W} mask")
    n = xy.shape[0]
    dev = logits.device
    out = torch.empty((n,), dtype=torch.int32, device=dev)
    if n == 0:
        return out.cpu()
    # device copies held in locals: a temporary built inside the argument list is freed before the launch reads it
    logits, gt_u8 = logits.contiguous(), gt_u8.contiguous()
    xy_d, labels_d = xy.to(dev), labels.to(dev, torch.int32).contiguous()
    ctx = native.get_context(dev)
    native.check(native.lib().sampt_point_categories(
        ctx.handle, native.ptr(logits), native.ptr(gt_u8), c_int(H), c_int(W), native.ptr(xy_d), native.ptr(labels_d), c_int(n),
        native.ptr(out), native.stream_ptr()), "point_categories")
    return out.cpu()


def dbscan_labels(points_yx: torch.Tensor, eps: float, min_samples: int) -> torch.Tensor:
    """`DBSCAN(eps, min_samples).fit(points).labels_` for integer-valued float32 points (n,2) on the GPU -> (n,) int32."""
    if not points_yx.is_cuda:
        raise RuntimeError("dbscan_labels runs in libsampt_b200 on a CUDA device; there is no CPU fallback")
    pts = points_yx.float().contiguous()
    n = pts.shape[0]
    labels = torch.empty((n,), dtype=torch.int32, device=pts.device)
    scratch = torch.empty((3 * n,), dtype=torch.int32, device=pts.device)
    ctx = native.get_context(pts.device)
    native.check(native.lib().sampt_dbscan(ctx.handle, native.ptr(pts), c_int(n), c_double(eps), c_int(min_samples),
                                           native.ptr(labels), native.ptr(scratch), native.stream_ptr()), "dbscan")
    return labels


def largest_cluster_label(labels: np.ndarray):
    """`Counter(labels).most_common(1)` without the noise label: the highest count, ties to the label seen first in `labels`
    order.  None when every point is noise."""
    uniq, first, counts = np.unique(labels, return_index=True, return_counts=True)
    keep = uniq != -1
    if not keep.any():
        return None
    uniq, first, counts = uniq[keep], first[keep], counts[keep]
    return int(uniq[np.lexsort((first, -counts))[0]])


def extract_largest_cluster_points(mask, n_points_to_select, dbscan_points=18000, db_largest_cluster_min_points=180,
                                   kmedian_points=720):
    """reference sam_pt_interactive.py:678-729: `n_points_to_select` k-medoids of (a random subset of) the largest DBSCAN
    cluster of a random subset of the mask's pixels -> (n, 2) float32 (x, y) on the mask's device.  `mask` (H, W) on the GPU."""
    mask_pixels = mask.nonzero().float()
    mask_pixels = mask_pixels[torch.randperm(len(mask_pixels))[:dbscan_points].to(mask_pixels.device)]
    assert len(mask_pixels) > 0
    dbscan_eps = 2.4 * (mask.shape[0] * mask.shape[1]) / dbscan_points
    labels = dbscan_labels(mask_pixels, dbscan_eps, 10)
    largest = largest_cluster_label(labels.cpu().numpy())
    if largest is None:
        print(f"WARNING: No clusters found in a mask of mask.sum()={mask.sum()} pixels, using the mask instead")
        largest_cluster_points = mask.nonzero().float()
    else:
        largest_cluster_points = mask_pixels[labels == largest]
        if len(largest_cluster_points) < db_largest_cluster_min_points:
            print(f"WARNING: Largest cluster has only {len(largest_cluster_points)} points, using the mask instead")
            largest_cluster_points = mask.nonzero().float()
    sel = torch.randperm(len(largest_cluster_points))[:kmedian_points].to(largest_cluster_points.device)
    selected_points = kmedoids_gpu(largest_cluster_points[sel], n_points_to_select)
    return selected_points.flip(1)


# ------------------------------------------------------------------------------------------------------------ the model
class SamPtInteractive(SamPt):
    def __init__(self, interactions_max=300, interactions_max_per_frame=3, online_interactive_iou_threshold=0.9,
                 disable_point_tracking=False, online=False, font_path=None, visualize_all_interactions_separately=False,
                 visualize_all_interactions_as_mp4=False, **kwargs):
        super().__init__(**kwargs)
        for name, on in (("visualize_all_interactions_separately", visualize_all_interactions_separately),
                         ("visualize_all_interactions_as_mp4", visualize_all_interactions_as_mp4)):
            if on:
                raise NotImplementedError(f"{name}=True is not built: it only draws the interactions (cv2 / PIL images, an "
                                          "imageio mp4 and a wandb upload); the segmentation results do not depend on it")
        self.disable_point_tracking = disable_point_tracking
        self.interactions_max = interactions_max
        self.interactions_max_per_frame = interactions_max_per_frame
        self.online = online
        self.font_path = font_path
        self.visualize_all_interactions_separately = visualize_all_interactions_separately
        self.visualize_all_interactions_as_mp4 = visualize_all_interactions_as_mp4
        self.online_interactive_iou_threshold = online_interactive_iou_threshold
        self.offline_interactive_iou_thresholds = [
            0.10, 0.20, 0.30, 0.40, 0.50,
            0.60, 0.65, 0.70, 0.75, 0.80,
            0.85, 0.88, 0.90, 0.92, 0.95,
        ]
        # per-frame decode cache (see the module docstring); tests switch it off to show it changes no result
        self._reuse_decodes = True

    # -------------------------------------------------------------------------------------------- frame evaluation
    def _prompt(self, frame_idx, trajectories, visibilities, point_labels):
        vis = visibilities[frame_idx, 0, :]
        return vis, trajectories[frame_idx, 0, :, :][vis == 1], point_labels[vis == 1]

    @torch.no_grad()
    def _decode(self, frame_ids, prompts):
        """Decode `frame_ids` (prompts[f] = (coords, labels) on the host) into self._logits[f] / self._scores[f]."""
        pred = self.sam_predictor
        dev = self.device
        main = torch.cuda.current_stream()
        nslot = max(1, int(self.decode_streams))
        if not getattr(pred.model, "use_cuda_graphs", True) or not pred.model.has_decoder_slab():
            nslot = 1
        if nslot > 1 and (self._dec_streams is None or len(self._dec_streams) != nslot):
            self._dec_streams = [torch.cuda.Stream(device=dev) for _ in range(nslot)]
        n_ref = int(self.iterative_refinement_iterations) if self.iterative_refinement_iterations else 0
        used = set()
        k = 0
        for f in frame_ids:
            coords, labels = prompts[f]
            if len(coords) == 0 or labels.sum() == 0:     # sam_pt_interactive.py:134-135
                self._logits[f].zero_()
                self._scores[f].zero_()
                continue
            slot = k % nslot
            k += 1
            stream = self._dec_streams[slot] if nslot > 1 else main
            if nslot > 1 and slot not in used:
                stream.wait_stream(main)
                used.add(slot)
            with torch.cuda.stream(stream):
                feats = self._feats[f:f + 1]
                pred.set_frames_features(self._hw, (feats, self._interm[-1:]) if self._interm is not None else feats)
                c1024 = pred.transform.apply_coords_torch(coords, pred.original_size).to(dev)
                lab = labels.to(dev, torch.int32)
                has_neg = bool((labels == 0).any())
                pos_idx = (labels == 1).nonzero()[:, 0].tolist() if has_neg else None
                iou, _, _ = pred.predict_refine(c1024, lab, 1 if has_neg else 0, n_ref, self._logits[f], slot=slot,
                                                positive_index=pos_idx)
                self._scores[f:f + 1].copy_(iou)
        for sl in used:
            main.wait_stream(self._dec_streams[sl])

    def _refresh(self, frame_ids, trajectories, visibilities, point_labels):
        """Decode the frames of `frame_ids` whose visible prompt set differs from the one of their last decode."""
        prompts, stale = {}, []
        for f in frame_ids:
            _, coords, labels = self._prompt(f, trajectories, visibilities, point_labels)
            key = (coords.numpy().tobytes(), labels.numpy().tobytes())
            if not self._reuse_decodes or self._keys[f] != key:
                prompts[f] = (coords, labels)
                stale.append(f)
                self._keys[f] = key
        if stale:
            self._decode(stale, prompts)

    def _evaluate(self, frame_ids):
        """-> per frame (iou, boundary) tensors as the reference's predict_mask_against_gt_mask makes them, + the counts."""
        f0, f1 = frame_ids[0], frame_ids[-1] + 1
        assert list(frame_ids) == list(range(f0, f1))
        counts = jf_counts(self._logits[f0:f1], self._gt[f0:f1]).cpu().numpy()
        out = []
        for c in counts:
            j, f = jf_from_counts(c)
            out.append((torch.tensor(j), torch.tensor(f), c))
        return out

    # -------------------------------------------------------------------------------------------- forward
    @torch.no_grad()
    def forward(self, video, debug=True):
        if self.training:
            raise NotImplementedError(f"{self._get_name()} does not support training...")
        frames = video["image"]
        assert frames[0].dtype == torch.uint8, "Input images must be in uint8 format (0-255)"
        images = torch.stack([f.to(self.device, non_blocking=True) for f in frames], dim=0)
        n_frames, channels, height, width = images.shape
        if video.get("query_masks") is not None:
            assert video.get("query_points") is None
            print("SAM-PT: Using query masks")
            query_points = self.extract_query_points(images, video["query_masks"].float(), video["query_point_timestep"])
        elif video.get("query_points") is not None:
            print("SAM-PT: Using query points")
            query_points = video["query_points"]
        else:
            raise ValueError("No query points or masks provided")
        query_points = query_points.cpu()
        n_masks, n_points_per_mask, _ = query_points.shape

        if self.online:
            interactive_iou_thresholds = [self.online_interactive_iou_threshold]
        else:
            interactive_iou_thresholds = list(self.offline_interactive_iou_thresholds)
        interactions_max = self.interactions_max
        interactions_max_per_frame = self.interactions_max_per_frame
        interactions_left = interactions_max
        if self.disable_point_tracking:
            interactive_iou_thresholds = [1.0]
            interactions_max = interactions_max_per_frame * n_frames

        assert n_masks == 1, "Interactive point correction only works with a single mask"
        assert "gt_masks" in video, "Ground truth masks must be provided for interactive point correction"
        gt_masks = torch.stack(video["gt_masks"]).squeeze(1).bool()

        # 1. encoder features of every frame, once
        pred = self.sam_predictor
        want_interm = pred._uses_interm()
        B = max(1, int(self.encoder_batch))
        enc = [pred.encode_frames(images[f0:f0 + B], want_interm=want_interm) for f0 in range(0, n_frames, B)]
        if want_interm:
            self._feats, self._interm = torch.cat([e[0] for e in enc]), torch.cat([e[1] for e in enc])
        else:
            self._feats, self._interm = torch.cat(enc), None
        del enc
        self._hw = (height, width)
        self._gt = gt_masks.to(self.device, torch.uint8)
        self._logits = torch.zeros((n_frames, height, width), dtype=torch.float32, device=self.device)
        self._scores = torch.zeros((n_frames,), dtype=torch.float32, device=self.device)
        self._keys = [None] * n_frames

        def predict_mask_against_gt_mask(frame_idx, trajectories, visibilities, point_labels):
            self._refresh([frame_idx], trajectories, visibilities, point_labels)
            iou_score, boundary_score, counts = self._evaluate([frame_idx])[0]
            return iou_score, boundary_score, counts

        def full_pass(trajectories, visibilities, point_labels, logits_to_host=False):
            self._refresh(range(n_frames), trajectories, visibilities, point_labels)
            ev = self._evaluate(range(n_frames))
            scores_per_frame = self._scores.cpu()[:, None].clone()
            logits = self._logits.cpu()[None] if logits_to_host else None
            return logits, scores_per_frame.mean(dim=0), scores_per_frame, [e[0] for e in ev], [e[1] for e in ev]

        # 2. initial tracking
        if self.disable_point_tracking:
            trajectories = torch.zeros((n_frames, 1, 1, 2), dtype=torch.float32)
            visibilities = torch.zeros((n_frames, 1, 1), dtype=torch.float32)
            point_labels = torch.ones((1,), dtype=torch.int)
            interactions_left = interactions_max
            print(f"Point tracking is disabled. Interactions left: {interactions_left}")
        else:
            print(f"Running initial point tracking using {n_points_per_mask} query points...")
            trajectories, visibilities = self._track_points(images, query_points)
            trajectories, visibilities = trajectories.cpu(), visibilities.cpu()
            point_labels = torch.ones((n_points_per_mask,), dtype=torch.int)
            point_labels[self.positive_points_per_mask:] = 0
            interactions_left -= len(query_points[0])
            print(f"Initial point tracking done. Interactions used: {len(query_points[0])} of {interactions_left}")

        # 3. correct until the budget is spent (sam_pt_interactive.py:252-523)
        achieved_iou_thresholds_cache = []
        current_threshold = interactive_iou_thresholds.pop(0)
        interaction_history: List[HistoryEntry] = []
        current_pass_ious = []
        current_pass_boundary_scores = []
        frame_idx = 0
        frame_interactions = 0
        _, _, _, prev_iou, prev_boundary_score = full_pass(trajectories, visibilities, point_labels)
        prev_iou = np.mean(prev_iou)
        prev_boundary_score = np.mean(prev_boundary_score)
        while interactions_left > 0:
            if frame_idx == n_frames:
                assert len(current_pass_ious) == n_frames, f"Expected {n_frames} IoUs, got {len(current_pass_ious)}"
                achieved_iou_thresholds_cache += [{
                    "current_threshold": current_threshold,
                    "trajectories": trajectories.clone(),
                    "visibilities": visibilities.clone(),
                    "point_labels": point_labels.clone(),
                    "interaction_history": interaction_history.copy(),
                    "interactions_left": interactions_left,
                    "average_iou": np.mean(current_pass_ious),
                    "average_boundary_score": np.mean(current_pass_boundary_scores),
                    "current_pass_ious": current_pass_ious,
                    "current_pass_boundary_scores": current_pass_boundary_scores,
                }]
                if len(interactive_iou_thresholds) == 0:
                    print(f"No more thresholds left. Interactions left: {interactions_left}. Stopping.")
                    break
                current_threshold = interactive_iou_thresholds.pop(0)
                print(f"New threshold: {current_threshold}")
                frame_idx = 0
                frame_interactions = 0
                current_pass_ious = []
                current_pass_boundary_scores = []

            iou_score, boundary_score, counts = predict_mask_against_gt_mask(frame_idx, trajectories, visibilities, point_labels)
            if iou_score >= current_threshold:
                frame_idx += 1
                frame_interactions = 0
                current_pass_ious += [iou_score]
                current_pass_boundary_scores += [boundary_score]
                continue

            # points of the frame: TP / TN / FP / FN at their rounded positions (sam_pt_interactive.py:341-361)
            vis = visibilities[frame_idx, 0, :] == 1
            vis_idx = vis.nonzero()[:, 0]
            cat = point_categories(self._logits[frame_idx], self._gt[frame_idx], trajectories[frame_idx, 0][vis],
                                   point_labels[vis]).tolist()
            incorrect_negative_points = [False] * trajectories.shape[2]
            incorrect_positive_points = [False] * trajectories.shape[2]
            for i, c in zip(vis_idx.tolist(), cat):
                positive = point_labels[i].item() == 1
                if not c & _CORRECT:
                    (incorrect_positive_points if positive else incorrect_negative_points)[i] = True

            if any(incorrect_negative_points):
                action_point_idx = incorrect_negative_points.index(True)
                visibilities[frame_idx:, 0, action_point_idx] = 0
                action_name, action_type = "remove", "negative"
            elif any(incorrect_positive_points):
                action_point_idx = incorrect_positive_points.index(True)
                visibilities[frame_idx:, 0, action_point_idx] = 0
                action_name, action_type = "remove", "positive"
            else:
                action_name = "add"
                action_point_idx = trajectories.shape[2]
                inter, n_p, n_g = int(counts[0]), int(counts[2]), int(counts[3])
                m = self._logits[frame_idx] > 0
                gt_m = self._gt[frame_idx].bool()
                if n_g - inter > n_p - inter:          # fn_mask.sum() > fp_mask.sum()
                    mask, label, action_type = m.logical_not() & gt_m, 1, "positive"
                    mask_sum = n_g - inter
                else:
                    mask, label, action_type = m & gt_m.logical_not(), 0, "negative"
                    mask_sum = n_p - inter
                assert mask_sum > 0
                x, y = extract_largest_cluster_points(mask, n_points_to_select=min(3, mask_sum))[0, :].tolist()
                if self.disable_point_tracking:
                    curr_trajectories = torch.zeros((n_frames, 1, 1, 2), dtype=torch.float32)
                    curr_visibilities = torch.zeros((n_frames, 1, 1), dtype=torch.float32)
                    curr_trajectories[frame_idx, 0, 0, :] = torch.tensor([x, y], dtype=torch.float32)
                    curr_visibilities[frame_idx, 0, 0] = 1
                else:
                    curr_query_points = torch.tensor([0, x, y], dtype=torch.int)[None, None, :]
                    curr_trajectories, curr_visibilities = self._track_points(images[frame_idx:], curr_query_points.float())
                    curr_trajectories, curr_visibilities = curr_trajectories.cpu(), curr_visibilities.cpu()
                    curr_trajectories[0, 0, 0, :] = torch.tensor([x, y], dtype=torch.float32)
                    curr_visibilities[0, 0, 0] = 1
                    curr_trajectories = torch.cat([torch.zeros((frame_idx, 1, 1, 2), dtype=torch.float32), curr_trajectories])
                    curr_visibilities = torch.cat([torch.zeros((frame_idx, 1, 1), dtype=torch.float32), curr_visibilities])
                trajectories = torch.cat([trajectories, curr_trajectories], dim=2)
                visibilities = torch.cat([visibilities, curr_visibilities], dim=2)
                point_labels = torch.cat([point_labels, torch.tensor([label], dtype=torch.int)], dim=0)

            iou_score_after, boundary_score_after, _ = predict_mask_against_gt_mask(frame_idx, trajectories, visibilities,
                                                                                    point_labels)
            if self.disable_point_tracking:
                next_iou = prev_iou
                next_boundary_score = prev_boundary_score
            else:
                _, _, _, next_iou, next_boundary_score = full_pass(trajectories, visibilities, point_labels)
                next_iou = np.mean(next_iou)
                next_boundary_score = np.mean(next_boundary_score)
            interaction_entry = HistoryEntry(
                action=action_name, type=action_type, frame_idx=frame_idx, point_idx=action_point_idx,
                iou_before=iou_score.item(), iou_after=iou_score_after.item(), interaction_idx=interactions_left,
                current_iou_threshold=current_threshold, overall_iou_before=prev_iou.item(), overall_iou_after=next_iou.item(),
                boundary_score_before=boundary_score.item(), boundary_score_after=boundary_score_after.item(),
                overall_boundary_score_before=prev_boundary_score.item(),
                overall_boundary_score_after=next_boundary_score.item(),
                jf_score_before=(prev_iou.item() + prev_boundary_score.item()) / 2,
                jf_score_after=(next_iou.item() + next_boundary_score.item()) / 2,
            )
            interaction_history += [interaction_entry]
            interactions_left -= 1
            frame_interactions += 1
            prev_iou = next_iou
            prev_boundary_score = next_boundary_score
            if iou_score_after >= current_threshold or frame_interactions >= interactions_max_per_frame:
                frame_idx += 1
                frame_interactions = 0
                current_pass_ious += [iou_score_after]
                current_pass_boundary_scores += [boundary_score_after]
            print(f"Interaction: {interaction_entry}")

        # 4. final pass, history files, best threshold (sam_pt_interactive.py:525-617)
        logits, scores, scores_per_frame, final_pass_ious, final_pass_boundary_scores = full_pass(
            trajectories, visibilities, point_labels, logits_to_host=True)
        final_iou = np.mean(final_pass_ious)
        print(f"Final IoU: {final_iou}")
        print(f"Interactions left: {interactions_left}")
        write_interaction_files(f"interactions/{video['video_id']}/", interaction_history, achieved_iou_thresholds_cache, {
            "trajectories": trajectories, "visibilities": visibilities, "point_labels": point_labels, "logits": logits,
            "scores": scores, "scores_per_frame": scores_per_frame})

        if len(achieved_iou_thresholds_cache) > 0:
            best = achieved_iou_thresholds_cache[int(np.argmax([x["average_iou"] for x in achieved_iou_thresholds_cache]))]
            if best["average_iou"] > final_iou:
                print(f"Using IoU threshold from cache: {best['current_threshold']}")
                trajectories, visibilities, point_labels = best["trajectories"], best["visibilities"], best["point_labels"]
                logits, scores, scores_per_frame, final_pass_ious, final_pass_boundary_scores = full_pass(
                    trajectories, visibilities, point_labels, logits_to_host=True)
                assert np.isclose(np.mean(final_pass_ious), best["average_iou"], atol=0.001)
                assert np.isclose(np.mean(final_pass_boundary_scores), best["average_boundary_score"], atol=0.001)
        self._feats = self._interm = self._logits = self._gt = None

        target_hw = tuple(int(v) for v in video["target_hw"])
        resize_factor = torch.tensor(target_hw) / torch.tensor(logits.shape[-2:])
        assert (resize_factor[0] - resize_factor[1]).abs().item() < 0.01, "The resizing should have been isotropic"
        if tuple(logits.shape[-2:]) != target_hw:
            logits = F.interpolate(logits, size=target_hw, mode="bilinear", align_corners=False)
        assert logits.shape == (n_masks, n_frames, target_hw[0], target_hw[1])
        assert scores.shape == (n_masks,)
        assert scores_per_frame.shape == (n_frames, n_masks)
        return {"logits": [m for m in logits], "scores": None, "scores_per_frame": None, "trajectories": None,
                "visibilities": None}


def write_interaction_files(interactions_root, interaction_history, achieved_iou_thresholds_cache, final):
    """history.json, achieved_iou_thresholds_cache.pkl, final.pkl and overall_iou_history.json (sam_pt_interactive.py:537-578).
    Like the reference, converts the cached histories to dicts in place."""
    os.makedirs(interactions_root, exist_ok=True)
    with open(f"{interactions_root}history.json", "w") as f:
        json.dump(interaction_history, f, indent=4)
    with open(f"{interactions_root}achieved_iou_thresholds_cache.pkl", "wb") as f:
        for x in achieved_iou_thresholds_cache:
            x["interaction_history"] = [he._asdict() for he in x["interaction_history"]]
        pickle.dump(achieved_iou_thresholds_cache, f)
    with open(f"{interactions_root}final.pkl", "wb") as f:
        pickle.dump(final, f)
    iou_threshold_list = [h.current_iou_threshold for h in interaction_history]
    achieved_iou_threshold_list = [
        max([0] + [iou for iou in iou_threshold_list[:i + 1] if iou < iou_threshold_list[i]])
        for i in range(len(iou_threshold_list))
    ]
    with open(f"{interactions_root}overall_iou_history.json", "w") as f:
        json.dump({
            "threshold": iou_threshold_list,
            "achieved_threshold": achieved_iou_threshold_list,
            "before": [h.overall_iou_before for h in interaction_history],
            "after": [h.overall_iou_after for h in interaction_history],
        }, f, indent=4)
