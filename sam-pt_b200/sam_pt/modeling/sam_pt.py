"""`SamPt` drop-in (reference sam_pt/modeling/sam_pt.py:21-866): same 18 constructor kwargs, `.device`, `forward(video)`
contract and output dict.  The per-frame work is re-organised for the GPU:

* the clip is uploaded once (uint8), the tracker consumes it on the device;
* SAM's encoder runs on batches of frames (tensor-core GEMMs need M = B*4096 rows to fill 132 SMs);
* `predict_mask`'s 1-2 + <=12 `predict_torch` calls per (frame, mask) are ONE native call with the `area < 2` break test
  evaluated on the device (the reference synchronises ~6x per refinement iteration, sam_pt.py:811-820);
* one device->host copy per clip (trajectories + visibilities, a few KB) replaces the per-frame copies; the host then
  prepares every frame's prompt exactly as `prepare_points` does (sam_pt.py:726-758).
"""
import os
from typing import Optional

import numpy as np
import torch
from torch import nn
from torch.nn import functional as F

from sam_pt.point_tracker import PointTracker
from sam_pt.utils.util import PointVisibilityType


class SamPt(nn.Module):
    def __init__(self, point_tracker: PointTracker, sam_predictor, sam_iou_threshold: float,
                 positive_point_selection_method: str, negative_point_selection_method: str, positive_points_per_mask: int,
                 negative_points_per_mask: int, add_other_objects_positive_points_as_negative_points: bool,
                 max_other_objects_positive_points: Optional[int], point_tracker_mask_batch_size: int,
                 iterative_refinement_iterations: bool, use_patch_matching_filtering: bool, patch_size: int,
                 patch_similarity_threshold: float, use_point_reinit: bool, reinit_point_tracker_horizon: int,
                 reinit_horizon: int, reinit_variant: str):
        super().__init__()
        self.point_tracker = point_tracker
        self.sam_predictor = sam_predictor
        self.sam_iou_threshold = sam_iou_threshold
        self._sam = sam_predictor.model  # makes .to(device) reach SAM (reference sam_pt.py:95-96)
        self.iterative_refinement_iterations = iterative_refinement_iterations
        self.positive_point_selection_method = positive_point_selection_method
        self.negative_point_selection_method = negative_point_selection_method
        self.positive_points_per_mask = positive_points_per_mask
        self.negative_points_per_mask = negative_points_per_mask
        self.add_other_objects_positive_points_as_negative_points = add_other_objects_positive_points_as_negative_points
        self.max_other_objects_positive_points = max_other_objects_positive_points
        self.point_tracker_mask_batch_size = point_tracker_mask_batch_size
        self.use_patch_matching_filtering = use_patch_matching_filtering
        self.patch_size = patch_size
        self.patch_similarity_threshold = patch_similarity_threshold
        self.use_point_reinit = use_point_reinit
        self.reinit_point_tracker_horizon = reinit_point_tracker_horizon
        self.reinit_horizon = reinit_horizon
        self.reinit_variant = reinit_variant
        self.encoder_batch = 8          # frames per ViT launch
        # run the ViT encoder (tensor pipe) on its own stream, concurrently with the PIPS tracker and the mask decoder
        # (fp32 CUDA-core pipes, latency bound): the two halves of the path do not depend on each other until decode
        self.overlap_streams = os.environ.get("SAMPT_OVERLAP", "1") != "0"
        self._enc_stream = None
        # the per-frame decode chains (13 predict_torch calls = ~500 tiny kernels each) are latency bound and independent:
        # replay them round-robin on several streams, each with its own CUDA-graph instance / buffers
        self.decode_streams = int(os.environ.get("SAMPT_DECODE_STREAMS", "8"))
        self._dec_streams = None
        # reference contract (sam_pt.py:863-864, tracker.py:72-76): logits / trajectories / visibilities are returned on the HOST
        # (vos_eval/eval.py:323-325 mixes them with CPU ground-truth masks).  Set False to keep the 82 MB of logits in HBM.
        self.outputs_on_cpu = True
        self.frame_annotations = []

    @property
    def device(self):
        return self._sam.device

    # ------------------------------------------------------------------------------------------------ forward
    def forward(self, video):
        """reference sam_pt.py:122-236."""
        if self.training:
            raise NotImplementedError(f"{self._get_name()} does not support training...")
        frames = video["image"]
        assert frames[0].dtype == torch.uint8, "Input images must be in uint8 format (0-255)"
        # upload frame by frame (async from pinned memory) and stack ON the device: no 60 MB host-side torch.stack copy
        images_dev = torch.stack([f.to(self.device, non_blocking=True) for f in frames], dim=0)
        n_frames, channels, height, width = images_dev.shape
        if video.get("query_masks") is not None:  # e.g. the VOS harness (sam_pt/vos_eval/eval.py:298): sample points from masks
            assert video.get("query_points") is None
            print("SAM-PT: Using query masks")
            query_masks = video["query_masks"].float()
            query_points = self.extract_query_points(images_dev, query_masks, video["query_point_timestep"])
        elif video.get("query_points") is not None:
            print("SAM-PT: Using query points")
            query_points = video["query_points"]
            # the reference also runs SAM on the query frames here (extract_query_masks, sam_pt.py:168-171) but only asserts on
            # the result's shape (and feeds SuperGlue, which is not on this path): results-neutral, skipped (DESIGN.md §4)
        else:
            raise ValueError("No query points or masks provided")
        n_masks, n_points_per_mask, _ = query_points.shape
        self.frame_annotations = [[] for _ in range(n_frames)]

        if not self.use_point_reinit:
            trajectories, visibilities, logits, scores, scores_per_frame = self._forward(images_dev, query_points)
        else:
            trajectories, visibilities, logits, scores, scores_per_frame = self._forward_w_reinit(images_dev, query_points)

        target_hw = tuple(int(v) for v in video["target_hw"])
        resize_factor = torch.tensor(target_hw) / torch.tensor(logits.shape[-2:])
        assert (resize_factor[0] - resize_factor[1]).abs().item() < 0.01, "The resizing should have been isotropic"
        if tuple(logits.shape[-2:]) != target_hw:
            logits = F.interpolate(logits, size=target_hw, mode="bilinear", align_corners=False)
        trajectories = trajectories * resize_factor.to(trajectories.device)

        assert logits.shape == (n_masks, n_frames, target_hw[0], target_hw[1])
        assert scores.shape == (n_masks,)
        assert scores_per_frame.shape == (n_frames, n_masks)
        assert trajectories.shape == (n_frames, n_masks, n_points_per_mask, 2)
        assert visibilities.shape == (n_frames, n_masks, n_points_per_mask)
        if self.outputs_on_cpu:
            logits, trajectories, visibilities = logits.cpu(), trajectories.cpu(), visibilities.cpu()
        return {"logits": [m for m in logits], "scores": scores.tolist(), "scores_per_frame": scores_per_frame.tolist(),
                "trajectories": trajectories, "visibilities": visibilities}

    # ------------------------------------------------------------------------------------------------ queries from masks
    def extract_query_points(self, images, query_masks, query_points_timestep):
        """reference sam_pt.py:238-285: positive (and negative) query points sampled from the query masks.
        images (T,3,H,W) uint8, query_masks (M,H,W) {0,1} float, query_points_timestep (M,) -> (M, P, 3) = (t, x, y) on the
        device.  The masks are moved to the device: the k-medoids run there (sam_pt/utils/query_points.py)."""
        dev = self.device
        query_masks = query_masks.to(dev)
        query_points_timestep = query_points_timestep.to(dev).float()
        query_points_xy = SamPt._extract_query_points_xy(images, query_masks, query_points_timestep,
                                                         self.positive_point_selection_method, self.positive_points_per_mask)
        if self.negative_points_per_mask > 0:
            negative_query_masks = [1 - qm for qm in query_masks]
            negative_xy = SamPt._extract_query_points_xy(images, negative_query_masks, query_points_timestep,
                                                         self.negative_point_selection_method, self.negative_points_per_mask)
            query_points_xy = [torch.cat(x, dim=0) for x in zip(query_points_xy, negative_xy)]
        query_points_xy = torch.stack(query_points_xy, dim=0)
        t = query_points_timestep[:, None, None].repeat(1, query_points_xy.shape[1], 1)
        return torch.concat([t, query_points_xy], dim=2)

    @staticmethod
    def _extract_query_points_xy(images, query_masks, query_points_timestep, point_selection_method, points_per_mask):
        """reference sam_pt.py:287-306"""
        from sam_pt.utils.query_points import (extract_corner_points, extract_kmedoid_points, extract_mixed_points,
                                               extract_random_mask_points)
        if point_selection_method == "kmedoids":
            return [extract_kmedoid_points(qm, points_per_mask) for qm in query_masks]
        if point_selection_method == "shi-tomasi":
            return [extract_corner_points(images[int(t.item()), :, :, :], qm, points_per_mask)
                    for qm, t in zip(query_masks, query_points_timestep)]
        if point_selection_method == "random":
            return [extract_random_mask_points(qm, points_per_mask) for qm in query_masks]
        if point_selection_method == "mixed":
            return extract_mixed_points(query_masks, query_points_timestep, images, points_per_mask)
        raise NotImplementedError(f"Point selection method {point_selection_method} not implemented")

    def extract_query_masks(self, images, query_points):
        """reference sam_pt.py:308-335: SAM applied to the query points on their query frames -> (M, H, W) bool.
        (As in the reference, every mask's points prompt frame-slot 0 of a one-frame 'clip' per mask.)"""
        frames = torch.stack([images[int(t.item())] for t in query_points[:, 0, 0]], dim=0).to(self.device)
        qp = query_points.to(self.device)
        # trajectories (n_frames = M, n_masks = 1, P, 2): frame slot i holds mask i's query frame and query points
        _, logits, _ = self._apply_sam_to_trajectories(frames, qp[:, None, :, 1:].contiguous(), torch.ones_like(qp[:, None, :, 0]))
        return (logits > self.sam_predictor.model.mask_threshold)[0]

    def _forward(self, images, query_points):
        pre = self._start_encoder(images) if self.overlap_streams else None
        trajectories, visibilities = self._track_points(images, query_points)
        _, logits, scores_per_frame = self._apply_sam_to_trajectories(images, trajectories, visibilities, pre=pre)
        scores = scores_per_frame.mean(dim=0)
        return trajectories, visibilities, logits, scores, scores_per_frame

    @torch.no_grad()
    def _start_encoder(self, images):
        """Enqueue the SAM image encoder for every chunk of `images` on the encoder stream; returns per-chunk
        (features, event) so the decode loop on the main stream can wait for exactly the chunk it needs."""
        pred = self.sam_predictor
        main = torch.cuda.current_stream()
        if self._enc_stream is None:
            pred.model.native_context()  # weight registration happens on the main stream, once
            self._enc_stream = torch.cuda.Stream(device=self.device)
        es = self._enc_stream
        es.wait_stream(main)  # the uploaded frames
        B = max(1, int(self.encoder_batch))
        want_interm = pred._uses_interm()
        out = []
        with torch.cuda.stream(es):
            for f0 in range(0, images.shape[0], B):
                enc = pred.encode_frames(images[f0:f0 + B], want_interm=want_interm)
                ev = torch.cuda.Event()
                ev.record(es)
                for t in (enc if isinstance(enc, tuple) else (enc,)):
                    t.record_stream(main)
                out.append((enc, ev))
        return out

    # ------------------------------------------------------------------------------------------------ tracking
    def _track_points(self, rgbs, query_points):
        """reference sam_pt.py:545-596,684-692: batches of `point_tracker_mask_batch_size` masks, flatten (M,P,3)->(1,N,3),
        bool->float visibilities, out-of-frame relabel.  Stays on the device."""
        num_masks, points_per_mask, _ = query_points.shape
        self.point_tracker.eval()
        trajs, viss = [], []
        h, w = rgbs.shape[-2:]
        for i in range(0, num_masks, self.point_tracker_mask_batch_size):
            q = query_points[i:i + self.point_tracker_mask_batch_size].to(self.device)
            m = q.shape[0]
            with torch.no_grad():
                traj, vis = self.point_tracker.to(self.device)(rgbs.unsqueeze(0), q.reshape(1, m * points_per_mask, 3))
            traj, vis = traj[0], vis[0].float()
            if self.use_patch_matching_filtering:
                vis = self._patch_filter(rgbs, q.reshape(m * points_per_mask, 3), traj, vis)
            traj = traj.reshape(-1, m, points_per_mask, 2)
            vis = vis.reshape(-1, m, points_per_mask)
            out = float(PointVisibilityType.OUTSIDE_FRAME.value)
            oob = (traj[..., 0] / w < 0.01) | (traj[..., 1] / h < 0.01) | (traj[..., 0] / w > 0.99) | (traj[..., 1] / h > 0.99)
            vis = torch.where(oob, torch.full_like(vis, out), vis)
            trajs.append(traj)
            viss.append(vis)
        return torch.cat(trajs, dim=1), torch.cat(viss, dim=1)

    def _patch_filter(self, rgbs, query_points, traj, vis):
        """reference sam_pt.py:643-682: Lab patch similarity between every tracked position and its query patch; visible points
        whose similarity is <= patch_similarity_threshold become PATCH_NON_SIMILAR, and everything after (before) the first
        such frame in the forward (backward) direction REJECTED_AFTER_PATCH_WAS_NON_SIMILAR.  One native call
        (csrc/patch_filter.cu); rgbs (T,3,H,W) uint8, query_points (N,3), traj (T,N,2), vis (T,N) float -> vis (T,N)."""
        from ctypes import c_float, c_int
        from sampt_b200 import native
        T, _, H, W = rgbs.shape
        N = query_points.shape[0]
        vis = vis.contiguous().clone()
        sim = torch.empty((T, N), device=rgbs.device, dtype=torch.float32)
        ctx = native.get_context(rgbs.device)
        native.check(native.lib().sampt_patch_filter(
            ctx.handle, native.ptr(rgbs.contiguous()), c_int(T), c_int(H), c_int(W), native.ptr(query_points.float().contiguous()),
            native.ptr(traj.float().contiguous()), c_int(N), c_int(int(self.patch_size)), c_float(float(self.patch_similarity_threshold)),
            native.ptr(vis), native.ptr(sim), native.stream_ptr()), "patch_filter")
        self._last_patch_similarities = sim
        return vis

    # ------------------------------------------------------------------------------------------------ re-initialisation
    def _forward_w_reinit(self, images, query_points):
        """reference sam_pt.py:355-410: forward pass with point re-initialisation from SAM's own masks, run left-to-right and on
        the time-flipped clip, stitched per mask at its query frame.  Control flow as the reference; every tensor on the device."""
        n_frames = images.shape[0]
        query_points = query_points.to(self.device)
        traj_r, vis_r, logits_r, _, spf_r = self._forward_w_reinit_inner(images, query_points)
        qf = query_points.clone()
        qf[:, :, 0] = n_frames - query_points[:, :, 0] - 1
        traj_l, vis_l, logits_l, _, spf_l = self._forward_w_reinit_inner(images.flip(0), qf)
        traj_l, vis_l, logits_l = traj_l.flip(0), vis_l.flip(0), logits_l.flip(1)
        # NB the reference does not flip scores_per_frame of the flipped pass (sam_pt.py:386-388,401-402): reproduced
        ts = query_points[:, 0, 0].int().tolist()
        trajectories = torch.full_like(traj_r, torch.nan)
        visibilities = torch.full_like(vis_r, False)
        logits = torch.full_like(logits_r, torch.nan)
        scores_per_frame = torch.full_like(spf_r, torch.nan)
        for m, t in enumerate(ts):
            trajectories[t:, m], trajectories[:t, m] = traj_r[t:, m], traj_l[:t, m]
            visibilities[t:, m], visibilities[:t, m] = vis_r[t:, m], vis_l[:t, m]
            logits[m, t:], logits[m, :t] = logits_r[m, t:], logits_l[m, :t]
            scores_per_frame[t:, m], scores_per_frame[:t, m] = spf_r[t:, m], spf_l[:t, m]
        assert not torch.isnan(trajectories).any()
        assert not torch.isnan(logits).any()
        scores = scores_per_frame.nanmean(dim=0)
        return trajectories, visibilities, logits, scores, scores_per_frame

    def _forward_w_reinit_inner(self, images, query_points):
        """reference sam_pt.py:412-543."""
        n_frames, _, height, width = images.shape
        n_masks, points_per_mask, _ = query_points.shape
        assert self.reinit_point_tracker_horizon >= self.reinit_horizon
        dev = self.device
        trajectories = torch.full((n_frames, n_masks, points_per_mask, 2), torch.nan, dtype=torch.float32, device=dev)
        visibilities = torch.full((n_frames, n_masks, points_per_mask), False, dtype=torch.float32, device=dev)
        scores_per_frame = torch.full((n_frames, n_masks), torch.nan, dtype=torch.float32, device=dev)
        logits = torch.full((n_masks, n_frames, height, width), torch.nan, dtype=torch.float32, device=dev)
        current_query_points = query_points.clone()
        for start_frame in range(int(query_points[:, 0, 0].int().min().item()), n_frames):
            end_frame = min(start_frame + self.reinit_horizon, n_frames)
            end_frame_tracker = min(start_frame + self.reinit_point_tracker_horizon, n_frames)
            current_timesteps = current_query_points[:, 0, 0].int()
            tracked = current_timesteps == start_frame
            if tracked.sum() == 0:
                continue
            query_points_i = current_query_points[tracked].clone()
            query_points_i[:, :, 0] -= start_frame
            assert (query_points_i[:, :, 0] == 0).all()
            traj_i, vis_i = self._track_points(images[start_frame:end_frame_tracker], query_points_i)
            traj_i, vis_i = traj_i[:self.reinit_horizon], vis_i[:self.reinit_horizon]
            _, logits_i, spf_i = self._apply_sam_to_trajectories(images[start_frame:end_frame], traj_i, vis_i)
            logits_i = logits_i.type(torch.float32)
            logits[tracked, start_frame:end_frame] = logits_i
            pred_masks = logits_i > 0
            trajectories[start_frame:end_frame, tracked] = traj_i
            visibilities[start_frame:end_frame, tracked] = vis_i
            scores_per_frame[start_frame:end_frame, tracked] = spf_i
            if end_frame == n_frames:
                continue
            area = pred_masks[:, 1:, :, :].sum([2, 3]).float()
            area[area <= 25] = torch.nan
            if self.reinit_horizon // 4 < area.shape[1]:
                area[:, :self.reinit_horizon // 4] = torch.nan
            if self.reinit_variant == "reinit-on-horizon-and-sync-masks":
                next_timestep = self.reinit_horizon - 1 - 1
                other = current_timesteps[current_timesteps > start_frame]
                if len(other) > 0:
                    next_timestep = min(next_timestep, int(other.min().item()) - start_frame - 1)
                qts = torch.full((pred_masks.shape[0],), next_timestep, dtype=torch.int64, device=dev)
            elif self.reinit_variant == "reinit-at-median-of-area-diff":
                # host nanmedian: which index is returned among equal medians is the CPU implementation's (the reference runs it there)
                qts = area.cpu().nanmedian(dim=1).indices.to(dev)
            elif self.reinit_variant == "reinit-on-similar-mask-area":
                target = pred_masks[:, 0, :, :].sum([1, 2])
                diff = torch.abs(area - target[:, None])
                diff[diff.isnan()] = torch.inf
                qts = diff.argmin(dim=1)
            elif self.reinit_variant == "reinit-on-similar-mask-area-and-sync-masks":
                target = pred_masks[:, 0, :, :].sum([1, 2])
                diff = torch.abs(area - target[:, None]) / target[:, None]
                diff[diff.isnan()] = 720
                per_frame = diff.sum(dim=0)
                other = current_timesteps[current_timesteps > start_frame]
                if len(other) > 0:
                    per_frame[int(other.min().item()) - start_frame - 1] -= 36
                qts = torch.full((pred_masks.shape[0],), int(per_frame.argmin(dim=0).item()), dtype=torch.int64, device=dev)
            else:
                raise ValueError(f"Unknown reinit variant: {self.reinit_variant}")
            print(f"Horizon: {self.reinit_horizon}, Tracking horizon: {self.reinit_point_tracker_horizon}, "
                  f"    Next Timesteps: {qts.tolist()} / {self.reinit_horizon - 1 - 1}")
            ar = torch.arange(len(qts), device=dev)
            invalid = area[ar, qts] <= 0            # (False for NaN areas, exactly as the reference's comparison, sam_pt.py:505)
            if (~invalid).sum() > 0:
                qmasks = pred_masks[:, 1:, :, :][ar, qts].type(torch.float32)
                update = self.extract_query_points(images[start_frame + 1:end_frame], qmasks[~invalid], qts[~invalid].float())
                valid_tracked = tracked.clone()
                valid_tracked[tracked] = ~invalid
                current_query_points[valid_tracked] = update.to(current_query_points.device)
                current_query_points[valid_tracked, :, 0] += start_frame + 1
            if invalid.sum() > 0:
                invalid_tracked = tracked.clone()
                invalid_tracked[tracked] = invalid
                current_query_points[invalid_tracked, :, 0] = n_frames
                current_query_points[invalid_tracked, :, 1:] = 0
                trajectories[end_frame:, invalid_tracked] = -72
                visibilities[end_frame:, tracked] = float(PointVisibilityType.REINIT_FAILED.value)
                logits[invalid_tracked, end_frame:] = -float("inf")
        scores = scores_per_frame.nanmean(dim=1)
        return trajectories, visibilities, logits, scores, scores_per_frame

    # ------------------------------------------------------------------------------------------------ SAM
    @torch.no_grad()
    def _apply_sam_to_trajectories(self, images, trajectories, visibilities, pre=None):
        """reference sam_pt.py:694-866.  images (T,3,H,W) uint8 on the device."""
        n_frames = images.shape[0]
        logits, scores_pf, counted = self._apply_sam_to_frames(images, list(range(n_frames)), trajectories, visibilities, pre=pre)
        counted_d = counted.to(self.device)
        cnt = counted_d.sum(dim=0).clamp(min=1)
        pred_scores = torch.where(counted_d, scores_pf, torch.zeros_like(scores_pf)).sum(dim=0) / cnt
        return pred_scores, logits, scores_pf

    @torch.no_grad()
    def _apply_sam_to_frames(self, images, frame_ids, trajectories, visibilities, pre=None):
        """SAM on a subset of frames: images (n,3,H,W) uint8 on the device are the frames `frame_ids` of the clip whose
        full-clip trajectories (T,M,P,2) / visibilities (T,M,P) are given.  Returns logits (M,n,H,W), scores (n,M) on the
        device and `counted` (n,M) bool on the host (frames with at least one visible point)."""
        return self._apply_sam_multi(images, [(0, f) for f in frame_ids], [(trajectories, visibilities)], pre=pre)[0]

    @torch.no_grad()
    def _apply_sam_multi(self, images, frame_specs, clips, pre=None):
        """SAM over frames that may belong to SEVERAL clips (the frame-sharded multi-GPU path batches the owned frames of all
        clips through the encoder together): images (n,3,H,W) uint8; frame_specs[i] = (clip index, frame id inside that clip);
        clips[c] = (trajectories (T,M,P,2), visibilities (T,M,P)).  Per clip, in the order its frames appear in `images`:
        (logits (M,n_c,H,W), scores (n_c,M) on the device, counted (n_c,M) bool on the host)."""
        n_sub, _, height, width = images.shape
        dev = self.device
        pred = self.sam_predictor
        # the only device->host copy before the results: a few KB of trajectories / visibility codes per clip
        host = [(t.detach().cpu(), v.detach().cpu()) for t, v in clips]
        for t, v in host:
            assert v.shape == t.shape[:3]

        def prepare_points(c, f, m):  # sam_pt.py:726-758
            traj_h, vis_h = host[c]
            n_masks = traj_h.shape[1]
            pc = traj_h[f, m]
            labels = np.ones((len(pc)), dtype=int)
            if self.negative_points_per_mask > 0:
                labels[self.positive_points_per_mask:] = 0
            vmask = (vis_h[f, m] == 1)
            coords = pc[vmask].numpy()
            labels = labels[vmask.numpy()]
            if n_masks > 1 and self.add_other_objects_positive_points_as_negative_points:
                other = torch.cat([traj_h[f, o, :self.positive_points_per_mask][vis_h[f, o, :self.positive_points_per_mask] == 1]
                                   for o in range(n_masks) if o != m], dim=0).numpy()
                if self.max_other_objects_positive_points is not None and len(other) > self.max_other_objects_positive_points:
                    idx = np.random.choice(len(other), self.max_other_objects_positive_points, replace=False)
                    other = other[idx]
                coords = np.concatenate([coords, other], axis=0)
                labels = np.concatenate([labels, np.zeros((len(other)), dtype=int)], axis=0)
            return coords, labels

        n_of = [sum(1 for c, _ in frame_specs if c == ci) for ci in range(len(clips))]
        outs = []
        for ci, (t, _) in enumerate(host):
            M = t.shape[1]
            outs.append([torch.full((M, n_of[ci], height, width), -float("inf"), device=dev, dtype=torch.float32),
                         torch.full((n_of[ci], M), -float("inf"), device=dev, dtype=torch.float32),
                         torch.zeros((n_of[ci], M), dtype=torch.bool)])
        pos_in_clip = [0] * len(clips)
        n_ref = int(self.iterative_refinement_iterations) if self.iterative_refinement_iterations else 0
        B = max(1, int(self.encoder_batch))
        want_interm = pred._uses_interm()
        main = torch.cuda.current_stream()
        nslot = max(1, int(self.decode_streams))
        if not getattr(pred.model, "use_cuda_graphs", True) or not pred.model.has_decoder_slab():
            nslot = 1   # the eager chain allocates from ONE shared workspace: concurrent streams would race on it
        if nslot > 1 and (self._dec_streams is None or len(self._dec_streams) != nslot):
            self._dec_streams = [torch.cuda.Stream(device=dev) for _ in range(nslot)]
        used = set()
        thr = float(self.sam_iou_threshold)
        for ci_chunk, f0 in enumerate(range(0, n_sub, B)):
            chunk = images[f0:f0 + B]
            ev = None
            if pre is not None:  # encoder output produced on the encoder stream (see _start_encoder)
                enc, ev = pre[ci_chunk]
            else:
                enc = pred.encode_frames(chunk, want_interm=want_interm)
                if nslot > 1:
                    ev = torch.cuda.Event()
                    ev.record(main)
            feats, interm = enc if want_interm else (enc, None)
            for j in range(chunk.shape[0]):
                i = f0 + j
                c, f = frame_specs[i]
                k = pos_in_clip[c]
                pos_in_clip[c] += 1
                logits, scores_pf, counted = outs[c]
                slot = i % nslot
                stream = self._dec_streams[slot] if nslot > 1 else main
                if nslot > 1 and slot not in used:
                    stream.wait_stream(main)  # logits / scores buffers were created on the main stream
                    used.add(slot)
                with torch.cuda.stream(stream):
                    if ev is not None:
                        stream.wait_event(ev)
                    pred.set_frames_features((height, width), (feats[j:j + 1], interm[j:j + 1]) if want_interm else feats[j:j + 1])
                    for m in range(logits.shape[0]):
                        coords, labels = prepare_points(c, f, m)
                        if len(coords) == 0:
                            continue  # all points invisible -> mask stays -inf, score -inf (sam_pt.py:766-767,855)
                        c1024 = torch.as_tensor(pred.transform.apply_coords(coords, pred.original_size), dtype=torch.float, device=dev)
                        lab = torch.as_tensor(labels, dtype=torch.int, device=dev)
                        pos_idx = np.nonzero(labels == 1)[0].tolist() if self.negative_points_per_mask > 0 else None
                        iou, _, _ = pred.predict_refine(c1024, lab, 1 if self.negative_points_per_mask > 0 else 0, n_ref, logits[m, k],
                                                        slot=slot, positive_index=pos_idx)
                        # "Mask is empty if SAM's IoU score is too low" (sam_pt.py:833-835), without a host round trip
                        logits[m, k] = torch.where(iou[0] < thr, torch.full_like(logits[m, k], -float("inf")), logits[m, k])
                        scores_pf[k, m] = iou[0]
                        counted[k, m] = True
            if nslot > 1:
                for t in (enc if isinstance(enc, tuple) else (enc,)):
                    for sl in used:
                        t.record_stream(self._dec_streams[sl])
        if nslot > 1:
            for sl in used:
                main.wait_stream(self._dec_streams[sl])
        return [tuple(o) for o in outs]

    # ------------------------------------------------------------------------------------------------ multi-GPU
    @torch.no_grad()
    def forward_clips_sharded(self, videos, gather_logits: bool = False):
        """Frame-sharded processing of `len(videos)` clips across the ranks of the default process group (SURVEY §8e):
        frame f of clip c belongs to rank (f + c) mod G (sampt_b200/sharding.py: rotated round-robin, every rank owns the same
        number of frames).
          A. local : the tracker's encoder (PIPS fnet on uint8 frames; CoTracker: resize to interp_shape + fnet) on ALL owned
                     frames of all clips in one pass; the SAM ViT on the same frames starts on its own stream, 10 frames per launch
          B. NCCL  : ONE all-gather of the fp32 feature maps (13 MB/frame @480x854 for PIPS, 6.3 MB/frame @384x512 for
                     CoTracker) -> every rank holds all features of every clip
          C. local : tracker chain of clip c on rank c mod G (pyramid built locally after the gather)
          D. NCCL  : all-gather of the (T,N,3) trajectories/visibilities (a few KB)
          E. local : prompt + mask decode on the owned frames
        Returns, per clip, {"trajectories","visibilities","logits" (M, n_owned, H, W), "frame_ids", "scores_per_frame"}
        (logits stay sharded unless gather_logits).  Every tensor stays on the device (`outputs_on_cpu` is `forward`'s).
        The masks of a clip are tracked `point_tracker_mask_batch_size` at a time, as `_track_points` does, so the results are
        those of `forward` also for trackers whose points interact (CoTracker).  Outside the path and raising before any
        launch: point re-initialisation, patch-matching filtering, queries given as masks, `target_hw` different from the
        frame size, clips of different frame sizes, a tracker without `shard_features` / `track_on_features`.
        The three local stages take (rank, world) explicitly, so that one process can run them for every rank in turn."""
        import torch.distributed as dist
        from sampt_b200 import sharding
        world, rank = dist.get_world_size(), dist.get_rank()
        state = self._sharded_encode(videos, rank, world)                                           # A
        fulls = sharding.allgather_clips(state["locs"], state["Ts"])                                # B (one collective for all clips)
        slab = self._sharded_track(state, fulls, rank, world)                                       # C
        del fulls
        gathered = torch.empty((world,) + tuple(slab.shape), device=slab.device)                    # D (tiny)
        dist.all_gather_into_tensor(gathered.view((world * slab.shape[0],) + tuple(slab.shape[1:])), slab)
        results = self._sharded_decode(state, gathered, rank, world)                                # E
        if gather_logits:
            for c, T in enumerate(state["Ts"]):   # (clips may carry different numbers of masks: one collective per clip)
                full = sharding.allgather_frames(results[c]["logits"].transpose(0, 1).contiguous(), T, clip=c)
                results[c]["logits"] = full.transpose(0, 1)
                results[c]["frame_ids"] = list(range(T))
        return results

    def _check_sharded_inputs(self, videos):
        """What `forward` does and the frame-sharded path does not is refused here, before anything is uploaded or launched."""
        trk = self.point_tracker
        if not (hasattr(trk, "shard_features") and hasattr(trk, "track_on_features")):
            raise NotImplementedError(f"{type(trk).__name__} has no frame-sharded path (needs shard_features / track_on_features)")
        if self.use_point_reinit:
            raise NotImplementedError("use_point_reinit is not built on the frame-sharded path (it re-tracks from SAM's own masks)")
        if self.use_patch_matching_filtering:
            raise NotImplementedError("use_patch_matching_filtering is not built on the frame-sharded path")
        hw = tuple(videos[0]["image"][0].shape[-2:])
        for c, v in enumerate(videos):
            if v.get("query_points") is None:
                raise NotImplementedError(f"clip {c}: the frame-sharded path takes query_points; query_masks are not sampled here")
            if any(tuple(f.shape[-2:]) != hw for f in v["image"]):
                raise ValueError(f"clip {c}: the frame-sharded path batches the frames of all clips, which must share one frame size "
                                 f"({hw} in clip 0)")
            if v.get("target_hw") is not None and tuple(int(x) for x in v["target_hw"]) != hw:
                raise ValueError(f"clip {c}: target_hw {tuple(v['target_hw'])} differs from the frame size {hw}; the frame-sharded "
                                 f"path returns masks and trajectories at the frame size only")

    @torch.no_grad()
    def _sharded_encode(self, videos, rank, world):
        """Stage A on `rank` of `world`: upload the owned frames of every clip as one batch, start the SAM encoder on them and
        run the tracker's encoder.  `locs[c]` = features of the owned frames of clip c (the all-gather payload)."""
        from sampt_b200 import sharding
        self._check_sharded_inputs(videos)
        dev = self.device
        trk = self.point_tracker.to(dev)
        C = len(videos)
        Ts = [len(v["image"]) for v in videos]
        own = [sharding.owned_frames(Ts[c], rank, world, c) for c in range(C)]
        h, w = videos[0]["image"][0].shape[-2:]
        # upload only the owned frames (async from pinned memory), one batch for every clip
        specs = [(c, f) for c in range(C) for f in own[c]]
        if len(specs) == 0:
            all_own = torch.empty((0, 3, h, w), dtype=torch.uint8, device=dev)
        else:
            all_own = torch.stack([videos[c]["image"][f].to(dev, non_blocking=True) for c, f in specs], dim=0)
        pre = self._start_encoder(all_own) if (self.overlap_streams and len(specs) > 0) else None
        fm_all = trk.shard_features(all_own)                      # (n_own_total, H4, W4, 128)
        locs, off = [], 0
        for c in range(C):
            locs.append(fm_all[off:off + len(own[c])])
            off += len(own[c])
        return {"Ts": Ts, "own": own, "hw": (h, w), "specs": specs, "all_own": all_own, "pre": pre, "locs": locs,
                "queries": [v["query_points"] for v in videos]}

    @torch.no_grad()
    def _sharded_track(self, state, fulls, rank, world):
        """Stage C: the tracker chain of clip c on rank c % world, on the gathered features `fulls[c]` (T_c, H4, W4, 128).
        Returns the (n_slots, T_max, N_max, 3) slab of (x, y, visibility) this rank contributes to the second all-gather:
        slot i holds clip rank + i * world."""
        dev = self.device
        trk = self.point_tracker
        Ts, queries = state["Ts"], state["queries"]
        bs = self.point_tracker_mask_batch_size
        N_max = max(q.shape[0] * q.shape[1] for q in queries)
        slab = torch.zeros(((len(Ts) + world - 1) // world, max(Ts), N_max, 3), device=dev)
        for c in range(rank, len(Ts), world):
            q = queries[c]
            P = q.shape[1]
            parts = []
            for i in range(0, q.shape[0], bs):   # the mask batches of _track_points: a CoTracker call mixes the points it is given
                qb = q[i:i + bs].to(dev)
                traj, vis = trk.track_on_features(fulls[c], qb.reshape(1, qb.shape[0] * P, 3), state["hw"])
                parts.append(torch.cat([traj[0], vis[0].float()[..., None]], dim=-1))  # (T, m * P, 3)
            tv = torch.cat(parts, dim=1)
            slab[c // world, : tv.shape[0], : tv.shape[1]] = tv
        return slab

    @torch.no_grad()
    def _sharded_decode(self, state, gathered, rank, world):
        """Stage E: gathered (world, n_slots, T_max, N_max, 3) = the slabs of `_sharded_track` of every rank, in rank order;
        out-of-frame relabel as in `_track_points`, then prompt + mask decode on the owned frames."""
        h, w = state["hw"]
        Ts = state["Ts"]
        clips = []
        for c, q in enumerate(state["queries"]):
            M, P, _ = q.shape
            tv = gathered[c % world, c // world, : Ts[c], : M * P]
            traj = tv[..., :2].reshape(Ts[c], M, P, 2)
            vis = tv[..., 2].reshape(Ts[c], M, P)
            out_code = float(PointVisibilityType.OUTSIDE_FRAME.value)
            oob = (traj[..., 0] / w < 0.01) | (traj[..., 1] / h < 0.01) | (traj[..., 0] / w > 0.99) | (traj[..., 1] / h > 0.99)
            clips.append((traj, torch.where(oob, torch.full_like(vis, out_code), vis)))
        decoded = self._apply_sam_multi(state["all_own"], state["specs"], clips, pre=state["pre"])
        return [{"trajectories": clips[c][0], "visibilities": clips[c][1], "logits": decoded[c][0], "frame_ids": state["own"][c],
                 "scores_per_frame": decoded[c][1]} for c in range(len(Ts))]
