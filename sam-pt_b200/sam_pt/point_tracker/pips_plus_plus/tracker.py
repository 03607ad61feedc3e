"""`PipsPlusPlusPointTracker` drop-in (reference sam_pt/point_tracker/pips_plus_plus/tracker.py:10-134): same constructor
kwargs (configs/model/point_tracker/pips_plus_plus.yaml), same forward contract; the work happens in libsampt_b200."""
from collections import defaultdict

import torch

from sam_pt.point_tracker.pips_plus_plus.pips_plus_plus import PipsPlusPlus, resize_frames
from sam_pt.point_tracker.tracker import PointTracker
from sam_pt.point_tracker.utils import saverloader


class PipsPlusPlusPointTracker(PointTracker):

    def __init__(self, checkpoint_path, stride=8, max_sequence_length=128, iters=16, image_size=(512, 896)):
        super().__init__()
        self.checkpoint_path = checkpoint_path
        self.stride = stride
        self.max_sequence_length = max_sequence_length
        self.iters = iters
        self.image_size = tuple(image_size) if image_size is not None else None
        print(f"Loading PIPS++ model from {self.checkpoint_path}")
        self.model = PipsPlusPlus(stride=self.stride)
        self._loaded_checkpoint_step = None
        if checkpoint_path is not None:
            self._loaded_checkpoint_step = saverloader.load(self.checkpoint_path, self.model)
        if torch.cuda.is_available():
            self.model = self.model.cuda()

    @property
    def device(self):
        return self.model.device

    def forward(self, rgbs, query_points):
        """rgbs (1,T,3,H,W) 0..255, query_points (1,N,3) (t,x,y) -> trajectories (1,T,N,2), visibilities (1,T,N) float ones.

        Per query timestep t: a left-to-right pass on frames t..T-1 and a time-reversed pass on frames t..0, merged as
        `right[:-1] ++ left` (reference tracker.py:81-122).  Where the reference breaks, each point gets its own stitched
        trajectory instead: with two or more distinct query timesteps (the reference raises IndexError, tracker.py:120-122
        rebinds `idx`) and with a query on the last frame (the reference returns T-1 frames; here frame t is the query).
        With image_size, x is scaled by image_size[0]/H and y by image_size[1]/W, in place on `query_points` as the reference
        does (tracker.py:78-79), and the trajectories are scaled back by the inverse ratios (:131-132)."""
        B, T, C, H, W = rgbs.shape
        if B != 1 or query_points.shape[0] != 1:
            raise NotImplementedError("Batch size > 1 is not supported for PIPS++ yet")
        if T < 2:
            raise ValueError("PIPS++ tracks over at least 2 frames")
        dev = self.device
        frames = rgbs[0].to(dev)
        if frames.dtype != torch.uint8:
            frames = frames.float()   # used as given, 2*(rgbs/255)-1 like the reference
        if self.image_size is not None:
            frames = resize_frames(self.model, frames, self.image_size)
            query_points[:, :, 1] *= self.image_size[0] / H
            query_points[:, :, 2] *= self.image_size[1] / W
        pyr = self.model.encode_frames(frames)
        groups = defaultdict(list)
        for idx, t in enumerate(query_points[0, :, 0].tolist()):
            groups[int(t)].append(idx)
        N = query_points.shape[1]
        traj = torch.empty((T, N, 2), device=dev, dtype=torch.float32)
        L, iters = int(self.max_sequence_length), int(self.iters)
        for t, idx in groups.items():
            ii = torch.tensor(idx, device=dev)
            q = query_points[0, idx, 1:].float().to(dev)
            left = self.model.track(pyr, q, t, 1, T - t, L, iters) if t < T - 1 else q[None]
            if t > 0:
                right = self.model.track(pyr, q, t, -1, t + 1, L, iters).flip(0)
                traj[:t, ii] = right[:-1]
            traj[t:, ii] = left
        if self.image_size is not None:
            traj[..., 0] *= H / self.image_size[0]
            traj[..., 1] *= W / self.image_size[1]
        return traj[None], torch.ones((1, T, N), device=dev, dtype=torch.float32)
