"""`PipsPointTracker` drop-in (reference sam_pt/point_tracker/pips/tracker.py:9-201): same constructor kwargs
(configs/model/point_tracker/pips.yaml), same forward contract; the work happens in libsampt_b200."""
import torch

from sam_pt.point_tracker.pips.pips import Pips
from sam_pt.point_tracker.tracker import PointTracker
from sam_pt.point_tracker.utils import saverloader


class PipsPointTracker(PointTracker):
    def __init__(self, checkpoint_path, stride, s, initial_next_frame_visibility_threshold=0.9):
        super().__init__()
        self.checkpoint_path = checkpoint_path
        self.stride = stride
        self.s = s
        self.initial_next_frame_visibility_threshold = initial_next_frame_visibility_threshold
        print(f"Loading PIPS model from {self.checkpoint_path}")
        self.model = Pips(S=s, stride=stride)
        self._loaded_checkpoint_step = None
        if checkpoint_path is not None:
            self._loaded_checkpoint_step = saverloader.load(self.checkpoint_path, self.model)
        if torch.cuda.is_available():
            self.model = self.model.cuda()

    @property
    def device(self):
        return self.model.norm.weight.device

    def forward(self, rgbs, query_points):
        """rgbs (1,T,3,H,W) uint8 on the GPU, query_points (1,N,3) -> (1,T,N,2) float32, (1,T,N) bool.
        L->R pass, time-reversed R->L pass, per-point stitch `left[:t_q] | right[t_q:]` (reference tracker.py:155-201)."""
        if rgbs.shape[0] != 1:
            raise NotImplementedError("Batch size > 1 is not supported for PIPS yet")
        dev = self.device
        frames = rgbs[0].to(dev)
        if frames.dtype != torch.uint8:
            frames = frames.round().clamp(0, 255).to(torch.uint8)
        pyr = self.model.encode_frames(frames)
        return self._track_pyramid(pyr, query_points)

    # ---- frame-sharded multi-GPU path (SamPt.forward_clips_sharded): encoder on the owned frames, chain on gathered features
    def shard_features(self, frames_u8):
        """(n,3,H,W) uint8 frames this rank owns -> (n,H/4,W/4,128) fp32 BasicEncoder features (the all-gather payload)."""
        frames_u8 = frames_u8.to(self.device)
        if frames_u8.shape[0] == 0:   # a rank that owns no frame (more ranks than frames) contributes an empty payload
            H, W = frames_u8.shape[-2:]
            return torch.empty((0, H // 4, W // 4, 128), device=self.device, dtype=torch.float32)
        return self.model.fnet_frames(frames_u8)

    def track_on_features(self, fmaps, query_points, frame_hw=None):
        """fmaps (T,H/4,W/4,128): every frame's features in frame order (after the all-gather); the pyramid is built locally."""
        return self._track_pyramid(self.model.build_pyramid(fmaps), query_points)

    def _track_pyramid(self, pyr, query_points):
        """The linked bidirectional chain on pre-computed feature pyramids."""
        dev = self.device
        q = query_points[0].float().to(dev)
        T = pyr[0].shape[0]
        thr = float(self.initial_next_frame_visibility_threshold)
        traj_r, vis_r = self.model.track(pyr, q, thr, iters=6, flip=False)
        start = q[:, 0].long()
        if bool((start > 0).any()):
            traj_l, vis_l = self.model.track(pyr, q, thr, iters=6, flip=True)
            traj_l, vis_l = traj_l.flip(0), vis_l.flip(0)
            left = torch.arange(T, device=dev)[:, None] < start[None, :]
            traj = torch.where(left[:, :, None], traj_l, traj_r)
            vis = torch.where(left, vis_l, vis_r)
        else:
            # every point is born at t=0: the reversed pass has no frame to process (reference tracker.py:67 never
            # reaches index T-1), so the stitched result is the L->R pass
            traj, vis = traj_r, vis_r
        return traj[None], (vis > 0.5)[None]
