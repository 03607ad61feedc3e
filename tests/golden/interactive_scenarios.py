"""Inputs of the interactive point-correction golden (tests/golden/interactive_forward.npz): seeded synthetic SAM (the ViT
structural twin `vit_test`) and PIPS weights, a 6-frame 96x128 clip with 3 query points and moving-ellipse ground truth, and
the three configurations the golden covers.  Everything is re-generated from seeds."""
import numpy as np
import torch

T, H, W, P = 6, 96, 128, 3
SAM_SEED, PIPS_SEED, CLIP_SEED, TORCH_SEED = 31, 7201, 11, 1234
REFINEMENTS = 12

SCENARIOS = {
    "online": dict(online=True, online_interactive_iou_threshold=0.95, interactions_max=14),
    "offline": dict(online=False, interactions_max=16),
    "no_tracking": dict(disable_point_tracking=True, interactions_max_per_frame=2),
}


def ellipse(h, w, cy, cx, ry, rx):
    yy, xx = np.mgrid[:h, :w]
    return ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1.0


def video():
    from sampt_b200 import synth
    v = synth.make_video_dict(T, H, W, P, seed=CLIP_SEED)
    v["video_id"] = "synthetic"
    v["gt_masks"] = [torch.from_numpy(ellipse(H, W, 40 + 2 * t, 50 + 3 * t, 22, 30))[None] for t in range(T)]
    return v


def sam_state_dict(hq=False):
    from oracle import sam_ref
    from sampt_b200 import synth
    return synth.condition_sam(synth.make_state_dict(sam_ref.sam_state_dict_shapes(sam_ref.VIT_TEST, hq=hq), SAM_SEED))


def pips_state_dict():
    from oracle import pips_ref
    from sampt_b200 import synth
    return synth.condition_pips(synth.make_state_dict(pips_ref.pips_state_dict_shapes(), PIPS_SEED))
