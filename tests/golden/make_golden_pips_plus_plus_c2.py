"""Golden fixture of SamPt with SAM ViT-B and PIPS++ on the first 16 frames of the C2 clip (480x854, seed 72, 8 positive
points), 12 refinements (build container only).

    python tests/golden/make_golden_pips_plus_plus_c2.py

What runs: the UNMODIFIED reference PipsPlusPlusPointTracker on CPU (imported as in make_golden_pips_plus_plus.py, with
`Tensor.cuda()` made the identity), configured as configs/model/point_tracker/pips_plus_plus.yaml (stride 8, 128-frame
windows, 16 iterations, image_size null), plugged into `oracle/sampt_ref.sampt_forward` with the SAM ViT-B oracle
`oracle/sam_ref.RefSamPredictor`.  Weights and clip are re-generated from seeds (`sampt_b200.synth`); only the outputs are
stored: tests/golden/pips_plus_plus_c2_16.npz with the reference tracker's trajectories (T,N,2), SamPt's trajectories and
visibilities, and the bit-packed `logits > 0` of every frame.  tests/test_gpu_pips_plus_plus.py reads it.
"""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for _p in (HERE, ROOT, os.path.join(ROOT, "sam-pt_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from sampt_b200 import synth  # noqa: E402

OUT = os.path.join(HERE, "pips_plus_plus_c2_16.npz")
T, H, W, P, SEED = 16, 480, 854, 8, 72
SAM_SEED = 61
REFINEMENTS = 12


def sam_state_dict():
    from oracle import sam_ref
    return synth.condition_sam(synth.make_state_dict(sam_ref.sam_state_dict_shapes(sam_ref.VIT_B), SAM_SEED))


def video():
    """The first T frames of the 50-frame C2 clip (query points on frame 0)."""
    v = synth.make_video_dict(50, H, W, P, seed=SEED)
    v["image"], v["info"] = v["image"][:T], v["info"][:T]
    return v


def main():
    from make_golden_pips_plus_plus import import_reference
    from oracle import sam_ref, sampt_ref
    torch.set_num_threads(8)
    torch.Tensor.cuda = lambda self, *a, **k: self
    R = import_reference()
    sd = synth.make_pips_plus_plus_state_dict()
    with tempfile.TemporaryDirectory() as d:
        synth.write_pips_checkpoint_dir(sd, d)
        trk = R["Tracker"](checkpoint_path=d, stride=8, max_sequence_length=128, iters=16, image_size=None).eval()
    raw = {}

    def tracker(images_u8, q):
        with torch.no_grad():
            traj, vis = trk(images_u8.float(), q.clone())
        raw.setdefault("traj", traj[0].clone())
        return traj, vis

    vid = video()
    ref = sampt_ref.sampt_forward(None, sam_ref.RefSamPredictor(sam_state_dict(), sam_ref.VIT_B), vid, positive_points_per_mask=P,
                                  iterative_refinement_iterations=REFINEMENTS, sam_iou_threshold=-1e9, tracker=tracker)
    masks = torch.stack([ref["logits"][0][f] > 0 for f in range(T)]).numpy()
    print("mask area per frame:", masks.reshape(T, -1).sum(1).tolist())
    np.savez_compressed(OUT, tracker_traj=raw["traj"].numpy(), traj=ref["trajectories"].numpy(), vis=ref["visibilities"].numpy(),
                        masks=np.packbits(masks.reshape(T, -1), axis=1))
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
