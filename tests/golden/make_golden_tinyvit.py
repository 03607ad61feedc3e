"""Golden fixture of SamPt with MobileSAM / Light HQ-SAM (TinyViT-5M) and PIPS on the first 16 frames of the C2 clip
(480x854, seed 72, 8 positive points), at 3 and at 12 refinements.

    python tests/golden/make_golden_tinyvit.py

What runs: `oracle/sampt_ref.sampt_forward` with the PIPS restatement `oracle/pips_ref.py` (equal to the unmodified reference
tracker bit for bit on the full C2 clip, DESIGN §2) and `oracle/tinyvit_ref.RefTinySamPredictor` (the float32 TinyViT
restatement in front of the SAM oracle).  Weights and clip are re-generated from seeds (`sampt_b200.synth`); only the outputs
are stored: tests/golden/tinyvit_c2_16.npz with, per "<model>_r<refinements>", trajectories (T,N,2), visibilities (T,N) and
the bit-packed `logits > 0` of every frame.  tests/test_gpu_tinyvit.py::test_sampt_pips_c2_16_frames reads it.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for _p in (ROOT, os.path.join(ROOT, "sam-pt_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from sampt_b200 import synth  # noqa: E402

OUT = os.path.join(HERE, "tinyvit_c2_16.npz")
T, H, W, P, SEED = 16, 480, 854, 8, 72
PIPS_SEED, SAM_SEED, TINYVIT_SEED = 7201, 61, 5
MODELS = (("mobile_sam", False), ("light_hq_sam", True))
REFINEMENTS = (3, 12)


def sam_state_dict(hq: bool):
    """MobileSAM (hq=False) / Light HQ-SAM (hq=True) checkpoint under upstream key names: conditioned random SAM prompt
    encoder and mask decoder (synth.condition_sam), TinyViT from synth.make_tinyvit_state_dict."""
    from sampt_b200 import factory
    sam = factory.build_sam(factory.TINY_VIT, hq=hq)
    shapes = {k: tuple(v.shape) for k, v in sam.state_dict().items()
              if not k.startswith("image_encoder.") and k not in ("pixel_mean", "pixel_std")}
    sd = synth.condition_sam(synth.make_state_dict(shapes, SAM_SEED))
    for k, v in synth.make_tinyvit_state_dict(TINYVIT_SEED).items():
        sd["image_encoder." + k] = v
    return sd


def pips_state_dict():
    from oracle import pips_ref
    return synth.condition_pips(synth.make_state_dict(pips_ref.pips_state_dict_shapes(), PIPS_SEED))


def video():
    """The first T frames of the 50-frame C2 clip (query points on frame 0)."""
    v = synth.make_video_dict(50, H, W, P, seed=SEED)
    v["image"], v["info"] = v["image"][:T], v["info"][:T]
    return v


def main():
    from oracle import sampt_ref, tinyvit_ref
    torch.manual_seed(0)
    pips_sd, vid = pips_state_dict(), video()
    out = {}
    for name, hq in MODELS:
        sd = sam_state_dict(hq)
        for n_ref in REFINEMENTS:
            ref = sampt_ref.sampt_forward(pips_sd, tinyvit_ref.RefTinySamPredictor(sd, hq=hq), vid, positive_points_per_mask=P,
                                          iterative_refinement_iterations=n_ref, sam_iou_threshold=-1e9)
            key = f"{name}_r{n_ref}"
            out[key + "_traj"] = ref["trajectories"].numpy()
            out[key + "_vis"] = ref["visibilities"].numpy()
            masks = torch.stack([ref["logits"][0][f] > 0 for f in range(T)]).numpy()
            out[key + "_masks"] = np.packbits(masks.reshape(T, -1), axis=1)
            print(key, "mask area per frame:", masks.reshape(T, -1).sum(1).tolist())
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
