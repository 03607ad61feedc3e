"""Seeded synthetic clips, query points and checkpoints (SURVEY.md §8d).

There are no datasets or checkpoints on the box (no network), so every parity
test, the smoke test and bench.py draw their inputs from here.  Nothing in this
file is model code; both the CUDA path and the oracle load the SAME state-dicts
produced here.

Recipe (all from ``torch.Generator().manual_seed(seed)``; 72 is the reference's
default seed, ``/root/reference/configs/vos_eval_root.yaml:14``):

* clip: smooth textured background (uniform noise at H/12 x W/12, bicubic
  up-sampled) translating (+2,+1) px/frame, plus one textured ellipse
  (axes 0.18W x 0.22H) on an independent pattern moving on a Lissajous path,
  occluded for 6 frames at mid-clip by a static bar;
* query points: P points drawn uniformly inside the ellipse at t=0;
* weights: torch-default-style init by shape; PIPS ``delta_block.to_delta.15``
  scaled x0.1 so the random-weight tracker is contractive (SURVEY §0.4).
"""
from __future__ import annotations

import math
import os
from typing import Dict, Tuple

import torch
import torch.nn.functional as F

REF_SEED = 72


# --------------------------------------------------------------------------- #
# clip
# --------------------------------------------------------------------------- #
def _texture(gen: torch.Generator, h: int, w: int, cell: int = 12) -> torch.Tensor:
    """(3,h,w) float in [0,1]: low-res uniform noise, bicubic up-sampled."""
    lo = torch.rand((1, 3, max(h // cell, 2), max(w // cell, 2)), generator=gen)
    up = F.interpolate(lo, size=(h, w), mode="bicubic", align_corners=False)
    return up[0].clamp(0, 1)


def make_clip(T: int, H: int, W: int, seed: int = REF_SEED) -> Dict[str, torch.Tensor]:
    """Returns {"frames": uint8 (T,3,H,W), "centers": (T,2) ellipse centre xy, "axes": (2,)}."""
    gen = torch.Generator().manual_seed(seed)
    pad = 2 * T + 8
    bg = _texture(gen, H + pad, W + 2 * pad)
    obj = _texture(gen, H, W, cell=6)
    ax, ay = 0.18 * W / 2 * 2, 0.22 * H / 2 * 2  # full axes per the survey recipe
    ax, ay = ax / 2, ay / 2  # semi-axes
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    frames = torch.empty((T, 3, H, W), dtype=torch.uint8)
    centers = torch.empty((T, 2))
    bar_x0, bar_x1 = int(0.47 * W), int(0.53 * W)
    occ0 = T // 2 - 3
    for t in range(T):
        dx, dy = 2 * t, 1 * t
        img = bg[:, dy:dy + H, dx:dx + W].clone()
        ph = 2 * math.pi * t / max(T, 2)
        cx = W * (0.5 + 0.22 * math.sin(ph))
        cy = H * (0.5 + 0.18 * math.sin(2 * ph + 0.5))
        centers[t, 0], centers[t, 1] = cx, cy
        inside = ((xs - cx) / ax) ** 2 + ((ys - cy) / ay) ** 2 <= 1.0
        # the object carries its own texture, sampled in object coordinates (integer shift)
        sx, sy = int(round(cx - W / 2)), int(round(cy - H / 2))
        obj_shift = torch.roll(obj, shifts=(sy, sx), dims=(1, 2))
        img = torch.where(inside[None], 0.25 + 0.75 * obj_shift, img)
        if occ0 <= t < occ0 + 6 and T >= 12:
            img[:, :, bar_x0:bar_x1] = 0.35
        frames[t] = (img * 255.0).round().clamp(0, 255).to(torch.uint8)
    return {"frames": frames, "centers": centers, "axes": torch.tensor([ax, ay])}


def make_query_points(clip: Dict[str, torch.Tensor], P: int, seed: int = REF_SEED, t: int = 0) -> torch.Tensor:
    """(1,P,3) float32 (t,x,y): P points uniformly inside the ellipse at frame t."""
    gen = torch.Generator().manual_seed(seed + 1000)
    cx, cy = clip["centers"][t].tolist()
    ax, ay = clip["axes"].tolist()
    r = torch.sqrt(torch.rand(P, generator=gen)) * 0.85
    th = torch.rand(P, generator=gen) * 2 * math.pi
    x = cx + ax * r * torch.cos(th)
    y = cy + ay * r * torch.sin(th)
    q = torch.stack([torch.full((P,), float(t)), x, y], dim=1)
    return q[None].float()


def make_video_dict(T: int, H: int, W: int, P: int, seed: int = REF_SEED):
    """The dict ``SamPt.forward`` takes (reference sam_pt/modeling/sam_pt.py:122-160; demo/demo.py:114-131)."""
    clip = make_clip(T, H, W, seed)
    return {
        "video_name": f"synthetic_{T}x{H}x{W}_seed{seed}",
        "video_id": 0,
        "image": [f for f in clip["frames"]],
        "info": [{"frame": i, "save": True, "shape": (H, W), "need_resize": False} for i in range(T)],
        "target_hw": (H, W),
        "query_points": make_query_points(clip, P, seed),
    }


# --------------------------------------------------------------------------- #
# weights
# --------------------------------------------------------------------------- #
def _init_like_torch(name: str, shape: Tuple[int, ...], gen: torch.Generator) -> torch.Tensor:
    """Default-torch-style init decided from the tensor's name/shape only."""
    leaf = name.rsplit(".", 1)[-1]
    if "rel_pos" in name or leaf == "pos_embed":
        return torch.randn(shape, generator=gen) * 0.02
    if "positional_encoding_gaussian_matrix" in name:
        return torch.randn(shape, generator=gen)
    if any(k in name for k in ("point_embeddings", "not_a_point_embed", "no_mask_embed", "iou_token", "mask_tokens",
                               "hf_token")):
        return torch.randn(shape, generator=gen)
    if len(shape) == 1:
        is_norm = any(k in name for k in ("norm", "neck.1.", "neck.3.", "mask_downscaling.1.", "mask_downscaling.4.",
                                          "output_upscaling.1.", "compress_vit_feat.1.", "embedding_encoder.1.",
                                          "embedding_maskfeature.1."))
        if is_norm:
            return torch.ones(shape) if leaf == "weight" else torch.zeros(shape)
        # bias of a linear/conv: bound 1/sqrt(fan_in) is not recoverable from a 1-D shape; use a small uniform
        return (torch.rand(shape, generator=gen) * 2 - 1) * 0.05
    fan_in = 1
    for d in shape[1:]:
        fan_in *= d
    if "output_upscaling.0.weight" in name or "output_upscaling.3.weight" in name or ".compress_vit_feat." in name \
            or ".embedding_encoder." in name:
        fan_in = shape[0]  # ConvTranspose2d: (in, out, kh, kw)
    bound = 1.0 / math.sqrt(fan_in)
    return (torch.rand(shape, generator=gen) * 2 - 1) * bound


def make_state_dict(shapes: Dict[str, Tuple[int, ...]], seed: int) -> Dict[str, torch.Tensor]:
    gen = torch.Generator().manual_seed(seed)
    return {k: _init_like_torch(k, tuple(shapes[k]), gen).float().contiguous() for k in sorted(shapes)}


def make_tinyvit_state_dict(seed: int, num_classes: int = 1000) -> Dict[str, torch.Tensor]:
    """TinyViT-5M state dict under upstream key names (mobile_sam/modeling/tiny_vit_sam.py), BatchNorm buffers included.
    Convs / linears as `_init_like_torch`; BatchNorm: weight U(0.5, 1.5), bias and running_mean U(-0.1, 0.1), running_var
    U(0.5, 2) (positive, so the folded scale stays O(1)), num_batches_tracked 0; attention_biases N(0, 1) (O(1) relative-position
    structure, where torch's zero init would hide the bias indexing)."""
    from mobile_sam.modeling.tiny_vit_sam import state_dict_shapes
    gen = torch.Generator().manual_seed(seed)
    out: Dict[str, torch.Tensor] = {}
    for k, shp in sorted(state_dict_shapes(num_classes).items()):
        leaf = k.rsplit(".", 1)[-1]
        if leaf == "num_batches_tracked":
            out[k] = torch.tensor(0, dtype=torch.long)
        elif ".bn." in k and leaf == "weight":
            out[k] = 0.5 + torch.rand(shp, generator=gen)
        elif ".bn." in k and leaf in ("bias", "running_mean"):
            out[k] = (torch.rand(shp, generator=gen) * 2 - 1) * 0.1
        elif leaf == "running_var":
            out[k] = 0.5 + 1.5 * torch.rand(shp, generator=gen)
        elif leaf == "attention_biases":
            out[k] = torch.randn(shp, generator=gen)
        elif ".norm." in k:   # a non-zero LayerNorm bias makes the padded window tokens (LN(0) = bias) matter
            out[k] = (1.0 if leaf == "weight" else 0.0) + (torch.rand(shp, generator=gen) * 2 - 1) * 0.3
        else:
            out[k] = _init_like_torch(k, shp, gen).float().contiguous()
    return out


def condition_pips(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """x0.1 on the delta head makes random-weight PIPS contractive (SURVEY §0.4)."""
    sd = dict(sd)
    sd["delta_block.to_delta.15.weight"] = sd["delta_block.to_delta.15.weight"] * 0.1
    sd["delta_block.to_delta.15.bias"] = sd["delta_block.to_delta.15.bias"] * 0.1
    return sd


def make_pips_plus_plus_state_dict(seed: int = 8201) -> Dict[str, torch.Tensor]:
    from sam_pt.point_tracker.pips_plus_plus.pips_plus_plus import state_dict_shapes
    return condition_pips_plus_plus(make_state_dict(state_dict_shapes(), seed))


def condition_pips_plus_plus(sd: Dict[str, torch.Tensor], scale: float = 0.03) -> Dict[str, torch.Tensor]:
    """Untrained, the DeltaBlock moves points by ~6 px per iteration and the 16-iteration chain wanders off (73 px after 16
    iterations at 128x160; float32 and float64 runs of it end 14 px apart).  x0.03 on `delta_block.dense`, as x0.1 on PIPS's
    delta head, makes it contractive: 2.5 px of motion after 16 iterations, float32 vs float64 5.6e-5 px (x0.1 still leaves
    4.1e-4 px)."""
    sd = dict(sd)
    sd["delta_block.dense.weight"] = sd["delta_block.dense.weight"] * scale
    sd["delta_block.dense.bias"] = sd["delta_block.dense.bias"] * scale
    return sd


def condition_sam(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """Make random-weight SAM produce non-degenerate, well-separated mask logits: give the mask-0 hyper-network
    a strong constant component so `logit = hyper . upscaled` has O(1) structure instead of ~0 noise (SURVEY §8d)."""
    sd = dict(sd)
    k = "mask_decoder.output_hypernetworks_mlps.0.layers.2.bias"
    if k in sd:
        g = torch.Generator().manual_seed(1234)
        sd[k] = torch.randn(sd[k].shape, generator=g) * 2.0
    return sd


def write_pips_checkpoint_dir(sd: Dict[str, torch.Tensor], path: str, step: int = 1) -> str:
    """Layout saverloader.load expects (reference sam_pt/point_tracker/utils/saverloader.py:30-73)."""
    os.makedirs(path, exist_ok=True)
    torch.save({"model_state_dict": sd}, os.path.join(path, "model-%09d.pth" % step))
    return path


def condition_cotracker(sd: Dict[str, torch.Tensor], vis_bias: float = -0.9, coord_scale: float = 0.003) -> Dict[str, torch.Tensor]:
    """Random-weight CoTracker is chaotic: the flow embedding carries frequencies up to ~970 rad per feature pixel, so with an
    untrained O(1) coordinate head any 1e-6 perturbation saturates at ~0.6 px after 18 iterations (measured on the oracle
    itself).  Scaling the two coordinate rows of the UpdateFormer's flow head by 0.003 (and the feature rows by 0.1) makes the
    iteration contractive like the trained checkpoint (1e-5 relative feature noise -> 2e-5 px), which is what a parity test needs.
    A visibility bias spreads sigmoid(vis) around the reference's 0.7 threshold (configs/model/point_tracker/cotracker.yaml:7):
    the random-weight visibility logits sit at -0.2 +- 0.5 (measured on the C3 clip), so `vis_bias=-0.9` (unit tests: exercises the
    invisible / fill-in paths) leaves almost every point invisible, while `vis_bias=+0.6` (the full-clip C3 / C5 configurations)
    puts ~90 % of the points above the threshold, with a tail of occluded ones, so that the mask decoder actually runs.
    `coord_scale` (coordinate rows of the flow head): 0.003 is contractive enough for the <= 12-frame unit tests; over the 12
    chained windows of a 50-frame clip it is NOT -- the CPU oracle run with 8 vs 3 BLAS threads (summation order only) drifts
    1.8e-3 px from ITSELF on the C3 clip, i.e. the 1e-3 px bar is below that fixture's own reproducibility -- so the full-clip
    configurations use 0.001 (oracle self-drift 9e-5 px; tests/golden/make_golden_full.py records both numbers)."""
    sd = dict(sd)
    w, b = sd["updateformer.flow_head.weight"].clone(), sd["updateformer.flow_head.bias"].clone()
    w[:2] *= coord_scale
    b[:2] *= coord_scale
    w[2:] *= 0.1
    b[2:] *= 0.1
    sd["updateformer.flow_head.weight"], sd["updateformer.flow_head.bias"] = w, b
    sd["vis_predictor.0.bias"] = sd["vis_predictor.0.bias"] + vis_bias
    return sd
