"""Programmatic construction of the SAM-PT object tree, with the same dotted classes and kwargs that
`hydra.utils.instantiate(cfg.model)` resolves from the reference's YAML (configs/model/sam_pt.yaml and the
configs/model/sam/**, configs/model/point_tracker/pips.yaml groups).  Used by tests, smoke() and bench.py, where Hydra
is not installed."""
from __future__ import annotations

from functools import partial
from typing import Dict, Optional

import torch

VIT_CFGS = {
    # configs/model/sam/image_encoder/vit_{base,large,huge}.yaml
    "vit_b": dict(depth=12, embed_dim=768, num_heads=12, global_attn_indexes=[2, 5, 8, 11]),
    "vit_l": dict(depth=24, embed_dim=1024, num_heads=16, global_attn_indexes=[5, 11, 17, 23]),
    "vit_h": dict(depth=32, embed_dim=1280, num_heads=16, global_attn_indexes=[7, 15, 23, 31]),
    # small structural twins for fast tests: hd 64 / hd 80, windowed + global blocks
    "vit_test": dict(depth=4, embed_dim=128, num_heads=2, global_attn_indexes=[1, 3]),
    "vit_test80": dict(depth=2, embed_dim=640, num_heads=8, global_attn_indexes=[1]),
}
# configs/model/sam/sam_mobile_vit_tiny.yaml / samhq_light_vit_tiny.yaml: TinyViT-5M (MobileSAM; Light HQ-SAM with vit_dim 160)
TINY_VIT = "vit_t"
TINY_VIT_CFG = dict(img_size=1024, in_chans=3, num_classes=1000, embed_dims=[64, 128, 160, 320], depths=[2, 2, 6, 2],
                    num_heads=[2, 4, 5, 10], window_sizes=[7, 7, 14, 7], mlp_ratio=4.0, drop_rate=0.0, drop_path_rate=0.0,
                    use_checkpoint=False, mbconv_expand_ratio=4.0, local_conv_size=3, layer_lr_decay=0.8)


def build_sam(vit: str = "vit_b", sam_state_dict: Optional[Dict[str, torch.Tensor]] = None, hq: bool = False):
    """vit: a VIT_CFGS key, or TINY_VIT for MobileSAM (hq=False) / Light HQ-SAM (hq=True)."""
    if vit == TINY_VIT:
        return _build_tiny_sam(sam_state_dict, hq)
    from sam_pt.modeling.sam import SamHydra
    from segment_anything.modeling.image_encoder import ImageEncoderViT
    from segment_anything.modeling.mask_decoder import MaskDecoder
    from segment_anything.modeling.prompt_encoder import PromptEncoder
    from segment_anything.modeling.transformer import TwoWayTransformer

    c = VIT_CFGS[vit]
    if hq:
        from sam_pt.modeling.sam import SamHQHydra
        from segment_anything_hq.modeling.image_encoder import ImageEncoderViT
        from segment_anything_hq.modeling.mask_decoder_hq import MaskDecoderHQ
    enc = ImageEncoderViT(depth=c["depth"], embed_dim=c["embed_dim"], img_size=1024, mlp_ratio=4,
                          norm_layer=partial(torch.nn.LayerNorm, eps=1e-6), num_heads=c["num_heads"], patch_size=16,
                          qkv_bias=True, use_rel_pos=True, global_attn_indexes=c["global_attn_indexes"], window_size=14,
                          out_chans=256)
    pe = PromptEncoder(embed_dim=256, image_embedding_size=(64, 64), input_image_size=(1024, 1024), mask_in_chans=16)
    tw = TwoWayTransformer(depth=2, embedding_dim=256, mlp_dim=2048, num_heads=8)
    if hq:
        md = MaskDecoderHQ(num_multimask_outputs=3, transformer=tw, transformer_dim=256, iou_head_depth=3, iou_head_hidden_dim=256,
                           vit_dim=c["embed_dim"])
    else:
        md = MaskDecoder(num_multimask_outputs=3, transformer=tw, transformer_dim=256, iou_head_depth=3, iou_head_hidden_dim=256)
    sam = (SamHQHydra if hq else SamHydra)(image_encoder=enc, prompt_encoder=pe, mask_decoder=md, pixel_mean=[123.675, 116.28, 103.53],
                   pixel_std=[58.395, 57.12, 57.375], checkpoint=None, prompt_embed_dim=256, image_size=1024, vit_patch_size=16,
                   image_embedding_size=64)
    if sam_state_dict is not None:
        missing, unexpected = sam.load_state_dict(sam_state_dict, strict=False)
        assert not unexpected, unexpected
        assert not missing, missing
    return sam


def _build_tiny_sam(sam_state_dict, hq: bool):
    from segment_anything.modeling.prompt_encoder import PromptEncoder
    from segment_anything.modeling.transformer import TwoWayTransformer
    pe = PromptEncoder(embed_dim=256, image_embedding_size=(64, 64), input_image_size=(1024, 1024), mask_in_chans=16)
    tw = TwoWayTransformer(depth=2, embedding_dim=256, mlp_dim=2048, num_heads=8)
    if hq:
        from sam_pt.modeling.sam import SamHQHydra as Hydra
        from segment_anything_hq.modeling.mask_decoder_hq import MaskDecoderHQ
        from segment_anything_hq.modeling.tiny_vit_sam import TinyViT
        md = MaskDecoderHQ(num_multimask_outputs=3, transformer=tw, transformer_dim=256, iou_head_depth=3, iou_head_hidden_dim=256,
                           vit_dim=160)
    else:
        from mobile_sam.modeling.mask_decoder import MaskDecoder
        from mobile_sam.modeling.tiny_vit_sam import TinyViT
        from sam_pt.modeling.sam import MobileSamHydra as Hydra
        md = MaskDecoder(num_multimask_outputs=3, transformer=tw, transformer_dim=256, iou_head_depth=3, iou_head_hidden_dim=256)
    sam = Hydra(image_encoder=TinyViT(**TINY_VIT_CFG), prompt_encoder=pe, mask_decoder=md, pixel_mean=[123.675, 116.28, 103.53],
                pixel_std=[58.395, 57.12, 57.375], checkpoint=None, prompt_embed_dim=256, image_size=1024, vit_patch_size=16,
                image_embedding_size=64)
    if sam_state_dict is not None:
        missing, unexpected = sam.load_state_dict(sam_state_dict, strict=False)
        assert not unexpected, unexpected
        assert not missing, missing
    return sam


def build_sam_pt(vit: str, sam_state_dict, pips_ckpt_dir: str, positive_points_per_mask: int, negative_points_per_mask: int = 0,
                 iterative_refinement_iterations: int = 12, sam_iou_threshold: float = 0.7, device="cuda", hq: bool = False,
                 cotracker_state_dict=None, cotracker_interp_shape=(384, 512), pips_plus_plus_state_dict=None):
    """configs/model/sam_pt.yaml with `model/point_tracker=pips`, `model/sam@...=sam_vit_*` and the demo-style overrides
    positive_points_per_mask=P negative_points_per_mask=0 (demo/demo.py:107-110)."""
    from sam_pt.modeling.sam_pt import SamPt
    from sam_pt.point_tracker.pips import PipsPointTracker
    if hq:
        from segment_anything_hq.predictor import SamPredictor
    else:
        from segment_anything.predictor import SamPredictor

    sam = build_sam(vit, sam_state_dict, hq=hq)
    if pips_plus_plus_state_dict is not None:
        # configs/model/point_tracker/pips_plus_plus.yaml
        from sam_pt.point_tracker.pips_plus_plus import PipsPlusPlusPointTracker
        tracker = PipsPlusPlusPointTracker(checkpoint_path=None, stride=8, max_sequence_length=128, iters=16, image_size=None)
        tracker.model.load_state_dict(pips_plus_plus_state_dict)
    elif cotracker_state_dict is not None:
        # configs/model/point_tracker/cotracker.yaml (the reference's default tracker group)
        from sam_pt.point_tracker.cotracker import CoTrackerPointTracker
        tracker = CoTrackerPointTracker(checkpoint_path=None, interp_shape=list(cotracker_interp_shape), visibility_threshold=0.7, support_grid_size=2,
                                        support_grid_every_n_frames=12, add_debug_visualisations=False)
        tracker.model.load_state_dict(cotracker_state_dict)
    else:
        tracker = PipsPointTracker(checkpoint_path=pips_ckpt_dir, stride=4, s=8, initial_next_frame_visibility_threshold=0.9)
    model = SamPt(point_tracker=tracker, sam_predictor=SamPredictor(sam_model=sam), sam_iou_threshold=sam_iou_threshold,
                  positive_point_selection_method="kmedoids", negative_point_selection_method="mixed",
                  positive_points_per_mask=positive_points_per_mask, negative_points_per_mask=negative_points_per_mask,
                  add_other_objects_positive_points_as_negative_points=True, max_other_objects_positive_points=None,
                  point_tracker_mask_batch_size=5, iterative_refinement_iterations=iterative_refinement_iterations,
                  use_patch_matching_filtering=False, patch_size=3, patch_similarity_threshold=0.01, use_point_reinit=False,
                  reinit_point_tracker_horizon=24, reinit_horizon=24, reinit_variant="reinit-at-median-of-area-diff")
    return model.to(device).eval()
