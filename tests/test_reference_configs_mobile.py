"""CPU: the reference's unmodified MobileSAM and Light HQ-SAM YAMLs (sam_mobile_vit_tiny.yaml, samhq_light_vit_tiny.yaml,
stored verbatim under tests/golden/reference_configs/) compose through hydra_lite and instantiate into this tree; an
upstream-keyed checkpoint loads; the HQ predictor refuses a model without an HQ mask decoder."""
import os

import pytest
import torch

REF_CFG = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_configs")


def _pips(tmp_path):
    from oracle import pips_ref
    from sampt_b200 import synth
    sd = synth.condition_pips(synth.make_state_dict(pips_ref.pips_state_dict_shapes(), 1))
    synth.write_pips_checkpoint_dir(sd, str(tmp_path / "models" / "pips_ckpts" / "reference_model"))


def _checkpoint(path, hq: bool):
    """Upstream key names: head.*, BatchNorm buffers and num_batches_tracked included."""
    from sampt_b200 import factory, synth
    sam = factory.build_sam(factory.TINY_VIT, hq=hq)
    sd = {k: v.clone() for k, v in sam.state_dict().items() if k not in ("pixel_mean", "pixel_std")}
    enc = synth.make_tinyvit_state_dict(11)
    for k, v in enc.items():
        sd["image_encoder." + k] = v
    os.makedirs(os.path.dirname(path), exist_ok=True)
    torch.save(sd, path)
    return sd


def test_mobile_sam_yaml_instantiates(tmp_path):
    from sampt_b200 import hydra_lite
    _pips(tmp_path)
    sd = _checkpoint(str(tmp_path / "models" / "sam_mobile_ckpts" / "sam_mobile_vit_t.pth"), hq=False)
    cfg = hydra_lite.compose_model(REF_CFG, {
        "point_tracker": "pips", "sam@sam_predictor.sam_model": "sam_mobile_vit_tiny",
        "sam_predictor._target_": "segment_anything.predictor.SamPredictor",
        "positive_points_per_mask": 8, "negative_points_per_mask": 0,
    }, cwd=str(tmp_path))
    sm = cfg["sam_predictor"]["sam_model"]
    assert sm["_target_"] == "sam_pt.modeling.sam.MobileSamHydra"
    assert sm["image_encoder"]["_target_"] == "mobile_sam.modeling.TinyViT"
    assert sm["image_encoder"]["img_size"] == 1024
    model = hydra_lite.instantiate(cfg)
    import mobile_sam.modeling as mm
    import segment_anything.predictor as sp
    from sam_pt.modeling.sam import MobileSamHydra
    pred = model.sam_predictor
    assert type(pred) is sp.SamPredictor
    assert isinstance(pred.model, MobileSamHydra) and isinstance(pred.model, mm.Sam)
    assert type(pred.model.image_encoder) is mm.TinyViT
    assert pred.model.image_encoder.returns_interm is False
    got = pred.model.state_dict()
    for k in ("image_encoder.head.weight", "image_encoder.layers.0.blocks.0.conv1.bn.running_var",
              "image_encoder.layers.3.blocks.1.attn.attention_biases", "image_encoder.patch_embed.seq.0.bn.num_batches_tracked"):
        assert torch.equal(got[k].cpu(), sd[k]), k
    missing, unexpected = pred.model.load_state_dict(sd, strict=False)
    assert not missing and not unexpected


def test_light_hq_sam_yaml_instantiates(tmp_path):
    from sampt_b200 import hydra_lite
    _pips(tmp_path)
    sd = _checkpoint(str(tmp_path / "models" / "samhq_ckpts" / "sam_hq_vit_t.pth"), hq=True)
    cfg = hydra_lite.compose_model(REF_CFG, {"point_tracker": "pips", "sam@sam_predictor.sam_model": "samhq_light_vit_tiny"},
                                   cwd=str(tmp_path))
    assert cfg["sam_predictor"]["_target_"] == "segment_anything_hq.predictor.SamPredictor"
    sm = cfg["sam_predictor"]["sam_model"]
    assert sm["image_encoder"]["_target_"] == "segment_anything_hq.modeling.TinyViT"
    assert sm["mask_decoder"]["vit_dim"] == 160
    model = hydra_lite.instantiate(cfg)
    import segment_anything_hq.modeling as hm
    import segment_anything_hq.predictor as hp
    pred = model.sam_predictor
    assert type(pred) is hp.SamPredictor
    assert type(pred.model.image_encoder) is hm.TinyViT and pred.model.image_encoder.returns_interm
    assert pred.model.state_dict()["mask_decoder.compress_vit_feat.0.weight"].shape[0] == 160
    missing, unexpected = pred.model.load_state_dict(sd, strict=False)
    assert not missing and not unexpected


def test_hq_predictor_refuses_mobile_sam(tmp_path):
    """The reference's MobileSAM command keeps sam_pt.yaml's default HQ predictor; that combination is refused at
    construction with the override to use."""
    from sampt_b200 import hydra_lite
    _pips(tmp_path)
    cfg = hydra_lite.compose_model(REF_CFG, {"point_tracker": "pips", "sam@sam_predictor.sam_model": "sam_mobile_vit_tiny",
                                             "sam_predictor.sam_model.checkpoint": None}, cwd=str(tmp_path))
    assert cfg["sam_predictor"]["_target_"] == "segment_anything_hq.predictor.SamPredictor"
    with pytest.raises(ValueError, match=r"model\.sam_predictor\._target_=segment_anything\.predictor\.SamPredictor"):
        hydra_lite.instantiate(cfg)
