"""GPU parity of the SAM path (resize, ViT encoder at the three precision settings, prompt+mask decoder, fused refinement
chain, and the C1 end-to-end SamPt run) against the CPU oracle.  Tolerances are stated per test."""
import numpy as np
import pytest
import torch

from oracle import pips_ref, sam_ref, sampt_ref
from sampt_b200 import factory, synth

pytestmark = pytest.mark.gpu


def _iou(a, b):
    a, b = a > 0, b > 0
    u = (a | b).sum().item()
    return (a & b).sum().item() / u if u else 1.0


def _sam_sd(cfg, seed):
    return synth.condition_sam(synth.make_state_dict(sam_ref.sam_state_dict_shapes(cfg), seed))


ORACLE_CFG = {"vit_test": sam_ref.VIT_TEST, "vit_b": sam_ref.VIT_B,
              "vit_test80": sam_ref.VitCfg(depth=2, embed_dim=640, num_heads=8, global_attn_indexes=(1,))}


def test_pil_resize_gpu_bit_exact():
    from PIL import Image
    from segment_anything.predictor import SamPredictor
    sam = factory.build_sam("vit_test").cuda()
    pred = SamPredictor(sam)
    rng = np.random.default_rng(0)
    for (h, w) in [(240, 320), (480, 854), (1080, 1920)]:
        img = rng.integers(0, 256, size=(2, h, w, 3), dtype=np.uint8)
        out = pred.resize_frames_u8(torch.from_numpy(img).permute(0, 3, 1, 2).contiguous().cuda())
        nh, nw = pred.transform.get_preprocess_shape(h, w, 1024)
        for b in range(2):
            ref = np.array(Image.fromarray(img[b]).resize((nw, nh), resample=Image.BILINEAR))
            assert np.array_equal(out[b].permute(1, 2, 0).cpu().numpy(), ref), (h, w)


@pytest.mark.parametrize("vit,precision,tol", [("vit_test", 1, 6e-3), ("vit_test", 2, 4e-3), ("vit_test", 3, 6e-4),
                                               ("vit_test", 4, 2e-4), ("vit_test80", 1, 6e-3), ("vit_test80", 3, 6e-4),
                                               ("vit_test80", 4, 2e-4), ("vit_test", 6, 2e-4), ("vit_test80", 6, 2e-4)])
def test_vit_encoder_matches_oracle(vit, precision, tol):
    """relative L2 error of the (B,256,64,64) embedding; batch of 2 frames exercises the frame batching."""
    from segment_anything.predictor import SamPredictor
    cfg = ORACLE_CFG[vit]
    sd = _sam_sd(cfg, 31)
    sam = factory.build_sam(vit, sd).cuda()
    sam.image_encoder.precision = precision
    pred = SamPredictor(sam)
    clip = synth.make_clip(2, 240, 320, seed=3)
    feats = pred.encode_frames(clip["frames"].cuda()).cpu()
    for b in range(2):
        x, _ = sam_ref.preprocess(clip["frames"][b].permute(1, 2, 0).numpy())
        ref = sam_ref.vit_encode(sd, x, cfg)[0]
        rel = ((feats[b] - ref).norm() / ref.norm()).item()
        assert rel < tol, (vit, precision, b, rel)


@pytest.mark.parametrize("precision", [4, 6])
def test_vit_b_precision3_embedding(precision):
    """ViT-B (every block GEMM on the tensor-core kernel): three fp16 passes (4) and fp16 + two e4m3 correction passes (6)."""
    from segment_anything.predictor import SamPredictor
    cfg = sam_ref.VIT_B
    sd = _sam_sd(cfg, 7202)
    sam = factory.build_sam("vit_b", sd).cuda()
    sam.image_encoder.precision = precision
    pred = SamPredictor(sam)
    clip = synth.make_clip(1, 240, 320, seed=72)
    feats = pred.encode_frames(clip["frames"].cuda()).cpu()
    x, _ = sam_ref.preprocess(clip["frames"][0].permute(1, 2, 0).numpy())
    ref = sam_ref.vit_encode(sd, x, cfg)[0]
    assert ((feats[0] - ref).norm() / ref.norm()).item() < 3e-4


@pytest.fixture(scope="module")
def decoder_setup():
    from segment_anything.predictor import SamPredictor
    cfg = sam_ref.VIT_TEST
    sd = _sam_sd(cfg, 41)
    sam = factory.build_sam("vit_test", sd).cuda()
    pred = SamPredictor(sam)
    g = torch.Generator().manual_seed(9)
    feats = torch.randn((1, 256, 64, 64), generator=g)
    ref = sam_ref.RefSamPredictor(sd, cfg)
    ref.features = feats
    ref.original_size, ref.input_size = (480, 854), (576, 1024)
    pred.set_frames_features((480, 854), feats.cuda())
    return sd, pred, ref, g


@pytest.mark.parametrize("with_mask,with_box,multimask", [(False, False, False), (True, False, False), (True, True, False),
                                                          (False, False, True)])
def test_predict_torch_matches_oracle(decoder_setup, with_mask, with_box, multimask):
    sd, pred, ref, g = decoder_setup
    pts = torch.rand((1, 6, 2), generator=g) * torch.tensor([1000.0, 560.0])
    labels = torch.tensor([[1, 1, 0, 1, 1, 1]], dtype=torch.int)
    mask_in = torch.randn((1, 1, 256, 256), generator=g) if with_mask else None
    box = torch.tensor([[[100.0, 150.0, 700.0, 440.0]]]) if with_box else None
    rm, ri, rl = ref.predict_torch(pts, labels, box[:, 0] if with_box else None, mask_in, multimask, True)
    cu = lambda t: t.cuda() if t is not None else None
    m, i, l = pred.predict_torch(cu(pts), cu(labels), cu(box), cu(mask_in), multimask, True)
    scale = max(1.0, rl.abs().max().item())
    assert (l.cpu() - rl).abs().max() < 2e-4 * scale
    assert (m.cpu() - rm).abs().max() < 2e-4 * scale
    assert (i.cpu() - ri).abs().max() < 1e-4


def test_predict_refine_chain_matches_oracle(decoder_setup):
    """the fused 1 + 12-iteration refinement chain vs the oracle's host loop (sam_pt.py:781-828 semantics)."""
    sd, pred, ref, g = decoder_setup
    pts = torch.rand((1, 8, 2), generator=g) * torch.tensor([1000.0, 560.0])
    labels = torch.ones((1, 8), dtype=torch.int)
    ml, iou, low = ref.predict_torch(pts, labels, None, None, False, True)
    n = 0
    for _ in range(12):
        mm = ml[0, 0] > 0
        if mm.sum() < 2:
            break
        yx = mm.nonzero()
        box = torch.tensor([yx[:, 1].min(), yx[:, 0].min(), yx[:, 1].max(), yx[:, 0].max()], dtype=torch.float)
        ml, iou, low = ref.predict_torch(pts, labels, box[None, None, :][:, 0], low, False, True)
        n += 1
    out = torch.empty((480, 854), device="cuda")
    g_iou, g_low, g_n = pred.predict_refine(pts[0].cuda(), labels[0].cuda(), 0, 12, out)
    assert int(g_n.item()) == n
    assert _iou(out.cpu(), ml[0, 0]) >= 0.999
    assert (g_iou.cpu() - iou[0]).abs().max() < 1e-3
    assert (g_low.cpu() - low[0, 0]).abs().max() < 5e-3 * max(1.0, low.abs().max().item())


@pytest.mark.parametrize("n_pos", [3, 0])
def test_predict_refine_two_call_form_matches_oracle(decoder_setup, n_pos):
    """negative_points_per_mask > 0 (sam_pt.py:792-807): first call on the positive points only, its low-res mask feeds the second
    call with all points; n_pos = 0 is the corner where every positive point is occluded and only negatives are visible."""
    sd, pred, ref, g = decoder_setup
    K = 6
    pts = torch.rand((1, K, 2), generator=g) * torch.tensor([1000.0, 560.0])
    labels = torch.zeros((1, K), dtype=torch.int)
    labels[0, :n_pos] = 1
    sel = labels[0] == 1
    _, _, low = ref.predict_torch(pts[:, sel], labels[:, sel], None, None, False, True)
    ml, iou, low = ref.predict_torch(pts, labels, None, low, False, True)
    n = 0
    for _ in range(12):
        mm = ml[0, 0] > 0
        if mm.sum() < 2:
            break
        yx = mm.nonzero()
        box = torch.tensor([yx[:, 1].min(), yx[:, 0].min(), yx[:, 1].max(), yx[:, 0].max()], dtype=torch.float)
        ml, iou, low = ref.predict_torch(pts, labels, box[None, None, :][:, 0], low, False, True)
        n += 1
    out = torch.empty((480, 854), device="cuda")
    g_iou, g_low, g_n = pred.predict_refine(pts[0].cuda(), labels[0].cuda(), 1, 12, out, positive_index=list(range(n_pos)))
    assert int(g_n.item()) == n
    assert _iou(out.cpu(), ml[0, 0]) >= 0.999
    assert (g_iou.cpu() - iou[0]).abs().max() < 1e-3
    assert (g_low.cpu() - low[0, 0]).abs().max() < 5e-3 * max(1.0, low.abs().max().item())


def test_sampt_c1_end_to_end(tmp_path):
    """BASELINE config C1: 2 x 240x320, ViT-B + PIPS, 4 points.  coords within 1e-3 px, per-frame IoU >= 0.999."""
    cfg = sam_ref.VIT_B
    sam_sd = _sam_sd(cfg, 7202)
    pips_sd = synth.condition_pips(synth.make_state_dict(pips_ref.pips_state_dict_shapes(), 7201))
    ckpt = synth.write_pips_checkpoint_dir(pips_sd, str(tmp_path / "pips"))
    video = synth.make_video_dict(2, 240, 320, 4)
    ref = sampt_ref.sampt_forward(pips_sd, sam_ref.RefSamPredictor(sam_sd, cfg), video, positive_points_per_mask=4,
                                  sam_iou_threshold=-1e9)
    model = factory.build_sam_pt("vit_b", sam_sd, ckpt, positive_points_per_mask=4, sam_iou_threshold=-1e9)
    out = model(video)
    assert (out["trajectories"].cpu() - ref["trajectories"]).abs().max() < 1e-3
    assert torch.equal(out["visibilities"].cpu(), ref["visibilities"])
    for f in range(2):
        iou = _iou(out["logits"][0][f].cpu(), ref["logits"][0][f])
        assert iou >= 0.999, (f, iou)
    assert np.allclose(np.array(out["scores"]), np.array(ref["scores"]), atol=2e-3)
    # reference invariants: background logits are finite where masks exist; output shapes (sam_pt.py:222-226)
    assert out["logits"][0].shape == (2, 240, 320)


def test_precision_dial_report(tmp_path):
    """Records mask IoU vs the oracle for the three ViT precision settings on C1 (documentation for DESIGN.md §5);
    only the parity-validated setting (3) is asserted."""
    import json
    import os
    cfg = sam_ref.VIT_B
    sam_sd = _sam_sd(cfg, 7202)
    pips_sd = synth.condition_pips(synth.make_state_dict(pips_ref.pips_state_dict_shapes(), 7201))
    ckpt = synth.write_pips_checkpoint_dir(pips_sd, str(tmp_path / "pips"))
    video = synth.make_video_dict(2, 240, 320, 4)
    ref = sampt_ref.sampt_forward(pips_sd, sam_ref.RefSamPredictor(sam_sd, cfg), video, positive_points_per_mask=4,
                                  sam_iou_threshold=-1e9)
    model = factory.build_sam_pt("vit_b", sam_sd, ckpt, positive_points_per_mask=4, sam_iou_threshold=-1e9)
    report = {}
    for p in (1, 2, 3, 4, 6):
        model.sam_predictor.model.image_encoder.precision = p
        out = model(video)
        report[p] = [_iou(out["logits"][0][f].cpu(), ref["logits"][0][f]) for f in range(2)]
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    os.makedirs(os.path.join(root, "gpurun_out"), exist_ok=True)
    with open(os.path.join(root, "gpurun_out", "precision_dial_c1.json"), "w") as fh:
        json.dump({"config": "C1 (2x240x320, ViT-B + PIPS, 4 pts), per-frame mask IoU vs CPU oracle", "iou_by_precision": report}, fh)
    assert min(report[3]) >= 0.999


# (the 2-frame C2 slice of round 1 is superseded by tests/test_gpu_full_configs.py: all 50 frames of C2 against the full-clip golden)


def test_image_encoder_forward_float_interface():
    """upstream `ImageEncoderViT.forward(x)`: x = Sam.preprocess output (normalised, zero-padded float image) -> (B,256,64,64)."""
    cfg = ORACLE_CFG["vit_test"]
    sd = _sam_sd(cfg, 31)
    sam = factory.build_sam("vit_test", sd).cuda()
    clip = synth.make_clip(2, 240, 320, seed=3)
    xs = torch.cat([sam_ref.preprocess(clip["frames"][b].permute(1, 2, 0).numpy())[0] for b in range(2)], dim=0)   # (2,3,1024,1024)
    got = sam.image_encoder(xs.cuda()).cpu()
    for b in range(2):
        ref = sam_ref.vit_encode(sd, xs[b:b + 1], cfg)[0]
        rel = ((got[b] - ref).norm() / ref.norm()).item()
        assert rel < 3e-4, rel
    # and it agrees with the fused uint8 path SamPredictor uses
    from segment_anything.predictor import SamPredictor
    feats = SamPredictor(sam).encode_frames(clip["frames"].cuda()).cpu()
    assert ((feats - got).norm() / got.norm()).item() < 1e-4


# ---------------------------------------------------------------------------------------------------------------- HQ-SAM
@pytest.fixture(scope="module")
def hq_setup():
    from segment_anything_hq.predictor import SamPredictor
    cfg = sam_ref.VIT_TEST
    sd = synth.condition_sam(synth.make_state_dict(sam_ref.sam_state_dict_shapes(cfg, hq=True), 43))
    sam = factory.build_sam("vit_test", sd, hq=True).cuda()
    pred = SamPredictor(sam)
    g = torch.Generator().manual_seed(19)
    feats = torch.randn((1, 256, 64, 64), generator=g)
    interm = torch.randn((1, 64, 64, cfg.embed_dim), generator=g)
    ref = sam_ref.RefSamPredictor(sd, cfg, hq=True)
    ref.features, ref.interm = feats, [interm]
    ref.original_size, ref.input_size = (480, 854), (576, 1024)
    pred.set_frames_features((480, 854), (feats.cuda(), interm.cuda()))
    return sd, pred, ref, g


@pytest.mark.parametrize("with_mask,with_box", [(False, False), (True, True)])
def test_hq_predict_torch_matches_oracle(hq_setup, with_mask, with_box):
    """MaskDecoderHQ single-mask output = SAM mask + HQ mask (hq_token_only=False), against the oracle restatement."""
    sd, pred, ref, g = hq_setup
    pts = torch.rand((1, 6, 2), generator=g) * torch.tensor([1000.0, 560.0])
    labels = torch.tensor([[1, 1, 0, 1, 1, 1]], dtype=torch.int)
    mask_in = torch.randn((1, 1, 256, 256), generator=g) if with_mask else None
    box = torch.tensor([[[100.0, 150.0, 700.0, 440.0]]]) if with_box else None
    rm, ri, rl = ref.predict_torch(pts, labels, box[:, 0] if with_box else None, mask_in, False, True)
    cu = lambda t: t.cuda() if t is not None else None
    m, i, l = pred.predict_torch(cu(pts), cu(labels), cu(box), cu(mask_in), False, True)
    scale = max(1.0, rl.abs().max().item())
    assert (l.cpu() - rl).abs().max() < 3e-4 * scale
    assert (m.cpu() - rm).abs().max() < 3e-4 * scale
    assert (i.cpu() - ri).abs().max() < 1e-4


def test_hq_encoder_interm_and_e2e(tmp_path):
    """HQ-SAM + PIPS end to end on a tiny clip (encoder returns the first global block's output; decoder adds the HQ mask)."""
    from segment_anything_hq.predictor import SamPredictor
    cfg = sam_ref.VIT_TEST
    sam_sd = synth.condition_sam(synth.make_state_dict(sam_ref.sam_state_dict_shapes(cfg, hq=True), 47))
    pips_sd = synth.condition_pips(synth.make_state_dict(pips_ref.pips_state_dict_shapes(), 7201))
    ckpt = synth.write_pips_checkpoint_dir(pips_sd, str(tmp_path / "pips"))
    video = synth.make_video_dict(3, 96, 128, 4)
    taps, cache = {}, {}
    ref = sampt_ref.sampt_forward(pips_sd, sam_ref.RefSamPredictor(sam_sd, cfg, hq=True), video, positive_points_per_mask=4,
                                  sam_iou_threshold=-1e9, taps=taps, features_cache=cache)
    # the oracle's own conditioning: the same decode on image features perturbed by 1e-5 relative (fp32 rounding level x 100).  With
    # random weights a few border pixels sit behind a LayerNorm2d with almost no variance and move by 1e-2 (4000x the median pixel)
    g = torch.Generator().manual_seed(1)

    def pert(t):
        if t is None:
            return None
        if isinstance(t, (list, tuple)):
            return [pert(x) for x in t]
        return t * (1 + 1e-5 * torch.randn(t.shape, generator=g))
    cache2 = {f: {"features": pert(v["features"]), "interm": pert(v.get("interm"))} for f, v in cache.items()}
    ref2 = sampt_ref.sampt_forward(pips_sd, sam_ref.RefSamPredictor(sam_sd, cfg, hq=True), video, positive_points_per_mask=4,
                                   sam_iou_threshold=-1e9, features_cache=cache2)
    model = factory.build_sam_pt("vit_test", sam_sd, ckpt, positive_points_per_mask=4, sam_iou_threshold=-1e9, hq=True)
    out = model(video)
    assert (out["trajectories"].cpu() - ref["trajectories"]).abs().max() < 1e-3
    assert torch.equal(out["visibilities"].cpu(), ref["visibilities"])
    for f in range(3):
        a, b = out["logits"][0][f].cpu(), ref["logits"][0][f]
        sens = (ref2["logits"][0][f] - b).abs()
        ill = sens > 20 * sens.median()                        # pixels where the ORACLE amplifies rounding noise > 20x the typical pixel
        # logits agree to 2e-3 of the frame's range (3e-4 per decoder call, 13 calls chained) on 99.9 % of the pixels; the amplification
        # is heavy-tailed (a handful of border pixels move by 1e-2 under the 1e-5 perturbation), so the bound is on a quantile
        tol = 2e-3 * max(1.0, float(b[torch.isfinite(b)].abs().max()))
        q999 = float(torch.quantile((a - b).abs().flatten(), 0.999))
        assert q999 < tol, (f, q999, tol)
        assert int(ill.sum()) <= 0.02 * ill.numel(), (f, int(ill.sum()))
        # masks: IoU >= 0.999, or -- the random-weight HQ branch yields masks of ~400 pixels, where ONE pixel is 0.0025 IoU -- every
        # disagreeing pixel is either undecided in the oracle (|logit| < tol) or ill-conditioned in the oracle itself, at most 2 of them
        diff = (a > 0) != (b > 0)
        nd = int(diff.sum())
        excused = nd <= 2 and bool(((b.abs() < tol) | ill)[diff].all())
        assert _iou(a, b) >= 0.999 or excused, (f, _iou(a, b), nd, int((b > 0).sum()))
