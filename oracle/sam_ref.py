"""ORACLE (test infrastructure, NOT product code): CPU restatement of SAM.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline /
``--impl reference`` leg may import this module.  The product path
(``sam-pt_b200/``) never does.

What is restated
----------------
The reference (SysCV/sam-pt) calls SAM through the un-vendored third-party
package ``segment-anything @ aac76a1`` (``/root/reference/requirements.txt:28``).
Its source is NOT in /root/reference, so this file restates the published
algorithm (SURVEY.md Appendix B.1/B.2/B.4) as pure functions over a flat
state-dict with the upstream key names.  Call sites in the reference that this
anchors to:

* ``sam_pt/modeling/sam_pt.py:771``      transform.apply_coords
* ``sam_pt/modeling/sam_pt.py:783-828``  SamPredictor.predict_torch
* ``sam_pt/modeling/sam_pt.py:849``      SamPredictor.set_image
* ``sam_pt/modeling/sam.py:18-31``       state-dict contract (strict=False)
* ``configs/model/sam/**.yaml``          constructor arguments

PARITY STATUS: "parity unpinned" against the pinned upstream package (absent, no
network, no golden vectors in the reference).  It IS pinned against the
independent implementation that exists in this image
(``transformers.models.sam``) by ``tests/test_oracle_sam_vs_hf.py`` via a key
remap — see that test.

Everything is torch on CPU, written for clarity not speed: float32 as upstream, and the prompt encoder, mask decoder and
``postprocess_masks`` follow the dtype of the state dict and inputs (float64 for the decoder's kernel tests).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

SD = Dict[str, torch.Tensor]


@dataclass
class VitCfg:
    depth: int = 12
    embed_dim: int = 768
    num_heads: int = 12
    global_attn_indexes: Tuple[int, ...] = (2, 5, 8, 11)
    window_size: int = 14
    patch_size: int = 16
    img_size: int = 1024
    out_chans: int = 256
    mlp_ratio: int = 4


VIT_B = VitCfg()
VIT_L = VitCfg(depth=24, embed_dim=1024, num_heads=16, global_attn_indexes=(5, 11, 17, 23))
VIT_H = VitCfg(depth=32, embed_dim=1280, num_heads=16, global_attn_indexes=(7, 15, 23, 31))
# small config used by fast unit tests (same structure, 2 windowed + 1 global pattern)
VIT_TEST = VitCfg(depth=4, embed_dim=128, num_heads=2, global_attn_indexes=(1, 3))

PIXEL_MEAN = (123.675, 116.28, 103.53)
PIXEL_STD = (58.395, 57.12, 57.375)


# --------------------------------------------------------------------------- #
# ResizeLongestSide  (upstream segment_anything/utils/transforms.py)
# --------------------------------------------------------------------------- #
def get_preprocess_shape(oldh: int, oldw: int, long_side_length: int = 1024) -> Tuple[int, int]:
    scale = long_side_length * 1.0 / max(oldh, oldw)
    newh, neww = oldh * scale, oldw * scale
    return int(newh + 0.5), int(neww + 0.5)


def apply_image(image_hwc_u8: np.ndarray, long_side: int = 1024) -> np.ndarray:
    """PIL bilinear uint8 resize exactly as upstream: np.array(resize(to_pil_image(img), size))."""
    from PIL import Image

    h, w = image_hwc_u8.shape[:2]
    newh, neww = get_preprocess_shape(h, w, long_side)
    pil = Image.fromarray(image_hwc_u8)
    return np.array(pil.resize((neww, newh), resample=Image.BILINEAR))


def apply_coords(coords: np.ndarray, original_size: Tuple[int, int], long_side: int = 1024) -> np.ndarray:
    old_h, old_w = original_size
    new_h, new_w = get_preprocess_shape(old_h, old_w, long_side)
    coords = np.array(coords, copy=True).astype(float)
    coords[..., 0] = coords[..., 0] * (new_w / old_w)
    coords[..., 1] = coords[..., 1] * (new_h / old_h)
    return coords


# --------------------------------------------------------------------------- #
# Image encoder (Appendix B.1)
# --------------------------------------------------------------------------- #
def _ln(x, w, b, eps):
    return F.layer_norm(x, (x.shape[-1],), w, b, eps)


def _ln2d(x, w, b, eps=1e-6):
    u = x.mean(1, keepdim=True)
    s = (x - u).pow(2).mean(1, keepdim=True)
    x = (x - u) / torch.sqrt(s + eps)
    return w[:, None, None] * x + b[:, None, None]


def window_partition(x, ws):
    B, H, W, C = x.shape
    pad_h = (ws - H % ws) % ws
    pad_w = (ws - W % ws) % ws
    if pad_h > 0 or pad_w > 0:
        x = F.pad(x, (0, 0, 0, pad_w, 0, pad_h))
    Hp, Wp = H + pad_h, W + pad_w
    x = x.view(B, Hp // ws, ws, Wp // ws, ws, C)
    windows = x.permute(0, 1, 3, 2, 4, 5).contiguous().view(-1, ws, ws, C)
    return windows, (Hp, Wp)


def window_unpartition(windows, ws, pad_hw, hw):
    Hp, Wp = pad_hw
    H, W = hw
    B = windows.shape[0] // (Hp * Wp // ws // ws)
    x = windows.view(B, Hp // ws, Wp // ws, ws, ws, -1)
    x = x.permute(0, 1, 3, 2, 4, 5).contiguous().view(B, Hp, Wp, -1)
    if Hp > H or Wp > W:
        x = x[:, :H, :W, :].contiguous()
    return x


def get_rel_pos(q_size, k_size, rel_pos):
    max_rel_dist = int(2 * max(q_size, k_size) - 1)
    if rel_pos.shape[0] != max_rel_dist:
        rp = F.interpolate(rel_pos.reshape(1, rel_pos.shape[0], -1).permute(0, 2, 1), size=max_rel_dist, mode="linear")
        rp = rp.reshape(-1, max_rel_dist).permute(1, 0)
    else:
        rp = rel_pos
    q_coords = torch.arange(q_size)[:, None] * max(k_size / q_size, 1.0)
    k_coords = torch.arange(k_size)[None, :] * max(q_size / k_size, 1.0)
    rel = (q_coords - k_coords) + (k_size - 1) * max(q_size / k_size, 1.0)
    return rp[rel.long()]


def vit_attention_core(qkv, rel_pos_h, rel_pos_w, H: int, W: int, num_heads: int):
    """Attention between the qkv and proj linears: qkv (B, H*W, 3D) -> per-head outputs (B, H*W, D), head h at columns
    h*hd.  Computes in the dtype of its inputs (float64 for kernel tests)."""
    B, L, D3 = qkv.shape
    hd = D3 // 3 // num_heads
    scale = hd ** -0.5
    qkv = qkv.reshape(B, L, 3, num_heads, -1).permute(2, 0, 3, 1, 4)
    q, k, v = qkv.reshape(3, B * num_heads, L, -1).unbind(0)
    attn = (q * scale) @ k.transpose(-2, -1)
    Rh = get_rel_pos(H, H, rel_pos_h)
    Rw = get_rel_pos(W, W, rel_pos_w)
    r_q = q.reshape(B * num_heads, H, W, hd)
    rel_h = torch.einsum("bhwc,hkc->bhwk", r_q, Rh)
    rel_w = torch.einsum("bhwc,wkc->bhwk", r_q, Rw)
    attn = (attn.view(-1, H, W, H, W) + rel_h[:, :, :, :, None] + rel_w[:, :, :, None, :]).view(-1, H * W, H * W)
    attn = attn.softmax(dim=-1)
    return (attn @ v).view(B, num_heads, L, -1).permute(0, 2, 1, 3).reshape(B, L, -1)


def vit_attention(sd: SD, p: str, x, num_heads: int):
    B, H, W, D = x.shape
    qkv = F.linear(x, sd[p + "qkv.weight"], sd[p + "qkv.bias"]).reshape(B, H * W, -1)
    x = vit_attention_core(qkv, sd[p + "rel_pos_h"], sd[p + "rel_pos_w"], H, W, num_heads).reshape(B, H, W, -1)
    return F.linear(x, sd[p + "proj.weight"], sd[p + "proj.bias"])


def vit_block(sd: SD, p: str, x, cfg: VitCfg, window_size: int):
    shortcut = x
    x = _ln(x, sd[p + "norm1.weight"], sd[p + "norm1.bias"], 1e-6)
    if window_size > 0:
        H, W = x.shape[1], x.shape[2]
        x, pad_hw = window_partition(x, window_size)
    x = vit_attention(sd, p + "attn.", x, cfg.num_heads)
    if window_size > 0:
        x = window_unpartition(x, window_size, pad_hw, (H, W))
    x = shortcut + x
    y = _ln(x, sd[p + "norm2.weight"], sd[p + "norm2.bias"], 1e-6)
    y = F.linear(y, sd[p + "mlp.lin1.weight"], sd[p + "mlp.lin1.bias"])
    y = F.gelu(y)
    y = F.linear(y, sd[p + "mlp.lin2.weight"], sd[p + "mlp.lin2.bias"])
    return x + y


def vit_encode(sd: SD, x, cfg: VitCfg, prefix="image_encoder.", return_interm=False, taps: Optional[dict] = None):
    """x: (B,3,1024,1024) preprocessed float32 -> (B,256,64,64) [+ list of global-block outputs (HQ-SAM)]."""
    p = prefix
    x = F.conv2d(x, sd[p + "patch_embed.proj.weight"], sd[p + "patch_embed.proj.bias"], stride=cfg.patch_size)
    x = x.permute(0, 2, 3, 1)
    x = x + sd[p + "pos_embed"]
    if taps is not None:
        taps["embed"] = x.clone()
    interm = []
    for i in range(cfg.depth):
        ws = 0 if i in cfg.global_attn_indexes else cfg.window_size
        x = vit_block(sd, f"{p}blocks.{i}.", x, cfg, ws)
        if ws == 0:
            interm.append(x)
        if taps is not None:
            taps[f"block{i}"] = x.clone()
    x = x.permute(0, 3, 1, 2)
    x = F.conv2d(x, sd[p + "neck.0.weight"])
    x = _ln2d(x, sd[p + "neck.1.weight"], sd[p + "neck.1.bias"])
    x = F.conv2d(x, sd[p + "neck.2.weight"], padding=1)
    x = _ln2d(x, sd[p + "neck.3.weight"], sd[p + "neck.3.bias"])
    if return_interm:
        return x, interm
    return x


def preprocess(image_u8_hwc: np.ndarray, img_size=1024, long_side=1024):
    """SamPredictor.set_image front half: PIL resize -> normalise -> zero pad. Returns (x, input_size)."""
    resized = apply_image(image_u8_hwc, long_side)
    x = torch.as_tensor(resized).permute(2, 0, 1).contiguous()[None].float()
    mean = torch.tensor(PIXEL_MEAN).view(1, 3, 1, 1)
    std = torch.tensor(PIXEL_STD).view(1, 3, 1, 1)
    x = (x - mean) / std
    h, w = x.shape[-2:]
    x = F.pad(x, (0, img_size - w, 0, img_size - h))
    return x, (h, w)


# --------------------------------------------------------------------------- #
# Prompt encoder (Appendix B.2)
# --------------------------------------------------------------------------- #
def _pe_encoding(sd: SD, coords, prefix="prompt_encoder."):
    coords = 2 * coords - 1
    coords = coords @ sd[prefix + "pe_layer.positional_encoding_gaussian_matrix"]
    coords = 2 * math.pi * coords
    return torch.cat([torch.sin(coords), torch.cos(coords)], dim=-1)


def get_dense_pe(sd: SD, emb_hw=(64, 64), prefix="prompt_encoder."):
    h, w = emb_hw
    grid = torch.ones((h, w), dtype=sd[prefix + "pe_layer.positional_encoding_gaussian_matrix"].dtype)
    y_embed = (grid.cumsum(dim=0) - 0.5) / h
    x_embed = (grid.cumsum(dim=1) - 0.5) / w
    pe = _pe_encoding(sd, torch.stack([x_embed, y_embed], dim=-1), prefix)
    return pe.permute(2, 0, 1)[None]


def _pe_with_coords(sd, coords, image_size, prefix):
    coords = coords.clone()
    coords[:, :, 0] = coords[:, :, 0] / image_size[1]
    coords[:, :, 1] = coords[:, :, 1] / image_size[0]
    return _pe_encoding(sd, coords.to(sd[prefix + "pe_layer.positional_encoding_gaussian_matrix"].dtype), prefix)


def prompt_encode(sd: SD, points, boxes, masks, img_size=1024, emb_hw=(64, 64), prefix="prompt_encoder."):
    """points = (coords (B,K,2) float in the 1024 frame, labels (B,K) int) or None; boxes (B,4)/(B,1,4) or None;
    masks (B,1,256,256) or None.  Returns sparse (B,K',256), dense (B,256,64,64), in the dtype of the state dict."""
    p = prefix
    dt = sd[p + "pe_layer.positional_encoding_gaussian_matrix"].dtype
    bs = 1
    if points is not None:
        bs = points[0].shape[0]
    elif boxes is not None:
        bs = boxes.shape[0]
    elif masks is not None:
        bs = masks.shape[0]
    sparse = torch.empty((bs, 0, 256), dtype=dt)
    if points is not None:
        coords, labels = points
        coords = coords + 0.5
        if boxes is None:
            coords = torch.cat([coords, torch.zeros((bs, 1, 2), dtype=coords.dtype)], dim=1)
            labels = torch.cat([labels, -torch.ones((bs, 1), dtype=labels.dtype)], dim=1)
        pe = _pe_with_coords(sd, coords, (img_size, img_size), p)
        pe[labels == -1] = 0.0
        pe[labels == -1] += sd[p + "not_a_point_embed.weight"][0]
        pe[labels == 0] += sd[p + "point_embeddings.0.weight"][0]
        pe[labels == 1] += sd[p + "point_embeddings.1.weight"][0]
        sparse = torch.cat([sparse, pe], dim=1)
    if boxes is not None:
        b = boxes + 0.5
        c = b.reshape(-1, 2, 2)
        ce = _pe_with_coords(sd, c, (img_size, img_size), p)
        ce[:, 0, :] += sd[p + "point_embeddings.2.weight"][0]
        ce[:, 1, :] += sd[p + "point_embeddings.3.weight"][0]
        sparse = torch.cat([sparse, ce], dim=1)
    if masks is not None:
        m = F.conv2d(masks, sd[p + "mask_downscaling.0.weight"], sd[p + "mask_downscaling.0.bias"], stride=2)
        m = F.gelu(_ln2d(m, sd[p + "mask_downscaling.1.weight"], sd[p + "mask_downscaling.1.bias"]))
        m = F.conv2d(m, sd[p + "mask_downscaling.3.weight"], sd[p + "mask_downscaling.3.bias"], stride=2)
        m = F.gelu(_ln2d(m, sd[p + "mask_downscaling.4.weight"], sd[p + "mask_downscaling.4.bias"]))
        dense = F.conv2d(m, sd[p + "mask_downscaling.6.weight"], sd[p + "mask_downscaling.6.bias"])
    else:
        dense = sd[p + "no_mask_embed.weight"].reshape(1, -1, 1, 1).expand(bs, -1, emb_hw[0], emb_hw[1])
    return sparse, dense


# --------------------------------------------------------------------------- #
# Two-way transformer + mask decoder (Appendix B.2)
# --------------------------------------------------------------------------- #
def _attn(sd: SD, p: str, q, k, v, num_heads=8):
    q = F.linear(q, sd[p + "q_proj.weight"], sd[p + "q_proj.bias"])
    k = F.linear(k, sd[p + "k_proj.weight"], sd[p + "k_proj.bias"])
    v = F.linear(v, sd[p + "v_proj.weight"], sd[p + "v_proj.bias"])

    def sep(x):
        b, n, c = x.shape
        return x.reshape(b, n, num_heads, c // num_heads).transpose(1, 2)

    q, k, v = sep(q), sep(k), sep(v)
    cph = q.shape[-1]
    attn = (q @ k.permute(0, 1, 3, 2)) / math.sqrt(cph)
    attn = torch.softmax(attn, dim=-1)
    out = attn @ v
    b, h, n, c = out.shape
    out = out.transpose(1, 2).reshape(b, n, h * c)
    return F.linear(out, sd[p + "out_proj.weight"], sd[p + "out_proj.bias"])


def two_way_transformer(sd: SD, p: str, image_embedding, image_pe, point_embedding, depth=2, num_heads=8):
    bs, c, h, w = image_embedding.shape
    keys = image_embedding.flatten(2).permute(0, 2, 1)
    key_pe = image_pe.flatten(2).permute(0, 2, 1)
    queries = point_embedding
    query_pe = point_embedding
    for i in range(depth):
        lp = f"{p}layers.{i}."
        if i == 0:
            queries = _attn(sd, lp + "self_attn.", queries, queries, queries, num_heads)
        else:
            q = queries + query_pe
            queries = queries + _attn(sd, lp + "self_attn.", q, q, queries, num_heads)
        queries = _ln(queries, sd[lp + "norm1.weight"], sd[lp + "norm1.bias"], 1e-5)
        q = queries + query_pe
        k = keys + key_pe
        queries = queries + _attn(sd, lp + "cross_attn_token_to_image.", q, k, keys, num_heads)
        queries = _ln(queries, sd[lp + "norm2.weight"], sd[lp + "norm2.bias"], 1e-5)
        m = F.linear(queries, sd[lp + "mlp.lin1.weight"], sd[lp + "mlp.lin1.bias"])
        m = F.linear(F.relu(m), sd[lp + "mlp.lin2.weight"], sd[lp + "mlp.lin2.bias"])
        queries = _ln(queries + m, sd[lp + "norm3.weight"], sd[lp + "norm3.bias"], 1e-5)
        q = queries + query_pe
        k = keys + key_pe
        keys = keys + _attn(sd, lp + "cross_attn_image_to_token.", k, q, queries, num_heads)
        keys = _ln(keys, sd[lp + "norm4.weight"], sd[lp + "norm4.bias"], 1e-5)
    q = queries + query_pe
    k = keys + key_pe
    queries = queries + _attn(sd, p + "final_attn_token_to_image.", q, k, keys, num_heads)
    queries = _ln(queries, sd[p + "norm_final_attn.weight"], sd[p + "norm_final_attn.bias"], 1e-5)
    return queries, keys


def _mlp(sd: SD, p: str, x, n_layers=3):
    for i in range(n_layers):
        x = F.linear(x, sd[f"{p}layers.{i}.weight"], sd[f"{p}layers.{i}.bias"])
        if i < n_layers - 1:
            x = F.relu(x)
    return x


def mask_decode(sd: SD, image_embeddings, image_pe, sparse, dense, multimask_output=False, prefix="mask_decoder.",
                hq: Optional[dict] = None):
    """-> (masks (B,1|3,256,256), iou (B,1|3)).  `hq` = {"interm": (B,64,64,vit_dim), "hq_token_only": bool}
    selects the MaskDecoderHQ variant (SURVEY Appendix B.2 last paragraph)."""
    p = prefix
    n_mask_tok = 4
    toks = [sd[p + "iou_token.weight"], sd[p + "mask_tokens.weight"]]
    if hq is not None:
        toks.append(sd[p + "hf_token.weight"])
    output_tokens = torch.cat(toks, dim=0)
    output_tokens = output_tokens.unsqueeze(0).expand(sparse.shape[0], -1, -1)
    tokens = torch.cat((output_tokens, sparse), dim=1)
    src = torch.repeat_interleave(image_embeddings, tokens.shape[0], dim=0) + dense
    pos_src = torch.repeat_interleave(image_pe, tokens.shape[0], dim=0)
    b, c, h, w = src.shape
    if hq is not None:
        hq = dict(hq)
        hq["_pre_src"] = src
    hs, src = two_way_transformer(sd, p + "transformer.", src, pos_src, tokens)
    iou_token_out = hs[:, 0, :]
    ntok = n_mask_tok + (1 if hq is not None else 0)
    mask_tokens_out = hs[:, 1:1 + ntok, :]
    src = src.transpose(1, 2).view(b, c, h, w)
    if hq is not None and hq.get("hf_upscale_quirk", False):
        # transformers' sam_hq port up-scales the PRE-transformer embedding, spatially transposed
        # (modeling_sam_hq.py: `image_embeddings.transpose(2, 3).reshape(...)` on the (B,C,H,W) input); upstream m43/sam-hq
        # up-scales the transformer's output.  Only used to cross-check the remaining HQ pieces against HF.
        src = hq["_pre_src"].transpose(2, 3).reshape(b, c, h, w)
    u = F.conv_transpose2d(src, sd[p + "output_upscaling.0.weight"], sd[p + "output_upscaling.0.bias"], stride=2)
    u = F.gelu(_ln2d(u, sd[p + "output_upscaling.1.weight"], sd[p + "output_upscaling.1.bias"]))
    u = F.gelu(F.conv_transpose2d(u, sd[p + "output_upscaling.3.weight"], sd[p + "output_upscaling.3.bias"], stride=2))
    hyper = [
        _mlp(sd, f"{p}output_hypernetworks_mlps.{i}.", mask_tokens_out[:, i, :]) for i in range(n_mask_tok)
    ]
    if hq is not None:
        # HQ features = embedding_encoder(image_embeddings) + compress_vit_feat(interm[0])
        vit = hq["interm"].permute(0, 3, 1, 2)
        e = F.conv_transpose2d(image_embeddings, sd[p + "embedding_encoder.0.weight"], sd[p + "embedding_encoder.0.bias"], stride=2)
        e = F.gelu(_ln2d(e, sd[p + "embedding_encoder.1.weight"], sd[p + "embedding_encoder.1.bias"]))
        e = F.conv_transpose2d(e, sd[p + "embedding_encoder.3.weight"], sd[p + "embedding_encoder.3.bias"], stride=2)
        cv = F.conv_transpose2d(vit, sd[p + "compress_vit_feat.0.weight"], sd[p + "compress_vit_feat.0.bias"], stride=2)
        cv = F.gelu(_ln2d(cv, sd[p + "compress_vit_feat.1.weight"], sd[p + "compress_vit_feat.1.bias"]))
        cv = F.conv_transpose2d(cv, sd[p + "compress_vit_feat.3.weight"], sd[p + "compress_vit_feat.3.bias"], stride=2)
        hq_feat = e + cv
        hq_feat = hq_feat.repeat(b, 1, 1, 1)
        mf = F.conv2d(u, sd[p + "embedding_maskfeature.0.weight"], sd[p + "embedding_maskfeature.0.bias"], padding=1)
        mf = F.gelu(_ln2d(mf, sd[p + "embedding_maskfeature.1.weight"], sd[p + "embedding_maskfeature.1.bias"]))
        mf = F.conv2d(mf, sd[p + "embedding_maskfeature.3.weight"], sd[p + "embedding_maskfeature.3.bias"], padding=1)
        u_hq = mf + hq_feat
        hyper.append(_mlp(sd, p + "hf_mlp.", mask_tokens_out[:, n_mask_tok, :]))
    hyper_in = torch.stack(hyper, dim=1)
    b, c, h, w = u.shape
    masks = (hyper_in[:, :n_mask_tok] @ u.view(b, c, h * w)).view(b, -1, h, w)
    if hq is not None:
        m_hq = (hyper_in[:, n_mask_tok:] @ u_hq.view(b, c, h * w)).view(b, -1, h, w)
    iou = _mlp(sd, p + "iou_prediction_head.", iou_token_out)
    if multimask_output:
        sl = slice(1, n_mask_tok)
        if hq is not None:
            iou_s = iou[:, sl]
            iou_s, idx = torch.max(iou_s, dim=1)
            masks_s = masks[:, sl][torch.arange(masks.shape[0]), idx].unsqueeze(1)
            out = masks_s if hq.get("hq_token_only", False) else masks_s + m_hq
            return (m_hq if hq.get("hq_token_only", False) else out), iou_s.unsqueeze(1)
        return masks[:, sl], iou[:, sl]
    sl = slice(0, 1)
    if hq is not None:
        m = m_hq if hq.get("hq_token_only", False) else masks[:, sl] + m_hq
        return m, iou[:, sl]
    return masks[:, sl], iou[:, sl]


def postprocess_masks(masks, input_size, original_size, img_size=1024):
    masks = F.interpolate(masks, (img_size, img_size), mode="bilinear", align_corners=False)
    masks = masks[..., : input_size[0], : input_size[1]]
    return F.interpolate(masks, original_size, mode="bilinear", align_corners=False)


# --------------------------------------------------------------------------- #
# SamPredictor restatement
# --------------------------------------------------------------------------- #
class RefSamPredictor:
    """Functional stand-in for segment_anything.predictor.SamPredictor (members used by the reference,
    SURVEY §8b): set_image, predict_torch, transform.apply_coords, original_size, input_size, features."""

    mask_threshold = 0.0

    class _Transform:
        def __init__(self, long_side):
            self.target_length = long_side

        def apply_coords(self, coords, original_size):
            return apply_coords(coords, original_size, self.target_length)

    def __init__(self, sd: SD, cfg: VitCfg, hq: bool = False):
        self.sd, self.cfg, self.hq = sd, cfg, hq
        self.transform = self._Transform(cfg.img_size)
        self.features = None
        self.interm = None
        self._dense_pe = get_dense_pe(sd)

    @torch.no_grad()
    def set_image(self, image_hwc_u8: np.ndarray):
        x, self.input_size = preprocess(image_hwc_u8, self.cfg.img_size, self.cfg.img_size)
        self.original_size = tuple(image_hwc_u8.shape[:2])
        if self.hq:
            self.features, self.interm = vit_encode(self.sd, x, self.cfg, return_interm=True)
        else:
            self.features = vit_encode(self.sd, x, self.cfg)

    @torch.no_grad()
    def predict_torch(self, point_coords, point_labels, boxes=None, mask_input=None, multimask_output=True,
                      return_logits=False):
        points = (point_coords, point_labels) if point_coords is not None else None
        sparse, dense = prompt_encode(self.sd, points, boxes, mask_input, self.cfg.img_size)
        hq = {"interm": self.interm[0], "hq_token_only": False} if self.hq else None
        low_res, iou = mask_decode(self.sd, self.features, self._dense_pe, sparse, dense, multimask_output, hq=hq)
        masks = postprocess_masks(low_res, self.input_size, self.original_size, self.cfg.img_size)
        if not return_logits:
            masks = masks > self.mask_threshold
        return masks, iou, low_res


# --------------------------------------------------------------------------- #
# state-dict construction (shapes = SURVEY Appendix B.4)
# --------------------------------------------------------------------------- #
def sam_state_dict_shapes(cfg: VitCfg, hq: bool = False) -> Dict[str, Tuple[int, ...]]:
    D, hd = cfg.embed_dim, cfg.embed_dim // cfg.num_heads
    g = cfg.img_size // cfg.patch_size
    s: Dict[str, Tuple[int, ...]] = {}
    p = "image_encoder."
    s[p + "pos_embed"] = (1, g, g, D)
    s[p + "patch_embed.proj.weight"] = (D, 3, cfg.patch_size, cfg.patch_size)
    s[p + "patch_embed.proj.bias"] = (D,)
    for i in range(cfg.depth):
        b = f"{p}blocks.{i}."
        S = g if i in cfg.global_attn_indexes else cfg.window_size
        s[b + "norm1.weight"] = (D,); s[b + "norm1.bias"] = (D,)
        s[b + "attn.rel_pos_h"] = (2 * S - 1, hd); s[b + "attn.rel_pos_w"] = (2 * S - 1, hd)
        s[b + "attn.qkv.weight"] = (3 * D, D); s[b + "attn.qkv.bias"] = (3 * D,)
        s[b + "attn.proj.weight"] = (D, D); s[b + "attn.proj.bias"] = (D,)
        s[b + "norm2.weight"] = (D,); s[b + "norm2.bias"] = (D,)
        s[b + "mlp.lin1.weight"] = (cfg.mlp_ratio * D, D); s[b + "mlp.lin1.bias"] = (cfg.mlp_ratio * D,)
        s[b + "mlp.lin2.weight"] = (D, cfg.mlp_ratio * D); s[b + "mlp.lin2.bias"] = (D,)
    C = cfg.out_chans
    s[p + "neck.0.weight"] = (C, D, 1, 1)
    s[p + "neck.1.weight"] = (C,); s[p + "neck.1.bias"] = (C,)
    s[p + "neck.2.weight"] = (C, C, 3, 3)
    s[p + "neck.3.weight"] = (C,); s[p + "neck.3.bias"] = (C,)
    p = "prompt_encoder."
    s[p + "pe_layer.positional_encoding_gaussian_matrix"] = (2, C // 2)
    for i in range(4):
        s[f"{p}point_embeddings.{i}.weight"] = (1, C)
    s[p + "not_a_point_embed.weight"] = (1, C)
    s[p + "no_mask_embed.weight"] = (1, C)
    s[p + "mask_downscaling.0.weight"] = (4, 1, 2, 2); s[p + "mask_downscaling.0.bias"] = (4,)
    s[p + "mask_downscaling.1.weight"] = (4,); s[p + "mask_downscaling.1.bias"] = (4,)
    s[p + "mask_downscaling.3.weight"] = (16, 4, 2, 2); s[p + "mask_downscaling.3.bias"] = (16,)
    s[p + "mask_downscaling.4.weight"] = (16,); s[p + "mask_downscaling.4.bias"] = (16,)
    s[p + "mask_downscaling.6.weight"] = (C, 16, 1, 1); s[p + "mask_downscaling.6.bias"] = (C,)
    p = "mask_decoder."

    def attn(pp, internal):
        for n in ("q_proj", "k_proj", "v_proj"):
            s[f"{pp}{n}.weight"] = (internal, C); s[f"{pp}{n}.bias"] = (internal,)
        s[pp + "out_proj.weight"] = (C, internal); s[pp + "out_proj.bias"] = (C,)

    for i in range(2):
        lp = f"{p}transformer.layers.{i}."
        attn(lp + "self_attn.", C)
        attn(lp + "cross_attn_token_to_image.", C // 2)
        attn(lp + "cross_attn_image_to_token.", C // 2)
        for n in range(1, 5):
            s[f"{lp}norm{n}.weight"] = (C,); s[f"{lp}norm{n}.bias"] = (C,)
        s[lp + "mlp.lin1.weight"] = (2048, C); s[lp + "mlp.lin1.bias"] = (2048,)
        s[lp + "mlp.lin2.weight"] = (C, 2048); s[lp + "mlp.lin2.bias"] = (C,)
    attn(p + "transformer.final_attn_token_to_image.", C // 2)
    s[p + "transformer.norm_final_attn.weight"] = (C,); s[p + "transformer.norm_final_attn.bias"] = (C,)
    s[p + "iou_token.weight"] = (1, C)
    s[p + "mask_tokens.weight"] = (4, C)
    s[p + "output_upscaling.0.weight"] = (C, C // 4, 2, 2); s[p + "output_upscaling.0.bias"] = (C // 4,)
    s[p + "output_upscaling.1.weight"] = (C // 4,); s[p + "output_upscaling.1.bias"] = (C // 4,)
    s[p + "output_upscaling.3.weight"] = (C // 4, C // 8, 2, 2); s[p + "output_upscaling.3.bias"] = (C // 8,)
    for i in range(4):
        mp = f"{p}output_hypernetworks_mlps.{i}."
        s[mp + "layers.0.weight"] = (C, C); s[mp + "layers.0.bias"] = (C,)
        s[mp + "layers.1.weight"] = (C, C); s[mp + "layers.1.bias"] = (C,)
        s[mp + "layers.2.weight"] = (C // 8, C); s[mp + "layers.2.bias"] = (C // 8,)
    mp = p + "iou_prediction_head."
    s[mp + "layers.0.weight"] = (256, C); s[mp + "layers.0.bias"] = (256,)
    s[mp + "layers.1.weight"] = (256, 256); s[mp + "layers.1.bias"] = (256,)
    s[mp + "layers.2.weight"] = (4, 256); s[mp + "layers.2.bias"] = (4,)
    if hq:
        s[p + "hf_token.weight"] = (1, C)
        mp = p + "hf_mlp."
        s[mp + "layers.0.weight"] = (C, C); s[mp + "layers.0.bias"] = (C,)
        s[mp + "layers.1.weight"] = (C, C); s[mp + "layers.1.bias"] = (C,)
        s[mp + "layers.2.weight"] = (C // 8, C); s[mp + "layers.2.bias"] = (C // 8,)
        s[p + "compress_vit_feat.0.weight"] = (D, C, 2, 2); s[p + "compress_vit_feat.0.bias"] = (C,)
        s[p + "compress_vit_feat.1.weight"] = (C,); s[p + "compress_vit_feat.1.bias"] = (C,)
        s[p + "compress_vit_feat.3.weight"] = (C, C // 8, 2, 2); s[p + "compress_vit_feat.3.bias"] = (C // 8,)
        s[p + "embedding_encoder.0.weight"] = (C, C // 4, 2, 2); s[p + "embedding_encoder.0.bias"] = (C // 4,)
        s[p + "embedding_encoder.1.weight"] = (C // 4,); s[p + "embedding_encoder.1.bias"] = (C // 4,)
        s[p + "embedding_encoder.3.weight"] = (C // 4, C // 8, 2, 2); s[p + "embedding_encoder.3.bias"] = (C // 8,)
        s[p + "embedding_maskfeature.0.weight"] = (C // 4, C // 8, 3, 3); s[p + "embedding_maskfeature.0.bias"] = (C // 4,)
        s[p + "embedding_maskfeature.1.weight"] = (C // 4,); s[p + "embedding_maskfeature.1.bias"] = (C // 4,)
        s[p + "embedding_maskfeature.3.weight"] = (C // 8, C // 4, 3, 3); s[p + "embedding_maskfeature.3.bias"] = (C // 8,)
    return s
