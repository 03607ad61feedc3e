"""The oracle's prompt encoder / mask decoder / postprocess follow the dtype of the state dict: float64 serves as the reference
of the decoder's kernel tests (tests/test_gpu_decoder.py), and the float32 path, the one pinned against transformers' SAM, is
bit-identical to the float32-only restatement it replaced (kept below verbatim)."""
import math

import torch

from oracle import sam_ref
from sampt_b200 import synth


def _f32_pe_with_coords(sd, coords, image_size, prefix):
    coords = coords.clone()
    coords[:, :, 0] = coords[:, :, 0] / image_size[1]
    coords[:, :, 1] = coords[:, :, 1] / image_size[0]
    c = 2 * coords.float() - 1
    c = c @ sd[prefix + "pe_layer.positional_encoding_gaussian_matrix"]
    c = 2 * math.pi * c
    return torch.cat([torch.sin(c), torch.cos(c)], dim=-1)


def _f32_dense_pe(sd, emb_hw=(64, 64), prefix="prompt_encoder."):
    h, w = emb_hw
    grid = torch.ones((h, w), dtype=torch.float32)
    y_embed = (grid.cumsum(dim=0) - 0.5) / h
    x_embed = (grid.cumsum(dim=1) - 0.5) / w
    return sam_ref._pe_encoding(sd, torch.stack([x_embed, y_embed], dim=-1), prefix).permute(2, 0, 1)[None]


def _f32_prompt_encode(sd, points, boxes, masks, p="prompt_encoder."):
    bs = points[0].shape[0]
    coords, labels = points
    coords = coords + 0.5
    if boxes is None:
        coords = torch.cat([coords, torch.zeros((bs, 1, 2))], dim=1)
        labels = torch.cat([labels, -torch.ones((bs, 1), dtype=labels.dtype)], dim=1)
    pe = _f32_pe_with_coords(sd, coords, (1024, 1024), p)
    pe[labels == -1] = 0.0
    pe[labels == -1] += sd[p + "not_a_point_embed.weight"][0]
    pe[labels == 0] += sd[p + "point_embeddings.0.weight"][0]
    pe[labels == 1] += sd[p + "point_embeddings.1.weight"][0]
    sparse = torch.cat([torch.empty((bs, 0, 256)), pe], dim=1)
    if boxes is not None:
        ce = _f32_pe_with_coords(sd, (boxes + 0.5).reshape(-1, 2, 2), (1024, 1024), p)
        ce[:, 0, :] += sd[p + "point_embeddings.2.weight"][0]
        ce[:, 1, :] += sd[p + "point_embeddings.3.weight"][0]
        sparse = torch.cat([sparse, ce], dim=1)
    _, dense = sam_ref.prompt_encode(sd, None, None, masks)
    return sparse, dense


def _decode(sd, feats, pts, labels, box, mask_in, encode, dense_pe):
    sparse, dense = encode(sd, (pts, labels), box, mask_in)
    low, iou = sam_ref.mask_decode(sd, feats, dense_pe, sparse, dense, multimask_output=True)
    return sparse, dense, low, iou, sam_ref.postprocess_masks(low, (576, 1024), (480, 854))


def test_decoder_oracle_float32_bit_identical_and_float64_runs():
    sd = synth.condition_sam(synth.make_state_dict(sam_ref.sam_state_dict_shapes(sam_ref.VIT_TEST), 41))
    g = torch.Generator().manual_seed(2)
    feats = torch.randn((1, 256, 64, 64), generator=g)
    pts = torch.rand((1, 7, 2), generator=g) * torch.tensor([1000.0, 560.0])
    labels = torch.tensor([[1, 0, -1, 1, 1, 0, 1]])
    box = torch.tensor([[100.0, 150.0, 700.0, 440.0]])
    mask_in = torch.randn((1, 1, 256, 256), generator=g)
    for b in (None, box):
        new = _decode(sd, feats, pts, labels, b, mask_in, sam_ref.prompt_encode, sam_ref.get_dense_pe(sd))
        old = _decode(sd, feats, pts, labels, b, mask_in, _f32_prompt_encode, _f32_dense_pe(sd))
        for a, o in zip(new, old):
            assert a.dtype == torch.float32 and torch.equal(a, o)
    sd64 = {k: v.double() for k, v in sd.items()}
    new64 = _decode(sd64, feats.double(), pts.double(), labels, box, mask_in.double(), sam_ref.prompt_encode,
                    sam_ref.get_dense_pe(sd64))
    for a, o in zip(new64, new):
        assert a.dtype == torch.float64
        assert (a - o.double()).abs().max() <= 1e-4 * max(1.0, o.abs().max().item())
