"""`PromptEncoder` parameter container (upstream segment_anything/modeling/prompt_encoder.py @ aac76a1; kwargs per
/root/reference/configs/model/sam/prompt_encoder/sam.yaml).  The arithmetic runs in csrc/decoder.cu
(prompt_tokens_kernel, dense_src_kernel); only `get_dense_pe` is evaluated here, once, with torch (constant table)."""
import math
from typing import Tuple

import torch
from torch import nn

from sampt_b200.param_tree import build_param_tree


class PromptEncoder(nn.Module):
    def __init__(self, embed_dim: int, image_embedding_size: Tuple[int, int], input_image_size: Tuple[int, int],
                 mask_in_chans: int, activation=nn.GELU) -> None:
        super().__init__()
        if embed_dim != 256 or mask_in_chans != 16:
            raise NotImplementedError("the H100 prompt encoder is built for embed_dim=256, mask_in_chans=16 (SAM)")
        self.embed_dim = embed_dim
        self.image_embedding_size = tuple(image_embedding_size)
        self.input_image_size = tuple(input_image_size)
        self.mask_input_size = (4 * self.image_embedding_size[0], 4 * self.image_embedding_size[1])
        c = embed_dim
        shapes = {"pe_layer.positional_encoding_gaussian_matrix": (2, c // 2), "not_a_point_embed.weight": (1, c),
                  "no_mask_embed.weight": (1, c), "mask_downscaling.0.weight": (4, 1, 2, 2), "mask_downscaling.0.bias": (4,),
                  "mask_downscaling.1.weight": (4,), "mask_downscaling.1.bias": (4,), "mask_downscaling.3.weight": (16, 4, 2, 2),
                  "mask_downscaling.3.bias": (16,), "mask_downscaling.4.weight": (16,), "mask_downscaling.4.bias": (16,),
                  "mask_downscaling.6.weight": (c, 16, 1, 1), "mask_downscaling.6.bias": (c,)}
        for i in range(4):
            shapes[f"point_embeddings.{i}.weight"] = (1, c)
        build_param_tree(self, shapes, seed=2048)

    @torch.no_grad()
    def get_dense_pe(self) -> torch.Tensor:
        """(1, C, h, w) positional encoding of the embedding grid (upstream PositionEmbeddingRandom.forward)."""
        h, w = self.image_embedding_size
        g = self.pe_layer.positional_encoding_gaussian_matrix
        grid = torch.ones((h, w), device=g.device, dtype=torch.float32)
        y = (grid.cumsum(dim=0) - 0.5) / h
        x = (grid.cumsum(dim=1) - 0.5) / w
        c = torch.stack([x, y], dim=-1)
        c = 2 * c - 1
        c = c @ g
        c = 2 * math.pi * c
        pe = torch.cat([torch.sin(c), torch.cos(c)], dim=-1)
        return pe.permute(2, 0, 1).unsqueeze(0)

    def forward(self, points, boxes, masks):
        raise NotImplementedError("prompt encoding is fused into libsampt_b200's decode step (SamPredictor.predict_torch)")
