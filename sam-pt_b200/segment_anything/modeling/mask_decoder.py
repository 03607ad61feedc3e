"""`MaskDecoder` parameter container (upstream segment_anything/modeling/mask_decoder.py @ aac76a1; kwargs per
/root/reference/configs/model/sam/mask_decoder/sam.yaml).  Arithmetic: csrc/decoder.cu."""
from torch import nn

from sampt_b200.param_tree import build_param_tree


class MaskDecoder(nn.Module):
    def __init__(self, *, transformer_dim: int, transformer: nn.Module, num_multimask_outputs: int = 3, activation=nn.GELU,
                 iou_head_depth: int = 3, iou_head_hidden_dim: int = 256) -> None:
        super().__init__()
        if (transformer_dim, num_multimask_outputs, iou_head_depth, iou_head_hidden_dim) != (256, 3, 3, 256):
            raise NotImplementedError("the H100 mask decoder is built for SAM: dim 256, 3 multimask outputs, 3-layer heads")
        self.transformer_dim = transformer_dim
        self.transformer = transformer
        self.num_multimask_outputs = num_multimask_outputs
        self.num_mask_tokens = num_multimask_outputs + 1
        c = transformer_dim
        shapes = {"iou_token.weight": (1, c), "mask_tokens.weight": (self.num_mask_tokens, c),
                  "output_upscaling.0.weight": (c, c // 4, 2, 2), "output_upscaling.0.bias": (c // 4,),
                  "output_upscaling.1.weight": (c // 4,), "output_upscaling.1.bias": (c // 4,),
                  "output_upscaling.3.weight": (c // 4, c // 8, 2, 2), "output_upscaling.3.bias": (c // 8,)}
        for i in range(self.num_mask_tokens):
            p = f"output_hypernetworks_mlps.{i}.layers"
            shapes.update({f"{p}.0.weight": (c, c), f"{p}.0.bias": (c,), f"{p}.1.weight": (c, c), f"{p}.1.bias": (c,),
                           f"{p}.2.weight": (c // 8, c), f"{p}.2.bias": (c // 8,)})
        p = "iou_prediction_head.layers"
        h = iou_head_hidden_dim
        shapes.update({f"{p}.0.weight": (h, c), f"{p}.0.bias": (h,), f"{p}.1.weight": (h, h), f"{p}.1.bias": (h,),
                       f"{p}.2.weight": (self.num_mask_tokens, h), f"{p}.2.bias": (self.num_mask_tokens,)})
        build_param_tree(self, shapes, seed=8192)
