"""`TwoWayTransformer` parameter container (upstream segment_anything/modeling/transformer.py @ aac76a1; kwargs per
/root/reference/configs/model/sam/mask_decoder/sam.yaml:3-8).  Arithmetic: csrc/decoder.cu (two_way_layer)."""
from torch import nn

from sampt_b200.param_tree import build_param_tree


class TwoWayTransformer(nn.Module):
    def __init__(self, depth: int, embedding_dim: int, num_heads: int, mlp_dim: int, activation=nn.ReLU,
                 attention_downsample_rate: int = 2) -> None:
        super().__init__()
        if (depth, embedding_dim, num_heads, mlp_dim, attention_downsample_rate) != (2, 256, 8, 2048, 2):
            raise NotImplementedError("the H100 mask decoder is built for SAM's two-way transformer: depth 2, dim 256, "
                                      "8 heads, mlp 2048, downsample 2")
        self.depth, self.embedding_dim, self.num_heads, self.mlp_dim = depth, embedding_dim, num_heads, mlp_dim
        c, ci = embedding_dim, embedding_dim // attention_downsample_rate
        shapes = {}

        def attn(p, internal):
            for n in ("q_proj", "k_proj", "v_proj"):
                shapes[f"{p}.{n}.weight"], shapes[f"{p}.{n}.bias"] = (internal, c), (internal,)
            shapes[f"{p}.out_proj.weight"], shapes[f"{p}.out_proj.bias"] = (c, internal), (c,)

        for i in range(depth):
            attn(f"layers.{i}.self_attn", c)
            attn(f"layers.{i}.cross_attn_token_to_image", ci)
            attn(f"layers.{i}.cross_attn_image_to_token", ci)
            for n in range(1, 5):
                shapes[f"layers.{i}.norm{n}.weight"] = shapes[f"layers.{i}.norm{n}.bias"] = (c,)
            shapes[f"layers.{i}.mlp.lin1.weight"], shapes[f"layers.{i}.mlp.lin1.bias"] = (mlp_dim, c), (mlp_dim,)
            shapes[f"layers.{i}.mlp.lin2.weight"], shapes[f"layers.{i}.mlp.lin2.bias"] = (c, mlp_dim), (c,)
        attn("final_attn_token_to_image", ci)
        shapes["norm_final_attn.weight"] = shapes["norm_final_attn.bias"] = (c,)
        build_param_tree(self, shapes, seed=4096)
