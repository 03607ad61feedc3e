"""sam-hq's TinyViT (Light HQ-SAM): MobileSAM's encoder whose forward also returns `interm_embeddings`, of which
MaskDecoderHQ reads the first: layers.1's output (after its PatchMerging) viewed as (B, 64, 64, 160), hence
`vit_dim: 160` in configs/model/sam/samhq_light_vit_tiny.yaml."""
from mobile_sam.modeling.tiny_vit_sam import TinyViT as _Base


class TinyViT(_Base):
    returns_interm = True
