"""mobile_sam.modeling: everything but the TinyViT encoder is upstream SAM's, re-exported from segment_anything."""
from segment_anything.modeling import MaskDecoder, PromptEncoder, Sam, TwoWayTransformer  # noqa: F401

from .tiny_vit_sam import TinyViT  # noqa: F401
