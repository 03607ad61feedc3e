"""MobileSAM's MaskDecoder is SAM's (segment_anything/modeling/mask_decoder.py)."""
from segment_anything.modeling.mask_decoder import MaskDecoder  # noqa: F401
