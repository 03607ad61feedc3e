"""MobileSAM's TwoWayTransformer is SAM's (segment_anything/modeling/transformer.py)."""
from segment_anything.modeling.transformer import TwoWayTransformer  # noqa: F401
