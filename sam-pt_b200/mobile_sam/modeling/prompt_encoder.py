"""MobileSAM's PromptEncoder is SAM's (segment_anything/modeling/prompt_encoder.py)."""
from segment_anything.modeling.prompt_encoder import PromptEncoder  # noqa: F401
