from .image_encoder import ImageEncoderViT  # noqa: F401
from .mask_decoder_hq import MaskDecoderHQ  # noqa: F401
from .prompt_encoder import PromptEncoder  # noqa: F401
from .sam import Sam  # noqa: F401
from .transformer import TwoWayTransformer  # noqa: F401
from .tiny_vit_sam import TinyViT  # noqa: F401
