"""Hydra wrappers `SamHydra` / `SamHQHydra` with the reference's constructor contract (sam_pt/modeling/sam.py:12-51):
(image_encoder, prompt_encoder, mask_decoder, pixel_mean, pixel_std, checkpoint, prompt_embed_dim, image_size,
vit_patch_size, image_embedding_size); checkpoint=None allowed; state-dict loaded strict=False."""
import torch

from segment_anything.modeling import Sam


class BaseHydra:
    def __init__(self, model, checkpoint, prompt_embed_dim, image_size, vit_patch_size, image_embedding_size, **kwargs):
        super().__init__(**kwargs)
        if checkpoint is not None:
            with open(checkpoint, "rb") as f:
                state_dict = torch.load(f, map_location="cpu")
            model.load_state_dict(self, state_dict, strict=False)
            print(f"Loaded checkpoint from {checkpoint}.")
        self.prompt_embed_dim = prompt_embed_dim
        self.image_size = image_size
        self.vit_patch_size = vit_patch_size
        self.image_embedding_size = image_embedding_size


class SamHydra(BaseHydra, Sam):
    def __init__(self, *args, **kwargs):
        super().__init__(Sam, *args, **kwargs)


def __getattr__(name):
    if name == "SamHQHydra":
        from segment_anything_hq.modeling import Sam as SamHQ

        class SamHQHydra(BaseHydra, SamHQ):
            def __init__(self, *args, **kwargs):
                super().__init__(SamHQ, *args, **kwargs)

        globals()["SamHQHydra"] = SamHQHydra
        return SamHQHydra
    if name == "MobileSamHydra":
        raise ImportError("MobileSAM is outside the H100 hot-path scope (SURVEY §2 row 2)")
    raise AttributeError(name)
