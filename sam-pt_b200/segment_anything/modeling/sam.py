"""`Sam` (upstream segment_anything/modeling/sam.py @ aac76a1): holds the three sub-modules + pixel statistics; the
reference sub-classes it as SamHydra (sam_pt/modeling/sam.py:34-41).  Here it also owns the registration of every weight
with libsampt_b200 in kernel-native layout."""
import os
from typing import List

import torch
from torch import nn

from sampt_b200 import native


class Sam(nn.Module):
    mask_threshold: float = 0.0
    image_format: str = "RGB"

    def __init__(self, image_encoder, prompt_encoder, mask_decoder, pixel_mean: List[float] = (123.675, 116.28, 103.53),
                 pixel_std: List[float] = (58.395, 57.12, 57.375)) -> None:
        super().__init__()
        self.image_encoder = image_encoder
        self.prompt_encoder = prompt_encoder
        self.mask_decoder = mask_decoder
        self.register_buffer("pixel_mean", torch.tensor(list(pixel_mean), dtype=torch.float32).view(-1, 1, 1), False)
        self.register_buffer("pixel_std", torch.tensor(list(pixel_std), dtype=torch.float32).view(-1, 1, 1), False)
        self._dec_registered = None
        self.use_cuda_graphs = os.environ.get("SAMPT_DECODE_GRAPHS", "1") != "0"

    @property
    def device(self):
        return self.pixel_mean.device

    def has_decoder_slab(self) -> bool:
        """True when the decode chain replays captured CUDA graphs out of per-slot buffers (several decode streams are safe)."""
        return bool(self.use_cuda_graphs)

    # ------------------------------------------------------------------ decoder weights -> libsampt_b200
    def native_context(self) -> native.Context:
        ctx = self.image_encoder.native_context()
        key = (id(ctx), tuple(p._version for p in self.prompt_encoder.parameters()),
               tuple(p._version for p in self.mask_decoder.parameters()), self.device)
        if self._dec_registered != key or not ctx.owns("sam.decoder", self):
            self._register_decoder(ctx)
            if self.use_cuda_graphs:
                ctx.set_decoder_workspace()  # also invalidates graphs captured with the previous weights
            else:
                ctx.clear_decoder_workspace()  # eager chain (single decode stream, see SamPt._apply_sam_to_frames)
            self._dec_registered = key
            ctx.claim("sam.decoder", self)
        return ctx

    @torch.no_grad()
    def _register_decoder(self, ctx: native.Context) -> None:
        pe, md = self.prompt_encoder, self.mask_decoder
        # another Sam (e.g. an HQ-SAM whose decoder has extra hf_* tensors) may have used these names on this device before
        torch.cuda.synchronize(ctx.device)
        ctx.unset_prefix("sam.prompt_encoder.")
        ctx.unset_prefix("sam.mask_decoder.")
        for k, v in pe.state_dict().items():
            ctx.set_tensor("sam.prompt_encoder." + k, v.float().reshape(-1) if v.dim() == 2 and v.shape[0] == 1 else v.float())
        sd = md.state_dict()
        for k, v in sd.items():
            ctx.set_tensor("sam.mask_decoder." + k, v.float())
        toks = [sd["iou_token.weight"], sd["mask_tokens.weight"]]
        if "hf_token.weight" in sd:
            toks.append(sd["hf_token.weight"])
        ctx.set_tensor("sam.mask_decoder.output_tokens", torch.cat(toks, dim=0).float())
        # ConvTranspose2d(256,64,2,2) as a GEMM: row n = (dy*2+dx)*64 + co, col = ci
        w0 = sd["output_upscaling.0.weight"].float()
        ctx.set_tensor("sam.mask_decoder.output_upscaling.0.weight_gemm", w0.permute(2, 3, 1, 0).reshape(-1, w0.shape[0]))
        ctx.set_tensor("sam.mask_decoder.output_upscaling.0.bias4", sd["output_upscaling.0.bias"].float().repeat(4))

        # image-side projections (4096-row operands) run on the tensor-core GEMM with the 3-pass fp16 hi|lo split (~fp32 products):
        # weights as [N, 2K] = hi | lo
        def w16(wm):
            wm = wm.float()
            hi = wm.half()
            return torch.cat([hi, (wm - hi.float()).half()], dim=1).contiguous()

        ctx.set_tensor("sam.mask_decoder.output_upscaling.0.w16", w16(w0.permute(2, 3, 1, 0).reshape(-1, w0.shape[0])))
        for name in [f"transformer.layers.{i}.cross_attn_token_to_image.{p}_proj" for i in range(2) for p in ("k", "v")] + \
                    [f"transformer.layers.{i}.cross_attn_image_to_token.{p}_proj" for i in range(2) for p in ("q", "out")] + \
                    [f"transformer.final_attn_token_to_image.{p}_proj" for p in ("k", "v")]:
            ctx.set_tensor(f"sam.mask_decoder.{name}.w16", w16(sd[name + ".weight"]))
        # key positional encoding folded through the (linear) k/q projections that consume `keys + key_pe`
        dense_pe = pe.get_dense_pe()[0].flatten(1).t().contiguous()  # (h*w, 256) token-major
        ctx.set_tensor("sam.dense_pe_tok", dense_pe)
        t = "sam.mask_decoder.transformer."
        for i in range(2):
            wk = sd[f"transformer.layers.{i}.cross_attn_token_to_image.k_proj.weight"].float()
            wq = sd[f"transformer.layers.{i}.cross_attn_image_to_token.q_proj.weight"].float()
            ctx.set_tensor(f"{t}layers.{i}.pek_t2i", dense_pe @ wk.t())
            ctx.set_tensor(f"{t}layers.{i}.peq_i2t", dense_pe @ wq.t())
        wk = sd["transformer.final_attn_token_to_image.k_proj.weight"].float()
        ctx.set_tensor(f"{t}pek_final", dense_pe @ wk.t())

    def forward(self, batched_input, multimask_output):
        raise NotImplementedError("use SamPredictor (set_image / predict_torch); the batched dict interface of upstream "
                                  "Sam.forward is not on the SAM-PT hot path")
