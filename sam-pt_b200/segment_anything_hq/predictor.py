"""`SamPredictor` of HQ-SAM (m43/sam-hq segment_anything/predictor.py): same interface as SAM's; `set_image` additionally
keeps `interm_features` and the per-frame HQ feature map; `predict_torch(..., hq_token_only=False)` returns SAM mask + HQ mask."""
from ctypes import c_int

import torch

from sampt_b200 import native
from segment_anything.predictor import SamPredictor as _Base


class SamPredictor(_Base):
    def __init__(self, sam_model) -> None:
        # sam-hq's predictor unpacks (features, interm_embeddings) from the encoder and runs MaskDecoderHQ.  A plain SAM or
        # MobileSAM model (sam_pt.yaml's default predictor with `model/sam@...=sam_mobile_vit_tiny`) would only fail on the
        # first frame, so it is refused here.
        if "hf_token.weight" not in sam_model.mask_decoder.state_dict():
            raise ValueError(
                f"segment_anything_hq.predictor.SamPredictor needs an HQ-SAM model (MaskDecoderHQ); "
                f"{type(sam_model).__name__} has a {type(sam_model.mask_decoder).__name__}. For SAM or MobileSAM select the "
                "plain predictor with model.sam_predictor._target_=segment_anything.predictor.SamPredictor")
        super().__init__(sam_model)

    def _uses_interm(self) -> bool:
        return True

    def reset_image(self) -> None:
        super().reset_image()
        self._hq_feat = None
        self._hq_src = None

    def _hq_features(self) -> torch.Tensor:
        """[256*256, 32] = embedding_encoder(features) + compress_vit_feat(interm_features[0]) for the current frame."""
        if self._hq_feat is None or self._hq_src is not self.features:
            if self.interm_features is None:
                raise RuntimeError("HQ-SAM needs the intermediate ViT embeddings; use set_image / encode_frames(want_interm=True)")
            ctx = self.model.native_context()
            tok = self._tokens()
            g = self.features.shape[-1]
            interm = self.interm_features
            interm = interm[0] if isinstance(interm, (list, tuple)) else interm
            it = interm.reshape(g * g, -1).contiguous().float()
            out = torch.empty((16 * g * g, 32), device=self.device, dtype=torch.float32)
            # per-call scratch from the (stream-aware) torch allocator: the decode chains of different frames run concurrently
            # on several streams, a shared workspace would race (round-1 advisor finding)
            scratch = torch.empty((g * g * 1280,), device=self.device, dtype=torch.float32)
            native.check(native.lib().sampt_sam_hq_features(ctx.handle, native.ptr(tok), native.ptr(it), c_int(g), native.ptr(scratch),
                                                            native.ptr(out), native.stream_ptr()), "sam_hq_features")
            self._hq_feat, self._hq_src = out, self.features
        return self._hq_feat

    def _select_hq(self, on: bool = True) -> None:
        ctx = self.model.native_context()
        native.check(native.lib().sampt_sam_set_hq_features(ctx.handle, native.ptr(self._hq_features()) if on else None), "set_hq")

    @torch.no_grad()
    def predict_torch(self, point_coords, point_labels, boxes=None, mask_input=None, multimask_output=True, return_logits=False,
                      hq_token_only=False):
        if hq_token_only or multimask_output:
            raise NotImplementedError("HQ-SAM on the SAM-PT path uses multimask_output=False, hq_token_only=False "
                                      "(sam_pt/modeling/sam_pt.py:783-828); other modes are not built")
        self._select_hq(True)
        try:
            return super().predict_torch(point_coords, point_labels, boxes, mask_input, multimask_output, return_logits)
        finally:
            native.check(native.lib().sampt_sam_set_hq_features(self.model.native_context().handle, None), "set_hq")

    @torch.no_grad()
    def predict_refine(self, coords_1024, labels, n_positive_first, n_refine, logits_out, slot=0, positive_index=None):
        self._select_hq(True)
        try:
            return super().predict_refine(coords_1024, labels, n_positive_first, n_refine, logits_out, slot, positive_index)
        finally:
            native.check(native.lib().sampt_sam_set_hq_features(self.model.native_context().handle, None), "set_hq")
