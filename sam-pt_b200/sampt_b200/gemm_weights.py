"""Weight operands of the split-precision tensor-core GEMM (csrc/gemm_tc.cu through tv_gemm), shared by the TinyViT encoder and
the PIPS++ DeltaBlock."""
import math
from typing import Tuple

import torch


def split_scaled(wm: torch.Tensor, kp: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """[N, K] float64 -> ([N, 2*kp] fp16 hi | lo of w 2^s with zero columns K..kp in both halves, [2^-s] fp32).

    The power of two 2^s puts max |w| 2^s in [2^14, 2^15): unscaled, the lo halves of weights of size ~1/sqrt(K) fall below
    fp16's normal range (6.1e-5), where their absolute precision of 2^-24 costs ~2^-19 of every product.  Scaled, lo keeps
    11 bits and the product error is the 2^-22 of the split itself.  gemm_tc multiplies the accumulator by 2^-s (exact)."""
    w = torch.zeros((wm.shape[0], kp), dtype=torch.float32)
    w[:, :wm.shape[1]] = wm.float()
    amax = float(w.abs().max())
    s = 15 - (math.frexp(amax)[1] if amax > 0 else 0)
    w = w * (2.0 ** s)
    hi = w.half()
    return torch.cat([hi, (w - hi.float()).half()], dim=1).contiguous(), torch.tensor([2.0 ** -s], dtype=torch.float32)
