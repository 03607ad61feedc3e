"""State-dict-compatible parameter containers.

The drop-in modules must load the reference's checkpoints unchanged (key names of SURVEY.md Appendix A.4 / B.4) but
their forward runs in libsampt_b200, so they do not need torch layers -- only correctly named parameters.
`build_param_tree` materialises a {dotted.key: shape} table as nested nn.Module containers."""
from __future__ import annotations

from typing import Callable, Dict, Optional, Tuple

import torch
from torch import nn

from . import synth


class ParamNode(nn.Module):
    """Anonymous container; exists only to give parameters their dotted names."""


def build_param_tree(root: nn.Module, shapes: Dict[str, Tuple[int, ...]], seed: int = 0, init: bool = True,
                     values: Optional[Dict[str, torch.Tensor]] = None, is_buffer: Optional[Callable[[str], bool]] = None) -> None:
    """`values` (optional): initial tensors by key instead of the seeded init; `is_buffer(key)` (optional): register that key as a
    buffer (BatchNorm running statistics) rather than a parameter, keeping its dtype."""
    gen = torch.Generator().manual_seed(seed)
    for key in sorted(shapes):
        shape = tuple(shapes[key])
        mod = root
        *path, leaf = key.split(".")
        for p in path:
            if p not in mod._modules:
                mod.add_module(p, ParamNode())
            mod = mod._modules[p]
        if values is not None:
            value = values[key]
        else:
            value = synth._init_like_torch(key, shape, gen) if init else torch.empty(shape)
        if is_buffer is not None and is_buffer(key):
            mod.register_buffer(leaf, value)
        else:
            mod.register_parameter(leaf, nn.Parameter(value.float(), requires_grad=False))
