"""ctypes binding of libsampt_b200.so (include/sampt_b200.h).  This is the ONLY way the Python host code reaches the GPU
kernels; there is no CPU or PyTorch-eager fallback: a missing library or a non-zero return code raises."""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_int, c_int64, c_longlong, c_size_t, c_void_p
from typing import Dict, Optional

import torch

from . import build as _build

_DTYPES = {torch.float32: 0, torch.float16: 1, torch.uint8: 2, torch.int32: 3, torch.bfloat16: 4}
_lib: Optional[ctypes.CDLL] = None


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        path = _build.LIB_PATH
        if not os.path.exists(path):
            raise RuntimeError(
                f"{path} is missing: the CUDA extension has not been built (run `python -c 'import __graft_entry__ as g; "
                f"g.build()'`). There is no CPU fallback for the SAM-PT hot path.")
        _lib = ctypes.CDLL(path)
        _lib.sampt_last_error.restype = c_char_p
        _lib.sampt_launch_count.restype = c_longlong
        _lib.sampt_launch_count.argtypes = [c_void_p]
    return _lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = lib().sampt_last_error()
        raise RuntimeError(f"libsampt_b200 {what} failed (code {rc}): {msg.decode() if msg else '?'}")


def ptr(t: Optional[torch.Tensor]) -> c_void_p:
    if t is None:
        return c_void_p(0)
    assert t.is_cuda and t.is_contiguous(), "native calls take contiguous CUDA tensors"
    return c_void_p(t.data_ptr())


def stream_ptr() -> c_void_p:
    return c_void_p(torch.cuda.current_stream().cuda_stream)


class Context:
    """Owns one sampt_ctx on a device, its workspace slab and references to every registered tensor."""

    def __init__(self, device: torch.device, workspace_bytes: int = 8 << 30):
        if not torch.cuda.is_available():
            raise RuntimeError("libsampt_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device(device)
        self._h = c_void_p()
        with torch.cuda.device(self.device):
            check(lib().sampt_ctx_create(c_int(self.device.index or 0), ctypes.byref(self._h)), "ctx_create")
        self._tensors: Dict[str, torch.Tensor] = {}
        self._owners: Dict[str, object] = {}
        self._ws = None
        self.set_workspace(workspace_bytes)

    @property
    def handle(self) -> c_void_p:
        return self._h

    def set_workspace(self, nbytes: int) -> None:
        self._ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        check(lib().sampt_ctx_set_workspace(self._h, ptr(self._ws), c_size_t(nbytes)), "set_workspace")

    def set_decoder_workspace(self, nbytes: int = 1536 << 20) -> None:
        """(Re)install the stable-address slab of the SAM decode chain; drops cached CUDA graphs."""
        self._dec_ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        check(lib().sampt_ctx_set_decoder_workspace(self._h, ptr(self._dec_ws), c_size_t(nbytes)), "set_decoder_workspace")

    def clear_decoder_workspace(self) -> None:
        """No decoder slab: sampt_sam_predict_refine runs its eager chain out of the shared workspace (one stream only)."""
        torch.cuda.synchronize(self.device)
        self._dec_ws = None
        check(lib().sampt_ctx_set_decoder_workspace(self._h, c_void_p(0), c_size_t(0)), "clear_decoder_workspace")

    def ensure_vit_workspace(self, nbytes: int) -> None:
        """Dedicated slab of the ViT encoder (lets it overlap with PIPS / decode on another stream)."""
        cur = getattr(self, "_vit_ws", None)
        if cur is None or cur.numel() < nbytes:
            torch.cuda.synchronize(self.device)  # nothing may still be running out of the old slab
            self._vit_ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
            check(lib().sampt_ctx_set_vit_workspace(self._h, ptr(self._vit_ws), c_size_t(nbytes)), "set_vit_workspace")

    def ensure_workspace(self, nbytes: int) -> None:
        if self._ws is None or self._ws.numel() < nbytes:
            self.set_workspace(nbytes)

    def set_tensor(self, name: str, t: torch.Tensor) -> None:
        t = t.to(self.device).contiguous()
        self._tensors[name] = t
        dims = (c_int64 * max(t.dim(), 1))(*t.shape)
        check(lib().sampt_set_tensor(self._h, name.encode(), ptr(t), c_int(_DTYPES[t.dtype]), c_int(t.dim()), dims),
              f"set_tensor({name})")

    def owns(self, namespace: str, owner) -> bool:
        """True when `owner` was the last module to register weights under `namespace` on this context.  Weight names are
        shared per device, so a second model of the same kind takes the namespace over and the first one must re-register
        before it runs again (its cached registration key alone cannot see that)."""
        ref = self._owners.get(namespace)
        return ref is not None and ref() is owner

    def claim(self, namespace: str, owner) -> None:
        import weakref
        self._owners[namespace] = weakref.ref(owner)

    def unset_prefix(self, prefix: str) -> None:
        """Drop every registered tensor whose name starts with `prefix` (C registry and the Python references)."""
        check(lib().sampt_unset_tensors(self._h, prefix.encode()), f"unset_tensors({prefix})")
        for k in [k for k in self._tensors if k.startswith(prefix)]:
            del self._tensors[k]

    def launch_count(self) -> int:
        return int(lib().sampt_launch_count(self._h))

    def __del__(self):
        try:
            if self._h:
                lib().sampt_ctx_destroy(self._h)
                self._h = c_void_p()
        except Exception:
            pass


_contexts: Dict[int, Context] = {}


def get_context(device) -> Context:
    """One shared context per device (weights of SAM and of the tracker are registered under distinct prefixes)."""
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError(f"the SAM-PT H100 path runs on CUDA only (got device {device}); there is no CPU fallback")
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if idx not in _contexts:
        _contexts[idx] = Context(torch.device("cuda", idx))
    return _contexts[idx]
