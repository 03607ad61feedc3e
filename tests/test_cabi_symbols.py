"""CPU: the C-ABI library builds (nvcc cross-compiles sm_90a without a GPU), loads, and exports every symbol that
include/sampt_b200.h declares.  No compute is called."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from sampt_b200 import build
    path = build.build_native()
    lib = ctypes.CDLL(path)
    header = open(os.path.join(ROOT, "include", "sampt_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    names = set(re.findall(r"\b(sampt_[a-z0-9_]+)\s*\(", header))
    assert len(names) >= 15
    missing = [n for n in sorted(names) if not hasattr(lib, n)]
    assert not missing, missing
    lib.sampt_version.restype = ctypes.c_int
    assert lib.sampt_version() >= 1


def test_product_never_imports_oracle():
    """The product path must not route through the oracle or any CPU fallback."""
    bad = []
    pkg = os.path.join(ROOT, "sam-pt_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith(".py"):
                src = open(os.path.join(dp, f)).read()
                if re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M):
                    bad.append(os.path.join(dp, f))
    assert not bad, bad


def test_missing_cuda_raises_loudly():
    import torch
    from sampt_b200 import native
    if torch.cuda.is_available():
        return
    import pytest
    with pytest.raises(RuntimeError):
        native.get_context("cuda")
    with pytest.raises(RuntimeError):
        native.get_context("cpu")
