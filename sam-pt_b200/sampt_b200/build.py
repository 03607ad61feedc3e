"""In-tree build of libsampt_b200.so with plain nvcc for sm_90a (no torch C++ extension: the boundary is a C ABI)."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

PKG_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))  # .../sam-pt_b200
CSRC = os.path.join(PKG_ROOT, "csrc")
LIB_DIR = os.path.join(PKG_ROOT, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libsampt_b200.so")

# sm_90a only (wgmma / TMA); no --use_fast_math: sinf/cosf/expf/erff must stay the accurate versions (flow embeddings reach ~1e5 rad)
NVCC_COMPILE_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found (needed to build libsampt_b200.so for sm_90a)")


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


OBJ_DIR = os.path.join(PKG_ROOT, "build")
FLAGS_STAMP = os.path.join(OBJ_DIR, "nvcc_flags.txt")   # objects built with other flags (another architecture) are rebuilt


def _flags_changed() -> bool:
    try:
        with open(FLAGS_STAMP) as f:
            return f.read() != " ".join(NVCC_COMPILE_FLAGS)
    except OSError:
        return True


def is_stale() -> bool:
    if not os.path.exists(LIB_PATH) or _flags_changed():
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [
        os.path.join(os.path.dirname(PKG_ROOT), "include", "sampt_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build_native(force: bool = False, verbose: bool = False) -> str:
    """Compile every .cu under csrc/ into lib/libsampt_b200.so.  Each .cu is compiled to an object in parallel, then linked."""
    if not force and not is_stale():
        return LIB_PATH
    os.makedirs(LIB_DIR, exist_ok=True)
    objdir = OBJ_DIR
    os.makedirs(objdir, exist_ok=True)
    force = force or _flags_changed()
    nvcc = _nvcc()
    procs = []
    objs = []
    for src in sources():
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        if (not force) and os.path.exists(obj) and os.path.getmtime(obj) > max(
                os.path.getmtime(src), *[os.path.getmtime(os.path.join(CSRC, h)) for h in os.listdir(CSRC) if h.endswith(".cuh")]):
            continue
        cmd = [nvcc] + NVCC_COMPILE_FLAGS + ["-c", src, "-o", obj]
        if verbose:
            cmd += ["-Xptxas", "-v"]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{out}")
        if verbose and out:
            print(out, file=sys.stderr)
    link = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", LIB_PATH] + objs + ["-lcudart"]
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}")
    with open(FLAGS_STAMP, "w") as f:
        f.write(" ".join(NVCC_COMPILE_FLAGS))
    return LIB_PATH


if __name__ == "__main__":
    print(build_native(force="--force" in sys.argv, verbose="-v" in sys.argv))
