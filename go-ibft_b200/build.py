"""In-tree build of the CUDA engine (libibftverify.so) for sm_90a (H100) with nvcc.

The shared object is a build product (git-ignored); nvcc cross-compiles it without a GPU.
"""
from __future__ import annotations

import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libibftverify.so")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
              "-shared", "-diag-suppress", "550"]


def sources():
    out = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cuh", ".inc"))]
    out.append(os.path.join(HERE, "..", "include", "ibft_verify.h"))
    return out


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(s) > t for s in sources())


def build(force: bool = False, verbose: bool = False) -> str:
    if force or needs_build():
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB, os.path.join(CSRC, "engine.cu")]
        subprocess.check_call(cmd, cwd=CSRC)
    return LIB
