"""Builds the C-ABI shared library ``mapdn_b200/libmapdn_b200.so`` in-tree with nvcc for sm_90a.

    python -m mapdn_b200.build [--force]

nvcc cross-compiles without a GPU, so this also runs on the CPU-only dev box
(``__graft_entry__.build()``). The library has no PyTorch dependency: torch only supplies device
memory / streams on the Python side (``mapdn_b200/_capi.py``).
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libmapdn_b200.so")
SOURCES = [os.path.join(CSRC, "mapdn_b200.cu")]
DEPS = SOURCES + [os.path.join(CSRC, f) for f in ("env_kernel.cuh", "kernel_params.h", "philox.cuh")] + [
    os.path.join(HERE, "..", "include", "mapdn_b200.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--shared", "-Xcompiler", "-fPIC", "-Xptxas", "-v", "--expt-relaxed-constexpr",
]


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(d) > t for d in DEPS)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    extra = ["-DMAPDN_PROFILE"] if os.environ.get("MAPDN_PROFILE_BUILD") else []
    cmd = [nvcc] + NVCC_FLAGS + extra + ["-o", LIB] + SOURCES
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed building libmapdn_b200.so")
    log = os.path.join(HERE, "csrc", "ptxas.log")
    with open(log, "w") as f:
        f.write(res.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
