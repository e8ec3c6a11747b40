"""TEST INFRASTRUCTURE ONLY. ``tests/emu/_build/libmapdn_b200_emu.so``: the product's C-ABI library compiled with g++
against ``tests/emu/cuda_runtime.h`` (a CPU SIMT emulation: one OS thread per CUDA thread), so that the CPU test tier
executes the kernel SOURCE (``mapdn_b200/csrc/env_kernel.cuh``) through the product's own ``BatchedVoltageControl``
against the oracle. "Device pointers" are host memory, so the env runs on the CPU device. The product never loads this
library by itself (``mapdn_b200/_capi.py`` only knows ``libmapdn_b200.so``)."""
import ctypes as C
import os
import subprocess

import pytest
import torch

from mapdn_b200 import _capi
from mapdn_b200.env import BatchedVoltageControl

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "mapdn_b200", "csrc")
LIB = os.path.join(HERE, "_build", "libmapdn_b200_emu.so")
DEPS = [os.path.join(CSRC, f) for f in ("mapdn_b200.cu", "env_kernel.cuh", "kernel_params.h", "philox.cuh")] + [
    os.path.join(HERE, "cuda_runtime.h"), os.path.join(ROOT, "include", "mapdn_b200.h")]


def build(force=False):
    if not force and os.path.exists(LIB) and all(os.path.getmtime(d) <= os.path.getmtime(LIB) for d in DEPS):
        return LIB
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    cmd = ["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-pthread", "-DMAPDN_HOST_EMU", "-DMAPDN_EMU_DEFINE_GLOBALS",
           "-I", HERE, "-x", "c++", os.path.join(CSRC, "mapdn_b200.cu"), "-o", LIB]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("g++ failed building the emulated library:\n" + res.stderr[-4000:])
    return LIB


_L = None


def lib():
    global _L
    if _L is None:
        _L = _capi.bind(C.CDLL(build()))
        _L.mapdn_emu_last_grid.argtypes, _L.mapdn_emu_last_grid.restype = [], C.c_int
    return _L


def last_grid():
    """CTAs of the last emulated kernel launch (the persistent loop runs ceil(ceil(B / epb) / grid) rounds)."""
    return int(lib().mapdn_emu_last_grid())


def make_env(net, prof, env_args=None, **kw):
    """``BatchedVoltageControl`` on the emulated library: CPU tensors, NumPy views through ``.numpy()``."""
    return BatchedVoltageControl(net, prof, env_args, library=lib(), device="cpu", **kw)


@pytest.fixture(autouse=True)
def nan_filled_outputs():
    """Imported into a test module: in deterministic mode ``torch.empty`` fills new float tensors with NaN (integer ones with
    their largest value), so the fresh output of a gather (``get_obs_stacked``, ``get_field``, ``solve``) holds a sentinel
    wherever the call wrote nothing."""
    before = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(before)
