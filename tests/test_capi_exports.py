"""The C-ABI library builds for sm_90a (nvcc cross-compiles on the CPU box), loads, and exports
every entry point declared in include/mapdn_b200.h. No compute calls - no GPU needed."""
import ctypes
import os
import re

from conftest import ROOT


def declared_functions():
    src = open(os.path.join(ROOT, "include", "mapdn_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(mapdn_[a-z_0-9]+)\s*\(", src)))


def test_header_declares_the_boundary():
    fns = declared_functions()
    for must in ("mapdn_create", "mapdn_destroy", "mapdn_reset", "mapdn_step", "mapdn_step_host", "mapdn_get_obs",
                 "mapdn_get_state", "mapdn_get_field", "mapdn_solve"):
        assert must in fns


def test_library_exports_every_declared_symbol(built_lib):
    L = ctypes.CDLL(built_lib)
    for fn in declared_functions():
        assert hasattr(L, fn), f"{fn} declared in the header but not exported"
    L.mapdn_abi_version.restype = ctypes.c_int32
    assert L.mapdn_abi_version() == 2


def test_binding_covers_the_header(built_lib):
    from mapdn_b200 import _capi
    assert sorted(_capi.EXPORTS) == declared_functions()
    assert _capi.lib().mapdn_abi_version() == _capi.ABI_VERSION == 2


def test_struct_layouts_match_header():
    """sizeof of the ctypes mirrors == sizeof computed by the C compiler for the header structs."""
    import subprocess, tempfile
    from mapdn_b200 import _capi
    prog = r'''
#include <stdio.h>
#include "mapdn_b200.h"
int main(void){ printf("%zu %zu %zu %zu\n", sizeof(mapdn_net_desc), sizeof(mapdn_profile_desc), sizeof(mapdn_cfg), sizeof(mapdn_dims)); return 0; }
'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "s.c")
        open(c, "w").write(prog)
        exe = os.path.join(d, "s")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        sizes = [int(x) for x in subprocess.check_output([exe]).split()]
    assert sizes == [ctypes.sizeof(_capi.NetDescC), ctypes.sizeof(_capi.ProfileDescC), ctypes.sizeof(_capi.CfgC),
                     ctypes.sizeof(_capi.DimsC)]


def test_no_oracle_import_in_product():
    """The product never routes through the oracle (or any CPU fallback)."""
    pkg = os.path.join(ROOT, "mapdn_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M), f


def test_create_validates_arguments_without_touching_the_gpu(built_lib):
    """Argument checks of mapdn_create run before any CUDA call: bad descriptions are refused with
    MAPDN_ERR_INVALID (1) and a message, also on a box without a GPU."""
    import ctypes as C
    import numpy as np
    from mapdn_b200 import _capi, cases
    L = _capi.lib()
    net = cases.case33()
    cfg = _capi.CfgC(batch=4, barrier=0, voltage_weight=1.0, q_weight=0.1, v_upper=1.05, v_lower=0.95, episode_limit=240,
                     action_low=-0.8, action_high=0.8, reset_action=1)
    h = C.c_void_p()

    def create(nd, c):
        return L.mapdn_create(C.byref(nd), None, C.byref(c), 0, C.byref(h))

    nd, keep = _capi.make_net_desc(net)
    nd.n_bus = 1
    assert create(nd, cfg) == 1 and b"n_bus" in L.mapdn_last_error()
    nd, keep = _capi.make_net_desc(net)
    nd.slack_bus = 99
    assert create(nd, cfg) == 1 and b"slack_bus" in L.mapdn_last_error()
    nd, keep = _capi.make_net_desc(net)
    bad = net.br_to.copy(); bad[3] = 1000
    nd.br_to = bad.ctypes.data_as(C.POINTER(C.c_int32))
    assert create(nd, cfg) == 1 and b"branch endpoint" in L.mapdn_last_error()
    nd, keep = _capi.make_net_desc(net)
    cfg2 = _capi.CfgC.from_buffer_copy(cfg); cfg2.barrier = 9
    assert create(nd, cfg2) == 1 and b"barrier" in L.mapdn_last_error()
    cfg3 = _capi.CfgC.from_buffer_copy(cfg); cfg3.lanes_per_env = 5
    assert create(nd, cfg3) == 1 and b"lanes_per_env" in L.mapdn_last_error()
    cfg4 = _capi.CfgC.from_buffer_copy(cfg); cfg4.batch = 0
    assert create(nd, cfg4) == 1
    assert L.mapdn_create(None, None, C.byref(cfg), 0, C.byref(h)) == 1
    assert not h.value
    # null handles are refused, not dereferenced
    assert L.mapdn_step(None, None, 0, None, None, None, None, None) == 1
    assert L.mapdn_destroy(None) == 0


def test_product_library_is_the_device_build_not_the_cpu_emulation(built_lib):
    """The shipped library is the nvcc build: it carries sm_90a device code and none of the emulation's symbols; the
    product's loader and build script know nothing of tests/emu (the CPU SIMT emulation is test infrastructure)."""
    import subprocess
    from mapdn_b200 import build
    assert "-DMAPDN_HOST_EMU" not in " ".join(build.NVCC_FLAGS) and any("sm_90a" in f for f in build.NVCC_FLAGS)
    syms = subprocess.run(["nm", "-DC", built_lib], capture_output=True, text=True).stdout
    assert "emu::" not in syms and "launch_impl" not in syms
    elf = subprocess.run(["cuobjdump", "-lelf", built_lib], capture_output=True, text=True)
    if elf.returncode == 0:
        assert "sm_90a" in elf.stdout
    for f in ("_capi.py", "build.py", "env.py"):
        src = open(os.path.join(ROOT, "mapdn_b200", f)).read()
        assert "emu" not in src.replace("enumerate", "") or f == "env.py" and "tests/emu" not in src
