"""ctypes binding of the C-ABI in ``include/mapdn_b200.h`` (``libmapdn_b200.so``).

The library is plain CUDA C++ with ``extern "C"`` entry points; PyTorch is used here only to
own device memory and streams (tensors are passed as raw ``data_ptr()``). There is no CPU
fallback: if the library is missing or cannot be loaded the import of :func:`lib` raises.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import numpy as np

from .network import NetDesc, ProfileDesc

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("MAPDN_B200_LIB") or os.path.join(_HERE, "libmapdn_b200.so")   # env override: kernel experiments

STATE_SPACE_BITS = {"demand": 1, "pv": 2, "reactive": 4, "vm_pu": 8, "va_degree": 16}
BARRIERS = {"l1": 0, "l2": 1, "bowl": 2, "bump": 3, "courant_beltrami": 4}
INFO_KEYS = ("percentage_of_v_out_of_control", "percentage_of_lower_than_lower_v",
             "percentage_of_higher_than_upper_v", "totally_controllable_ratio",
             "average_voltage_deviation", "average_voltage", "max_voltage_drop_deviation",
             "max_voltage_rise_deviation", "total_line_loss", "q_loss", "destroy")
FIELDS = dict(vm=0, va_deg=1, p_bus=2, q_bus=3, p_sgen=4, q_sgen=5, line_loss=6, p_load=7, q_load=8,
              sum_rewards=9, steps=10, start_row=11, nr_iters=12)

ABI_VERSION = 2

_pd = C.POINTER(C.c_double)
_pi = C.POINTER(C.c_int32)
_pb = C.POINTER(C.c_uint8)


class NetDescC(C.Structure):
    _fields_ = [("n_bus", C.c_int32), ("n_branch", C.c_int32), ("n_load", C.c_int32), ("n_sgen", C.c_int32),
                ("base_mva", C.c_double), ("slack_bus", C.c_int32), ("slack_vm", C.c_double),
                ("slack_va_deg", C.c_double), ("vm_init", C.c_double),
                ("br_from", _pi), ("br_to", _pi), ("br_r", _pd), ("br_x", _pd), ("br_b", _pd), ("br_g", _pd),
                ("br_tap", _pd), ("br_shift_deg", _pd), ("br_status", _pb), ("br_is_line", _pb),
                ("bus_gs_mw", _pd), ("bus_bs_mvar", _pd), ("bus_zone", _pi),
                ("load_bus", _pi), ("load_scaling", _pd),
                ("sgen_bus", _pi), ("sgen_zone", _pi), ("sgen_scaling", _pd)]


class ProfileDescC(C.Structure):
    _fields_ = [("n_rows", C.c_int64), ("steps_per_hour", C.c_int32), ("n_days", C.c_int32),
                ("pv", _pd), ("load_p", _pd), ("load_q", _pd),
                ("pv_std", _pd), ("load_p_std", _pd), ("load_q_std", _pd), ("s_max", _pd)]


class CfgC(C.Structure):
    _fields_ = [("batch", C.c_int32), ("barrier", C.c_int32), ("voltage_weight", C.c_double),
                ("q_weight", C.c_double), ("line_weight", C.c_double), ("use_line_weight", C.c_int32),
                ("v_upper", C.c_double), ("v_lower", C.c_double), ("episode_limit", C.c_int32),
                ("action_low", C.c_double), ("action_high", C.c_double), ("reset_action", C.c_int32),
                ("seed", C.c_uint64), ("env_id_offset", C.c_int64), ("tol", C.c_double),
                ("max_iter", C.c_int32), ("lanes_per_env", C.c_int32), ("state_space_mask", C.c_int32)]


class DimsC(C.Structure):
    _fields_ = [(k, C.c_int32) for k in
                ("batch", "n_bus", "n_branch", "n_line", "n_load", "n_sgen", "n_agents", "n_actions", "obs_dim",
                 "state_dim", "n_info", "lanes_per_env", "envs_per_block", "smem_bytes", "n_levels")] + [
        ("algorithmic_bytes_per_env_step", C.c_int64)]


EXPORTS = ("mapdn_abi_version", "mapdn_last_error", "mapdn_create", "mapdn_destroy", "mapdn_get_dims",
           "mapdn_reset", "mapdn_step", "mapdn_step_host", "mapdn_step_f32obs", "mapdn_step_host_f32obs", "mapdn_step_host_pinned", "mapdn_wait", "mapdn_obs_compact_layout", "mapdn_step_host_compact", "mapdn_get_obs", "mapdn_get_state",
           "mapdn_get_field", "mapdn_solve", "mapdn_droop", "mapdn_get_ybus_dense", "mapdn_launch_count",
           "mapdn_record_layout", "mapdn_record", "mapdn_step_record")
# tester record row blocks, in the reference tester's key order (utilities/tester.py:26-32); mapdn_record_layout
RECORD_KEYS = ("pv_active", "pv_reactive", "bus_active", "bus_reactive", "bus_voltage", "line_loss")

_lib: Optional[C.CDLL] = None


class MapdnError(RuntimeError):
    pass


def lib() -> C.CDLL:
    """Load ``libmapdn_b200.so`` (built by ``python -m mapdn_b200.build``). Fails loudly."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MapdnError(f"{LIB_PATH} not found - build it with `python -m mapdn_b200.build` "
                         "(there is no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    vp = C.c_void_p
    L.mapdn_abi_version.restype = C.c_int32
    L.mapdn_last_error.restype = C.c_char_p
    L.mapdn_create.argtypes = [C.POINTER(NetDescC), C.POINTER(ProfileDescC), C.POINTER(CfgC), C.c_int32,
                               C.POINTER(vp)]
    L.mapdn_destroy.argtypes = [vp]
    L.mapdn_get_dims.argtypes = [vp, C.POINTER(DimsC)]
    L.mapdn_reset.argtypes = [vp, vp, vp, C.c_int32, vp, vp, vp, vp]
    L.mapdn_step.argtypes = [vp, vp, C.c_int32, vp, vp, vp, vp, vp]
    L.mapdn_step_host.argtypes = [vp, vp, C.c_int32, vp, vp, vp, vp, vp]
    L.mapdn_step_f32obs.argtypes = [vp, vp, C.c_int32, vp, vp, vp, vp, vp]
    L.mapdn_step_host_f32obs.argtypes = [vp, vp, C.c_int32, vp, vp, vp, vp, vp]
    dev_override = bool(os.environ.get("MAPDN_B200_LIB"))       # A/B runs against libraries built from older commits
    try:
        L.mapdn_step_host_pinned.argtypes = [vp, vp, C.c_int32, vp, vp, vp, vp, C.c_int32, C.c_int32, C.c_int32, vp]
        L.mapdn_wait.argtypes = [vp, vp]
        L.mapdn_droop.argtypes = [vp, C.c_int32] + [vp] * 5 + [C.c_double, C.c_double, C.c_int32] + [vp] * 5
        L.mapdn_obs_compact_layout.argtypes = [vp, vp, vp, vp]
        L.mapdn_step_host_compact.argtypes = [vp, vp, C.c_int32, vp, vp, vp, vp, C.c_int32, C.c_int32, C.c_int32, vp]
        L.mapdn_record_layout.argtypes = [vp, vp, vp]
        L.mapdn_record.argtypes = [vp, vp, C.c_int64, vp]
        L.mapdn_step_record.argtypes = [vp, vp, C.c_int32, vp, vp, vp, vp, vp, C.c_int64, vp]
    except AttributeError:
        if not dev_override:
            raise
    L.mapdn_get_obs.argtypes = [vp, vp, vp]
    L.mapdn_get_state.argtypes = [vp, vp, vp]
    L.mapdn_get_field.argtypes = [vp, C.c_int32, vp, vp]
    L.mapdn_solve.argtypes = [vp, C.c_int32] + [vp] * 11 + [vp]
    L.mapdn_get_ybus_dense.argtypes = [vp, vp, vp]
    L.mapdn_launch_count.argtypes = [vp]
    L.mapdn_launch_count.restype = C.c_int64
    for name in EXPORTS:
        if dev_override and not hasattr(L, name):
            continue
        fn = getattr(L, name)
        if fn.restype is C.c_int and name not in ("mapdn_abi_version",):
            fn.restype = C.c_int32
    if L.mapdn_abi_version() != ABI_VERSION:
        raise MapdnError("ABI version mismatch between _capi.py and libmapdn_b200.so")
    _lib = L
    return L


def check(status: int):
    if status != 0:
        raise MapdnError(f"mapdn status {status}: {lib().mapdn_last_error().decode()}")


def _p(a: Optional[np.ndarray], typ):
    return None if a is None else a.ctypes.data_as(typ)


def make_net_desc(net: NetDesc):
    """(struct, keepalive list) for a :class:`NetDesc`."""
    keep = [net.br_from, net.br_to, net.br_r, net.br_x, net.br_b, net.br_g, net.br_tap, net.br_shift,
            net.br_status, net.br_is_line, net.bus_gs, net.bus_bs, net.bus_zone, net.load_bus,
            net.load_scaling, net.sgen_bus, net.sgen_zone, net.sgen_scaling]
    d = NetDescC(net.n_bus, net.n_branch, net.n_load, net.n_sgen, net.base_mva, net.slack_bus, net.slack_vm,
                 net.slack_va_deg, net.vm_init,
                 _p(net.br_from, _pi), _p(net.br_to, _pi), _p(net.br_r, _pd), _p(net.br_x, _pd),
                 _p(net.br_b, _pd), _p(net.br_g, _pd), _p(net.br_tap, _pd), _p(net.br_shift, _pd),
                 _p(net.br_status, _pb), _p(net.br_is_line, _pb), _p(net.bus_gs, _pd), _p(net.bus_bs, _pd),
                 _p(net.bus_zone, _pi), _p(net.load_bus, _pi), _p(net.load_scaling, _pd),
                 _p(net.sgen_bus, _pi), _p(net.sgen_zone, _pi), _p(net.sgen_scaling, _pd))
    return d, keep


def make_profile_desc(prof: ProfileDesc):
    keep = [prof.pv, prof.load_p, prof.load_q,
            np.ascontiguousarray(prof.pv_std), np.ascontiguousarray(prof.load_p_std),
            np.ascontiguousarray(prof.load_q_std), np.ascontiguousarray(prof.s_max)]
    d = ProfileDescC(prof.n_rows, prof.steps_per_hour, prof.n_days, *[_p(a, _pd) for a in keep])
    return d, keep
