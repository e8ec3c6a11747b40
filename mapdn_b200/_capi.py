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
# get_field columns per env: the dims entry named here; the fields not named have one
FIELD_DIMS = dict(vm="n_bus", va_deg="n_bus", p_bus="n_bus", q_bus="n_bus", p_sgen="n_sgen", q_sgen="n_sgen",
                  line_loss="n_line", p_load="n_load", q_load="n_load")

ABI_VERSION = 2

_pd, _pi, _pb = C.POINTER(C.c_double), C.POINTER(C.c_int32), C.POINTER(C.c_uint8)
_vp, _i32, _i64 = C.c_void_p, C.c_int32, C.c_int64


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


_STEP = [_vp, _vp, _i32] + [_vp] * 5                             # handle, actions, add_noise, four outputs, stream
_STEP_HOST = _STEP[:-1] + [_i32] * 3 + [_vp]                     # obs_is_f32 and two flags before the stream
# every entry point of include/mapdn_b200.h: name -> (argtypes, restype); a mapdn_status is an int32
SIGNATURES = dict(
    mapdn_abi_version=([], _i32), mapdn_last_error=([], C.c_char_p), mapdn_launch_count=([_vp], _i64),
    mapdn_create=([C.POINTER(NetDescC), C.POINTER(ProfileDescC), C.POINTER(CfgC), _i32, C.POINTER(_vp)], _i32),
    mapdn_destroy=([_vp], _i32), mapdn_get_dims=([_vp, C.POINTER(DimsC)], _i32), mapdn_wait=([_vp] * 2, _i32),
    mapdn_reset=([_vp, _vp, _vp, _i32] + [_vp] * 4, _i32), mapdn_step=(_STEP, _i32), mapdn_step_f32obs=(_STEP, _i32),
    mapdn_step_host=(_STEP, _i32), mapdn_step_host_f32obs=(_STEP, _i32), mapdn_step_host_pinned=(_STEP_HOST, _i32),
    mapdn_step_host_compact=(_STEP_HOST, _i32), mapdn_step_record=(_STEP[:-1] + [_vp, _i64, _vp], _i32),
    mapdn_obs_compact_layout=([_vp] * 4, _i32), mapdn_record_layout=([_vp] * 3, _i32),
    mapdn_record=([_vp, _vp, _i64, _vp], _i32), mapdn_set_history=([_vp, _i32], _i32),
    mapdn_step_stacked=(_STEP[:-1] + [_vp, _vp, _i64, _vp], _i32), mapdn_get_obs_stacked=([_vp] * 3, _i32),
    mapdn_step_autoreset=(_STEP[:-1] + [_vp] * 5, _i32),
    mapdn_snapshot_layout=([_vp] * 2, _i32), mapdn_snapshot=([_vp, _vp, _i32, _vp, _vp], _i32),
    mapdn_restore=([_vp, _vp, _i32, _vp, _vp], _i32),
    mapdn_get_obs=([_vp] * 3, _i32), mapdn_get_state=([_vp] * 3, _i32),
    mapdn_get_field=([_vp, _i32, _vp, _vp], _i32), mapdn_solve=([_vp, _i32] + [_vp] * 12, _i32),
    mapdn_droop=([_vp, _i32] + [_vp] * 5 + [C.c_double, C.c_double, _i32] + [_vp] * 5, _i32),
    mapdn_get_ybus_dense=([_vp] * 3, _i32))
EXPORTS = tuple(SIGNATURES)
# tester record row blocks, in the reference tester's key order (utilities/tester.py:26-32); mapdn_record_layout
RECORD_KEYS = ("pv_active", "pv_reactive", "bus_active", "bus_reactive", "bus_voltage", "line_loss")
# env state snapshot row segments, in the order of MAPDN_N_SNAPSHOT (mapdn_snapshot_layout) and their element types
SNAPSHOT_SEGMENTS = ("cur_pl", "cur_ql", "cur_pv", "cur_q", "res_vm", "res_va", "res_p", "res_q", "res_pl", "sum_rewards",
                     "start_row", "steps", "episode", "nr_iters", "hist")
SNAPSHOT_DTYPES = dict(start_row=np.int64, steps=np.int32, episode=np.uint32, nr_iters=np.int32)   # the others: fp64

_lib: Optional[C.CDLL] = None


class MapdnError(RuntimeError):
    pass


def bind(L: C.CDLL, skip_missing: bool = False) -> C.CDLL:
    """Sets argtypes and restype of every entry point in ``L``; ``skip_missing``: pass over the symbols ``L`` lacks."""
    for name, (argtypes, restype) in SIGNATURES.items():
        if hasattr(L, name) or not skip_missing:
            fn = getattr(L, name)
            fn.argtypes, fn.restype = argtypes, restype
    return L


def lib() -> C.CDLL:
    """Load ``libmapdn_b200.so`` (built by ``python -m mapdn_b200.build``). Fails loudly."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MapdnError(f"{LIB_PATH} not found - build it with `python -m mapdn_b200.build` "
                         "(there is no CPU fallback)")
    # MAPDN_B200_LIB: A/B runs against libraries built from older commits, which may lack the newer entry points
    L = bind(C.CDLL(LIB_PATH), skip_missing=bool(os.environ.get("MAPDN_B200_LIB")))
    if L.mapdn_abi_version() != ABI_VERSION:
        raise MapdnError("ABI version mismatch between _capi.py and libmapdn_b200.so")
    _lib = L
    return L


def check(status: int, L: C.CDLL):
    """Raises MapdnError with the error text of ``L``, the library that returned ``status``, unless it is 0."""
    if status != 0:
        raise MapdnError(f"mapdn status {status}: {L.mapdn_last_error().decode()}")


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


def make_cfg(args: dict, batch: int, env_id_offset=0, lanes_per_env=0, tol=0.0, max_iter=0) -> CfgC:
    """The ``mapdn_cfg`` of ``batch`` envs from the reference's ``env_args`` (every key of ``DEFAULT_ENV_ARGS``)."""
    a, qw, lw = args, args["q_weight"], args["line_weight"]
    return CfgC(batch=int(batch), barrier=BARRIERS[a["voltage_barrier_type"]],
                voltage_weight=float(a["voltage_weight"]), q_weight=float(qw if qw is not None else 0.0),
                line_weight=float(lw or 0.0), use_line_weight=int(lw is not None), v_upper=float(a["v_upper"]),
                v_lower=float(a["v_lower"]), episode_limit=int(a["episode_limit"]),
                action_low=float(-a["action_scale"] + a["action_bias"]),
                action_high=float(a["action_scale"] + a["action_bias"]), reset_action=int(bool(a["reset_action"])),
                seed=int(a["seed"]) & 0xFFFFFFFFFFFFFFFF, env_id_offset=int(env_id_offset), tol=float(tol),
                max_iter=int(max_iter), lanes_per_env=int(lanes_per_env),
                state_space_mask=sum(STATE_SPACE_BITS[k] for k in set(a["state_space"])))


def make_profile_desc(prof: ProfileDesc):
    keep = [prof.pv, prof.load_p, prof.load_q,
            np.ascontiguousarray(prof.pv_std), np.ascontiguousarray(prof.load_p_std),
            np.ascontiguousarray(prof.load_q_std), np.ascontiguousarray(prof.s_max)]
    d = ProfileDescC(prof.n_rows, prof.steps_per_hour, prof.n_days, *[_p(a, _pd) for a in keep])
    return d, keep
