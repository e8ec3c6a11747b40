"""CPU tier: the refusals of the C-ABI step and gather entry points, on the emulated library (tests/emu). Every mapdn_step*
entry point refuses a null handle, each required pointer set to NULL and a handle created without a profile store; a
record stride shorter than a row and an unknown field are refused too. Each refusal returns MAPDN_ERR_INVALID with its
mapdn_last_error text and launches nothing. The arguments are passed as ctypes objects, so the calls do not depend on
the argtypes a binding sets."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from conftest import ROOT
from mapdn_b200 import cases

sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
from emu_env import EmuEnv, lib                                     # noqa: E402

INVALID = 1
NULL_ARG, NO_PROFILE = "null argument", "handle was created without a profile store"
SHORT_STRIDE, UNKNOWN_FIELD = "record_stride shorter than a record row", "unknown field"
B = 2

# entry point -> (arguments after the handle, the pointer arguments that must not be NULL)
STEPS = {
    "mapdn_step": ("actions add_noise reward term info obs stream", "actions reward term"),
    "mapdn_step_f32obs": ("actions add_noise reward term info obs32 stream", "actions reward term"),
    "mapdn_step_record": ("actions add_noise reward term info obs record stride stream", "actions reward term"),
    "mapdn_step_host": ("actions add_noise reward term info obs stream", "actions reward term"),
    "mapdn_step_host_f32obs": ("actions add_noise reward term info obs32 stream", "actions reward term"),
    "mapdn_step_host_pinned": ("actions add_noise reward term info obs f32 flag flag stream", "actions reward term"),
    "mapdn_step_host_compact": ("actions add_noise reward term info obs f32 flag flag stream", "actions reward term obs"),
}


@pytest.fixture(scope="module")
def envs():
    net, prof = cases.make_case("case33"), cases.make_profiles("case33", n_days=3)
    env, bare = EmuEnv(net, prof, dict(voltage_barrier_type="l1"), batch=B), EmuEnv(net, None, dict(voltage_barrier_type="l1"), batch=B)
    env.reset()
    d = env.dims
    ng, row = d["n_sgen"], 2 * d["n_sgen"] + 3 * d["n_bus"] + d["n_line"]
    bufs = dict(actions=np.zeros((B, ng)), reward=np.zeros(B), term=np.zeros(B, np.uint8), info=np.zeros((B, 11)),
                obs=np.zeros((B, ng, d["obs_dim"])), obs32=np.zeros((B, ng, d["obs_dim"]), np.float32),
                record=np.zeros((B, row)))
    yield env, bare, bufs, row
    env.close(); bare.close()


def _args(names, bufs, row, null=None):
    out = []
    for k in names.split():
        if k == null or k == "stream":
            out.append(None)
        elif k in bufs:
            out.append(C.c_void_p(bufs[k].ctypes.data))
        elif k == "stride":
            out.append(C.c_int64(row))
        else:                                            # add_noise, obs_is_f32 and the 0 / 1 flags
            out.append(C.c_int32(1 if k == "flag" else 0))
    return out


def _refused(h, fn, args, text):
    L = lib()
    L.mapdn_launch_count.restype = C.c_int64
    L.mapdn_last_error.restype = C.c_char_p
    assert L.mapdn_record_layout(None, None, None) == INVALID       # another text first: the refusal must set its own
    before = L.mapdn_launch_count(h)
    assert getattr(L, fn)(h, *args) == INVALID, fn
    assert L.mapdn_last_error().decode() == text, fn
    assert L.mapdn_launch_count(h) == before, fn


@pytest.mark.parametrize("fn", sorted(STEPS))
def test_step_entry_point_refusals(envs, fn):
    env, bare, bufs, row = envs
    names, required = STEPS[fn]
    _refused(None, fn, _args(names, bufs, row), NULL_ARG)
    for k in required.split():
        _refused(env._h, fn, _args(names, bufs, row, null=k), NULL_ARG)
        _refused(bare._h, fn, _args(names, bufs, row, null=k), NULL_ARG)
    _refused(bare._h, fn, _args(names, bufs, row), NO_PROFILE)


def test_short_record_stride_and_unknown_field_are_refused(envs):
    env, _, bufs, row = envs
    short = _args(STEPS["mapdn_step_record"][0], bufs, row)
    short[7] = C.c_int64(row - 1)
    _refused(env._h, "mapdn_step_record", short, SHORT_STRIDE)
    _refused(env._h, "mapdn_record", [C.c_void_p(bufs["record"].ctypes.data), C.c_int64(row - 1), None], SHORT_STRIDE)
    _refused(env._h, "mapdn_record", [None, C.c_int64(row), None], NULL_ARG)
    out = C.c_void_p(bufs["record"].ctypes.data)
    for field in (-1, 13):
        _refused(env._h, "mapdn_get_field", [C.c_int32(field), out, None], UNKNOWN_FIELD)
    _refused(env._h, "mapdn_get_field", [C.c_int32(0), None, None], NULL_ARG)
    _refused(None, "mapdn_get_field", [C.c_int32(0), out, None], NULL_ARG)
    _refused(env._h, "mapdn_get_obs", [None, None], NULL_ARG)
    _refused(env._h, "mapdn_get_state", [None, None], NULL_ARG)


def test_accepted_calls_count_their_launches(envs):
    """The counter the refusals are checked against does move: one launch per accepted step or gather."""
    env, _, bufs, row = envs
    L = lib()
    L.mapdn_launch_count.restype = C.c_int64
    for fn, args in (("mapdn_step", _args(STEPS["mapdn_step"][0], bufs, row)),
                     ("mapdn_step_record", _args(STEPS["mapdn_step_record"][0], bufs, row)),
                     ("mapdn_record", [C.c_void_p(bufs["record"].ctypes.data), C.c_int64(row), None]),
                     ("mapdn_get_field", [C.c_int32(0), C.c_void_p(bufs["record"].ctypes.data), None])):
        before = L.mapdn_launch_count(env._h)
        assert getattr(L, fn)(env._h, *args) == 0, fn
        assert L.mapdn_launch_count(env._h) == before + 1, fn
