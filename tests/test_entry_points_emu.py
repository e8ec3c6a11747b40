"""CPU tier: the refusals of the C-ABI step and gather entry points, on the emulated library (tests/emu). Every mapdn_step*
entry point refuses a null handle, each required pointer set to NULL and a handle created without a profile store; a
record stride shorter than a row and an unknown field are refused too. Each refusal returns MAPDN_ERR_INVALID with its
mapdn_last_error text and launches nothing. The arguments are passed as ctypes objects, so the calls do not depend on
the argtypes a binding sets.

mapdn_create refuses a bad description with its status, its text and a null handle; when several conditions hold, the
one checked first decides."""
import copy
import ctypes as C
import os
import sys

import numpy as np
import pytest

import geometry_cases as GC
from conftest import ROOT
from mapdn_b200 import _capi, cases
from mapdn_b200.env import DEFAULT_ENV_ARGS
from mapdn_b200.network import NetDesc

sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
from emu_env import lib, make_env                                   # noqa: E402

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
    env, bare = make_env(net, prof, dict(voltage_barrier_type="l1"), batch=B), make_env(net, None, dict(voltage_barrier_type="l1"), batch=B)
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


# ---- mapdn_create ----
TOPOLOGY, UNSUPPORTED = 3, 4
BAD_LANES = "lanes_per_env must be 0, 4, 8, 16, 32, 64 or 128"
MESHED_257 = ("network is meshed (1 loop-closing branches) and has more than 256 PQ buses: the dense fallback solver only "
              "covers small meshed feeders")


def _case33(**changes):
    """case33 with elements of its branch arrays overwritten (name=(index, value)), also with what NetDesc refuses."""
    net = copy.deepcopy(cases.make_case("case33"))
    for k, (i, v) in changes.items():
        getattr(net, k)[i] = v
    return net


def _wide_hub(n_children):
    """One PQ bus behind the slack with n_children leaves."""
    n = n_children + 2
    return NetDesc(base_mva=1.0, n_bus=n, slack_bus=0, slack_vm=1.0, br_from=[0] + [1] * n_children, br_to=list(range(1, n)),
                   br_r=[0.01] * (n - 1), br_x=[0.01] * (n - 1), load_bus=np.arange(1, n), sgen_bus=[2], sgen_zone=[1],
                   bus_zone=[0] + [1] * (n - 1), name="wide_hub")


# what to create -> (status, text). net: a NetDesc; desc / prof / cfg: fields of the C structs set after they are filled in
# (None: a NULL pointer); no_profile: create without a profile store
CREATE_REFUSALS = {
    "null_net": (dict(null="net"), INVALID, NULL_ARG),
    "null_cfg": (dict(null="cfg"), INVALID, NULL_ARG),
    "null_out": (dict(null="out"), INVALID, NULL_ARG),
    "one_bus": (dict(desc=dict(n_bus=1)), INVALID, "n_bus must be in [2, 65000]"),
    "too_many_buses": (dict(desc=dict(n_bus=65001)), INVALID, "n_bus must be in [2, 65000]"),
    "no_sgen": (dict(desc=dict(n_sgen=0)), INVALID, "need >=1 branch and >=1 sgen"),
    "batch_0": (dict(cfg=dict(batch=0)), INVALID, "batch must be >= 1"),
    "missing_array": (dict(desc=dict(br_x=None)), INVALID, "missing required network array"),
    "slack_out_of_range": (dict(desc=dict(slack_bus=33)), INVALID, "slack_bus out of range"),
    "base_mva_0": (dict(desc=dict(base_mva=0.0)), INVALID, "base_mva must be positive"),
    "barrier_9": (dict(cfg=dict(barrier=9)), INVALID, "unknown voltage barrier"),
    "lanes_5": (dict(cfg=dict(lanes_per_env=5)), INVALID, BAD_LANES),
    "lanes_256": (dict(cfg=dict(lanes_per_env=256)), INVALID, BAD_LANES),
    "branch_endpoint": (dict(net=_case33(br_to=(3, 1000))), INVALID, "branch endpoint out of range"),
    "self_loop": (dict(net=_case33(br_to=(3, 3))), INVALID, "branch endpoint out of range"),
    "incomplete_profile": (dict(prof=dict(pv_std=None)), INVALID, "incomplete profile description"),
    "one_profile_row": (dict(prof=dict(n_rows=1)), INVALID, "incomplete profile description"),
    "zero_impedance": (dict(net=_case33(br_r=(5, 0.0), br_x=(5, 0.0))), INVALID, "zero-impedance branch"),
    "unreachable_1": (dict(net=_case33(br_status=(31, 0))), TOPOLOGY,
                      "network is not connected to the slack bus (1 unreachable buses)"),
    "unreachable_4": (dict(net=_case33(br_status=(28, 0))), TOPOLOGY,
                      "network is not connected to the slack bus (4 unreachable buses)"),
    "meshed_257": (dict(net=GC.meshed_chain(257), no_profile=True), TOPOLOGY, MESHED_257),
    "children_258": (dict(net=_wide_hub(258), no_profile=True), UNSUPPORTED, "a bus with more than 257 children"),
    "short_store": (dict(prof=dict(n_days=1)), INVALID, "profile store shorter than one episode"),
    "fewer_rows_than_days": (dict(prof=dict(n_days=10)), INVALID, "profile store shorter than n_days claims"),
    # several conditions at once: the argument checks, then zero impedance, then connectivity, then the profile store
    "lanes_before_zero_impedance": (dict(net=_case33(br_r=(5, 0.0), br_x=(5, 0.0)), cfg=dict(lanes_per_env=5)), INVALID, BAD_LANES),
    "profile_description_before_topology": (dict(net=_case33(br_status=(31, 0)), prof=dict(s_max=None)), INVALID,
                                            "incomplete profile description"),
    "zero_impedance_before_unreachable": (dict(net=_case33(br_r=(5, 0.0), br_x=(5, 0.0), br_status=(31, 0))), INVALID,
                                          "zero-impedance branch"),
    "unreachable_before_short_store": (dict(net=_case33(br_status=(31, 0)), prof=dict(n_days=1)), TOPOLOGY,
                                       "network is not connected to the slack bus (1 unreachable buses)"),
}


@pytest.mark.parametrize("case", sorted(CREATE_REFUSALS))
def test_create_refusals(case):
    what, status, text = CREATE_REFUSALS[case]
    L = lib()
    net = what.get("net") or cases.make_case("case33")
    nd, keep_net = _capi.make_net_desc(net)
    pd_, keep_prof = _capi.make_profile_desc(cases.make_profiles("case33", n_days=3))
    cfg = _capi.make_cfg(dict(DEFAULT_ENV_ARGS), B)
    for struct, key in ((nd, "desc"), (pd_, "prof"), (cfg, "cfg")):
        for k, v in what.get(key, {}).items():
            setattr(struct, k, v)
    h = C.c_void_p(0xDEAD)                                           # create clears it before it looks at anything else
    null = what.get("null")
    assert L.mapdn_record_layout(None, None, None) == INVALID       # another text first: the refusal must set its own
    st = L.mapdn_create(None if null == "net" else C.byref(nd), None if what.get("no_profile") else C.byref(pd_),
                        None if null == "cfg" else C.byref(cfg), 0, None if null == "out" else C.byref(h))
    assert st == status, L.mapdn_last_error()
    assert L.mapdn_last_error().decode() == text
    assert null in ("net", "cfg", "out") or not h.value


def test_create_launches_the_two_ybus_kernels():
    env = make_env(cases.make_case("case33"), None, batch=B)
    assert env.launch_count == 2
    env.close()
