"""CPU tier for the tester records (mapdn_record_layout / mapdn_record / mapdn_step_record), on the kernel source compiled
for the CPU SIMT emulation (tests/emu). The fused rows written by the step kernel's epilogue must equal the gather
launch and the six mapdn_get_field columns BIT FOR BIT, and the step itself must be the one mapdn_step takes."""
import os
import re
import sys

import numpy as np
import pytest

from conftest import ROOT
from mapdn_b200 import _capi, cases
from mapdn_b200.network import NetDesc, ProfileDesc

sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
from emu_env import EmuEnv                                          # noqa: E402

FIELD_ORDER = ("p_sgen", "q_sgen", "p_bus", "q_bus", "vm", "line_loss")     # = RECORD_KEYS, getter by getter


def _fields(env):
    return np.concatenate([env.get_field(k) for k in FIELD_ORDER], axis=1)


def _overload(name):
    """The named case with a profile whose rows 60..459 carry a demand the feeder cannot serve (divergence branch)."""
    net, prof = cases.make_case(name), cases.make_profiles(name, n_days=4)
    lp = prof.load_p.copy(); lp[60:460] *= 60.0
    return net, ProfileDesc(pv=prof.pv, load_p=lp, load_q=prof.load_q, steps_per_hour=prof.steps_per_hour, n_days=prof.n_days)


def _mesh():
    z = np.array([0.02 + 0.04j, 0.01 + 0.03j, 0.0125 + 0.025j, 0.015 + 0.03j])
    net = NetDesc(base_mva=100.0, n_bus=4, slack_bus=0, slack_vm=1.03, br_from=np.array([0, 0, 1, 2]), br_to=np.array([1, 2, 2, 3]),
                  br_r=z.real, br_x=z.imag, load_bus=np.array([1, 2, 3]), sgen_bus=np.array([2, 3]), sgen_zone=np.array([1, 1]),
                  bus_zone=np.array([0, 1, 1, 1]), name="mesh4")
    rng = np.random.default_rng(3)
    T = 3 * 24 * 20 + 1
    prof = ProfileDesc(pv=rng.uniform(0, 40, (T, 2)), load_p=rng.uniform(60, 180, (T, 3)), load_q=rng.uniform(10, 60, (T, 3)),
                       steps_per_hour=20)
    return net, prof


def _run(net, prof, args, batch, lanes, start, n_steps, noise, expect_diverged=False):
    plain = EmuEnv(net, prof, args, batch=batch, lanes_per_env=lanes)
    fused = EmuEnv(net, prof, args, batch=batch, lanes_per_env=lanes)
    off, R = fused.record_layout()
    ng, n, nl = net.n_sgen, net.n_bus, fused.dims["n_line"]
    assert off == [0, ng, 2 * ng, 2 * ng + n, 2 * ng + 2 * n, 2 * ng + 3 * n] and R == 2 * ng + 3 * n + nl
    buf = np.full((batch, n_steps + 1, R + 3), np.nan)            # [B, T+1, R] rows with a row stride != R
    for e in (plain, fused):
        e.reset(start, add_noise=start is None)
    assert np.array_equal(plain.obs, fused.obs)
    fused.record(buf[:, 0, :R])
    assert np.array_equal(buf[:, 0, :R], _fields(fused))
    rng = np.random.default_rng(lanes)
    scale = float(args.get("action_scale", 0.8))
    diverged = False
    for t in range(n_steps):
        a = rng.uniform(-scale, scale, (batch, ng))
        r0, t0, i0 = [x.copy() for x in plain.step(a, add_noise=noise)]
        r1, t1, i1 = fused.step_record(a, buf[:, t + 1, :R], add_noise=noise)
        assert np.array_equal(r0, r1) and np.array_equal(t0, t1) and np.array_equal(i0, i1) and np.array_equal(plain.obs, fused.obs)
        row = buf[:, t + 1, :R]
        assert np.array_equal(row, _fields(fused)), t
        assert np.array_equal(row, _fields(plain)), t
        gathered = np.full((batch, R), np.nan)
        assert np.array_equal(fused.record(gathered), row), t
        diverged |= bool(np.any(i1[:, 10] == 1.0))
    assert np.all(np.isnan(buf[:, :, R:]))                          # nothing past the row
    assert diverged == expect_diverged
    plain.close(); fused.close()


@pytest.mark.parametrize("name,lanes", [("case33", 8), ("case33", 32), ("case141", 32), ("case141", 64), ("case322", 64)])
def test_fused_record_rows_equal_gather_and_get_field(name, lanes):
    """Every lane count in use (8 / 32 / 64: sub-warp groups, a whole warp, a two-warp group), helper warps drawing noisy
    next rows, sampled resets."""
    net, prof = cases.make_case(name), cases.make_profiles(name, n_days=3)
    _run(net, prof, dict(voltage_barrier_type="l1", seed=3, action_scale=cases.SCENARIOS[name]["action_scale"]),
         batch=3, lanes=lanes, start=None, n_steps=2 if name == "case322" else 3, noise=True)


@pytest.mark.parametrize("lanes", [8, 32, 64])
def test_record_of_a_diverged_step_is_the_previous_result(lanes):
    """Env 1 walks into rows the feeder cannot serve: its step diverges (reference :188-196) and its record row reports the
    previous power flow, as mapdn_get_field does; the other envs of its warp carry on."""
    net, prof = _overload("case33")
    start = np.array([[1, 0, 0], [0, 2, 17], [1, 5, 3], [2, 1, 9]], np.int32)
    _run(net, prof, dict(voltage_barrier_type="bowl", seed=4), batch=4, lanes=lanes, start=start, n_steps=4, noise=False,
         expect_diverged=True)


def test_record_on_the_dense_meshed_fallback():
    net, prof = _mesh()
    start = np.array([[0, 3, 1], [1, 12, 7]], np.int32)
    _run(net, prof, dict(voltage_barrier_type="l2", seed=2, episode_limit=48), batch=2, lanes=0, start=start, n_steps=3,
         noise=True)


def test_record_layout_matches_the_header():
    """MAPDN_N_RECORD and the key order documented in include/mapdn_b200.h agree with the binding and with the layout call."""
    src = open(os.path.join(ROOT, "include", "mapdn_b200.h")).read()
    assert int(re.search(r"#define\s+MAPDN_N_RECORD\s+(\d+)", src).group(1)) == len(_capi.RECORD_KEYS) == 6
    doc = re.search(r"\[(pv_active[^\]]*)\]", src).group(1)
    assert [tok.split()[0] for tok in doc.split("|")] == list(_capi.RECORD_KEYS)
    net, prof = cases.make_case("case141"), cases.make_profiles("case141", n_days=3)
    env = EmuEnv(net, prof, None, batch=1)
    off, R = env.record_layout()
    widths = [net.n_sgen, net.n_sgen, net.n_bus, net.n_bus, net.n_bus, env.dims["n_line"]]
    assert off == list(np.cumsum([0] + widths[:-1])) and R == sum(widths)
    bad = np.zeros((1, R - 1))
    with pytest.raises(RuntimeError, match="record_stride"):
        env.record(bad)
    env.close()
