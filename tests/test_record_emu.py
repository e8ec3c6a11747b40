"""CPU tier for the tester records (mapdn_record_layout / mapdn_record / mapdn_step_record), on the kernel source compiled
for the CPU SIMT emulation (tests/emu). The fused rows written by the step kernel's epilogue must equal the gather
launch and the six mapdn_get_field columns BIT FOR BIT, and the step itself must be the one mapdn_step takes."""
import os
import re
import sys

import numpy as np
import pytest
import torch

import geometry_cases as GC
from conftest import ROOT
from mapdn_b200 import _capi, cases
from mapdn_b200._capi import MapdnError

sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
from emu_env import make_env, nan_filled_outputs                    # noqa: E402,F401  (autouse fixture)

FIELD_ORDER = ("p_sgen", "q_sgen", "p_bus", "q_bus", "vm", "line_loss")     # = RECORD_KEYS, getter by getter


def _fields(env):
    return np.concatenate([env.get_field(k).numpy() for k in FIELD_ORDER], axis=1)


def _run(net, prof, args, batch, lanes, start, n_steps, noise, expect_diverged=False):
    plain = make_env(net, prof, args, batch=batch, lanes_per_env=lanes)
    fused = make_env(net, prof, args, batch=batch, lanes_per_env=lanes)
    off, R = [o for o, _ in fused.record_slices.values()], fused.record_len
    ng, n, nl = net.n_sgen, net.n_bus, fused.dims["n_line"]
    assert off == [0, ng, 2 * ng, 2 * ng + n, 2 * ng + 2 * n, 2 * ng + 3 * n] and R == 2 * ng + 3 * n + nl
    buf = torch.full((batch, n_steps + 1, R + 3), np.nan, dtype=torch.float64)   # [B, T+1, R] rows with a row stride != R
    for e in (plain, fused):
        e.reset(None if start is None else torch.from_numpy(start), add_noise=start is None)
    assert np.array_equal(plain.obs.numpy(), fused.obs.numpy())
    fused.record(buf[:, 0, :R])
    assert np.array_equal(buf[:, 0, :R].numpy(), _fields(fused))
    rng = np.random.default_rng(lanes)
    scale = float(args.get("action_scale", 0.8))
    diverged = False
    for t in range(n_steps):
        a = torch.from_numpy(rng.uniform(-scale, scale, (batch, ng)))
        r0, t0, i0 = [x.numpy().copy() for x in plain.step(a, add_noise=noise)]
        r1, t1, i1 = [x.numpy() for x in fused.step(a, add_noise=noise, record=buf[:, t + 1, :R])]
        assert (np.array_equal(r0, r1) and np.array_equal(t0, t1) and np.array_equal(i0, i1)
                and np.array_equal(plain.obs.numpy(), fused.obs.numpy()))
        row = buf[:, t + 1, :R].numpy()
        assert np.array_equal(row, _fields(fused)), t
        assert np.array_equal(row, _fields(plain)), t
        gathered = torch.full((batch, R), np.nan, dtype=torch.float64)
        assert np.array_equal(fused.record(gathered).numpy(), row), t
        diverged |= bool(np.any(i1[:, 10] == 1.0))
    assert torch.all(buf[:, :, R:].isnan())                        # nothing past the row
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
    net, prof = GC.overload(cases.make_case("case33"), cases.make_profiles("case33", n_days=4))
    start = np.array([[1, 0, 0], [0, 2, 17], [1, 5, 3], [2, 1, 9]], np.int32)
    _run(net, prof, dict(voltage_barrier_type="bowl", seed=4), batch=4, lanes=lanes, start=start, n_steps=4, noise=False,
         expect_diverged=True)


def test_record_on_the_dense_meshed_fallback():
    net, prof = GC.mesh4()
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
    env = make_env(net, prof, None, batch=1)
    off, R = [o for o, _ in env.record_slices.values()], env.record_len
    widths = [net.n_sgen, net.n_sgen, net.n_bus, net.n_bus, net.n_bus, env.dims["n_line"]]
    assert off == list(np.cumsum([0] + widths[:-1])) and R == sum(widths)
    assert [n for _, n in env.record_slices.values()] == widths and list(env.record_slices) == list(_capi.RECORD_KEYS)
    bad = torch.zeros(1, R - 1, dtype=torch.float64)
    with pytest.raises(ValueError, match="record"):                  # the binding refuses a short row before the call
        env.record(bad)
    with pytest.raises(MapdnError, match="record_stride"):           # and so does the C-ABI
        _capi.check(env._L.mapdn_record(env._h, bad.data_ptr(), R - 1, None), env._L)
    env.close()
