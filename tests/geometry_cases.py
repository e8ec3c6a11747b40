"""Shared by the launch-geometry tests (tests/test_geometry_emu.py on the CPU emulation, tests/test_gpu_geometry.py on the
H100): one trajectory - a sampled noisy reset with the reset action, then noisy steps with tester records - replayed env by
env on the oracle, and the comparisons every geometry must pass.

A trajectory is a dict of NumPy arrays, env axis second: ``obs`` / ``state`` / ``rec`` / ``iters`` ``[T + 1, B, ...]`` (row
0 after the reset), ``reward`` / ``term`` / ``info`` ``[T, B, ...]``, and on the device side also ``fields`` (every
``get_field`` name, ``[T + 1, B, width]``) and ``reset_ok`` ``[B]``."""
import dataclasses
import multiprocessing as mp
import os

import numpy as np

from mapdn_b200 import cases
from mapdn_b200.network import NetDesc, ProfileDesc
from oracle.voltage_control_ref import INFO_KEYS, VoltageControlOracle

TOL = 1e-9            # reward, info, obs, vm, record rows
TOL_STATE = 1e-8      # state (bus p / q in MW, va in degrees)
FIELDS = ("vm", "va_deg", "p_bus", "q_bus", "p_sgen", "q_sgen", "line_loss", "p_load", "q_load", "sum_rewards", "steps",
          "start_row", "nr_iters")
RECORD_FIELDS = ("p_sgen", "q_sgen", "p_bus", "q_bus", "vm", "line_loss")   # the tester record row, block by block
OVERRIDES = ("MAPDN_PLAN", "MAPDN_EPB", "MAPDN_HELPERS", "MAPDN_EMU_SMS")   # the planner's overrides, emulated SM count


def set_geometry(monkeypatch, geom):
    """Exactly the overrides in ``geom`` for the handles created next."""
    for k in OVERRIDES:
        monkeypatch.delenv(k, raising=False)
    for k, v in geom.items():
        monkeypatch.setenv(k, str(v))


def same(a, b, exact, what, equal_nan=False):
    """Bit for bit when ``exact``, else within 1e-10. ``equal_nan``: NaN where both have it (a sentinel of rows a call must
    not write) counts as equal; without it any NaN fails."""
    if exact:
        assert np.array_equal(a, b, equal_nan=equal_nan), what
    elif equal_nan:
        assert a.shape == b.shape and np.array_equal(np.isnan(a), np.isnan(b)), what
        d = np.abs(np.nan_to_num(a) - np.nan_to_num(b))
        assert d.size == 0 or d.max() <= 1e-10, (what, float(d.max()))
    else:
        assert a.shape == b.shape and np.abs(a - b).max() <= 1e-10, (what, float(np.abs(a - b).max()))


def overload(net, prof, factor=60.0):
    """The profile with rows 60..459 carrying a demand the feeder cannot serve (the divergence branch of step)."""
    lp = prof.load_p.copy(); lp[60:460] *= factor
    return net, ProfileDesc(pv=prof.pv, load_p=lp, load_q=prof.load_q, steps_per_hour=prof.steps_per_hour, n_days=prof.n_days)


def overloaded_case(name, n_days=4):
    """A named case through :func:`overload` (case322's synthetic demand is light: 60 times of it can still be served)."""
    return overload(cases.make_case(name), cases.make_profiles(name, n_days=n_days), 3000.0 if name == "case322" else 60.0)


def mesh4():
    """A meshed 4-bus net (the dense fallback solver) with a random four-day profile."""
    z = np.array([0.02 + 0.04j, 0.01 + 0.03j, 0.0125 + 0.025j, 0.015 + 0.03j])
    net = NetDesc(base_mva=100.0, n_bus=4, slack_bus=0, slack_vm=1.03, br_from=np.array([0, 0, 1, 2]), br_to=np.array([1, 2, 2, 3]),
                  br_r=z.real, br_x=z.imag, load_bus=np.array([1, 2, 3]), sgen_bus=np.array([2, 3]), sgen_zone=np.array([1, 1]),
                  bus_zone=np.array([0, 1, 1, 1]), name="mesh4")
    rng = np.random.default_rng(3)
    T = 4 * 24 * 20 + 1
    prof = ProfileDesc(pv=rng.uniform(0, 40, (T, 2)), load_p=rng.uniform(60, 180, (T, 3)), load_q=rng.uniform(10, 60, (T, 3)),
                       steps_per_hour=20)
    return net, prof


def actions(batch, n_sgen, scale, n_steps, seed):
    return np.random.default_rng(seed).uniform(-scale, scale, (n_steps, batch, n_sgen))


def _oracle_env(net, prof, args, env_id, acts, start):
    """One env of the trajectory on the oracle: acts [T, n_sgen]."""
    o = VoltageControlOracle(net, prof, args, env_id=env_id)
    out = {k: [] for k in ("obs", "state", "rec", "iters", "vm", "reward", "term", "info")}

    def snap():
        r = o.g.res
        out["obs"].append(np.array(o.get_obs())); out["state"].append(o.get_state()); out["vm"].append(r.vm_pu.copy())
        out["rec"].append(np.concatenate([o.g.sgen_p, o.g.sgen_q, r.p_mw, r.q_mvar, r.vm_pu, r.pl_mw]))
    o.reset(None if start is None else tuple(int(x) for x in start))
    snap(); out["iters"].append(o.g.res.iterations)
    for a in acts:
        rw, tm, info = o.step(a)
        out["reward"].append(rw); out["term"].append(tm); out["info"].append([info[k] for k in INFO_KEYS])
        # a diverged step keeps the previous power flow; the kernel reports max_iter for it
        out["iters"].append(o.g.res.iterations if info["destroy"] == 0.0 else -1)
        snap()
    return {k: np.array(v) for k, v in out.items()}


_JOB = {}


def _job(i):
    net, prof, args, offset, acts, starts = _JOB["job"]
    return _oracle_env(net, prof, args, offset + i, acts[:, i], None if starts is None else starts[i])


def oracle_trajectory(net, prof, args, env_id_offset, acts, starts=None, procs=1):
    """Every env of the batch on the oracle (env_id = offset + i), over a fork pool when procs > 1. Same layout as the
    device trajectory: [T + 1, B, ...] / [T, B, ...]."""
    B = acts.shape[1]
    _JOB["job"] = (net, prof, args, env_id_offset, acts, starts)
    try:
        if procs > 1 and B > 1:
            with mp.get_context("fork").Pool(min(procs, B)) as pool:
                per_env = pool.map(_job, range(B), chunksize=max(1, B // (8 * procs)))
        else:
            per_env = [_job(i) for i in range(B)]
    finally:
        _JOB.clear()
    return {k: np.stack([e[k] for e in per_env], axis=1) for k in per_env[0]}


def default_procs():
    return max(1, min(32, os.cpu_count() or 1))


def assert_matches_oracle(got, want, max_iter=10):
    """Every env: reward, info, obs, vm and record rows to TOL, state to TOL_STATE, terminated and Newton iteration counts
    exactly. Returns the largest difference per quantity."""
    diffs = {}
    for k, tol in (("reward", TOL), ("info", TOL), ("obs", TOL), ("rec", TOL), ("state", TOL_STATE)):
        assert got[k].shape == want[k].shape, (k, got[k].shape, want[k].shape)
        d = np.abs(got[k] - want[k])
        diffs[k] = float(d.max())
        assert diffs[k] <= tol, (k, diffs[k], np.unravel_index(int(np.argmax(d)), d.shape))
    dvm = np.abs(got["fields"]["vm"] - want["vm"])
    diffs["vm"] = float(dvm.max())
    assert diffs["vm"] <= TOL, ("vm", diffs["vm"], np.unravel_index(int(np.argmax(dvm)), dvm.shape))
    assert np.array_equal(got["term"].astype(bool), want["term"].astype(bool))
    it = np.where(want["iters"] < 0, max_iter, want["iters"])
    bad = np.argwhere(got["iters"] != it)
    assert bad.size == 0, ("nr_iters", bad[:5].tolist())
    # the record rows are the env's own fields, bit for bit
    rec_fields = np.concatenate([got["fields"][k] for k in RECORD_FIELDS], axis=-1)
    assert np.array_equal(got["rec"], rec_fields)
    return diffs


def assert_bit_identical(a, b, what):
    """Two runs of the same trajectory that differ only in launch geometry."""
    for k in a:
        if isinstance(a[k], dict):
            assert_bit_identical(a[k], b[k], f"{what}.{k}")
        else:
            assert a[k].shape == b[k].shape and np.array_equal(a[k], b[k]), (what, k)


def with_ties(net, pairs, name):
    """The net plus loop-closing lines (the median branch impedance): a meshed net, solved by the dense fallback."""
    k = len(pairs)
    extra = dict(br_b=0.0, br_g=0.0, br_tap=1.0, br_shift=0.0, br_status=1, br_is_line=1)
    kw = {a: (None if getattr(net, a) is None else np.r_[getattr(net, a), [v] * k]) for a, v in extra.items()}
    return dataclasses.replace(net, br_from=np.r_[net.br_from, [f for f, _ in pairs]], br_to=np.r_[net.br_to, [t for _, t in pairs]],
                               br_r=np.r_[net.br_r, [np.median(net.br_r)] * k], br_x=np.r_[net.br_x, [np.median(net.br_x)] * k],
                               name=name, **kw)


def meshed_chain(n_pq):
    """A chain of n_pq PQ buses behind the slack, closed into a loop by one more line."""
    rng = np.random.default_rng(n_pq)
    n = n_pq + 1
    f, t = list(range(n - 1)) + [n // 3], list(range(1, n)) + [2 * n // 3]
    return NetDesc(base_mva=1.0, n_bus=n, slack_bus=0, slack_vm=1.0, br_from=f, br_to=t, br_r=rng.uniform(1e-4, 4e-4, n),
                   br_x=rng.uniform(1e-4, 4e-4, n), load_bus=np.arange(1, n), sgen_bus=[n // 2, n - 1], sgen_zone=[1, 1],
                   bus_zone=[0] + [1] * (n - 1), name=f"mesh{n_pq}")
