"""ORACLE - TEST INFRASTRUCTURE ONLY. The scenarios behind ``tests/golden/ref_env_*.npz``: golden trajectories produced by
the reference's own ``VoltageControl`` code (``oracle/ref_harness.py`` explains what is real and what is substituted),
written by ``scripts/make_reference_golden.py`` and replayed by ``tests/test_reference_golden.py`` through the oracle
restatement (CPU) and through the CUDA path (``-m gpu``).

A scenario = network + profile store + env args + the global env ids whose RNG streams are used + a list of operations:

    ("init",)                      the reset that the reference's ``__init__`` performs (:85) = first ``reset()`` here
    ("reset",)                     ``reset()``: sampled start, noise on, random reset action (:96-133)
    ("manual", day, hour, intv)    ``manual_reset(day, hour, interval)``: noise off (:135-176)
    ("reset_keep",)                ``reset(reset_time=False)``: the previous start again, noise / reset action re-drawn
    ("step", add_noise)            ``step(actions, add_noise)`` followed by ``get_obs()`` / ``get_state()`` (:178-316)

Actions are drawn from ``np.random.default_rng`` seeded per scenario, uniformly in the env's action range.
"""
from __future__ import annotations

import zlib

import numpy as np

from mapdn_b200 import cases
from mapdn_b200.network import NetDesc, ProfileDesc


def _random_tree_net(n_bus, n_sgen, seed):
    """General radial net: taps, line charging, bus shunts, element scaling, a parallel twin, an open branch, a non-zero
    slack index and angle (same construction as tests/conftest.random_tree_net, restated here so that the fixture does
    not depend on test code)."""
    rng = np.random.default_rng(seed)
    perm = rng.permutation(n_bus)
    f, t = [], []
    for k in range(1, n_bus):
        f.append(perm[rng.integers(0, k)])
        t.append(perm[k])
    f, t = np.array(f), np.array(t)
    flip = rng.random(n_bus - 1) < 0.5
    f, t = np.where(flip, t, f), np.where(flip, f, t)
    r = rng.uniform(1e-3, 2e-2, n_bus - 1)
    x = r * rng.uniform(0.3, 2.0, n_bus - 1)
    b = rng.uniform(0, 2e-3, n_bus - 1)
    g = rng.uniform(0, 1e-4, n_bus - 1)
    tap = np.ones(n_bus - 1)
    is_line = np.ones(n_bus - 1, np.uint8)
    k = rng.choice(n_bus - 1, max(1, (n_bus - 1) // 6), replace=False)
    tap[k] = rng.uniform(0.95, 1.05, len(k))
    is_line[k] = 0
    f = np.r_[f, f[0], f[1]]; t = np.r_[t, t[0], t[1]]
    r = np.r_[r, r[0] * 1.3, r[1]]; x = np.r_[x, x[0] * 0.9, x[1]]
    b = np.r_[b, 0.0, 0.0]; g = np.r_[g, 0.0, 0.0]; tap = np.r_[tap, tap[0], 1.0]
    is_line = np.r_[is_line, is_line[0], 1].astype(np.uint8)
    status = np.ones(n_bus + 1, np.uint8); status[-1] = 0
    zone = rng.integers(0, 4, n_bus).astype(np.int32)
    sgen_bus = rng.choice(n_bus, n_sgen, replace=False).astype(np.int32)
    zone[sgen_bus] = np.maximum(zone[sgen_bus], 1)
    n_load = n_bus + 3
    load_bus = np.r_[np.arange(n_bus), rng.integers(0, n_bus, 3)].astype(np.int32)
    return NetDesc(base_mva=10.0, n_bus=n_bus, slack_bus=int(perm[0]), slack_vm=1.02, slack_va_deg=3.0,
                   br_from=f, br_to=t, br_r=r, br_x=x, br_b=b, br_g=g, br_tap=tap, br_status=status,
                   br_is_line=is_line, bus_gs=rng.uniform(0, 0.05, n_bus), bus_bs=rng.uniform(-0.05, 0.05, n_bus),
                   load_bus=load_bus, load_scaling=rng.uniform(0.8, 1.2, n_load),
                   sgen_bus=sgen_bus, sgen_zone=zone[sgen_bus], sgen_scaling=rng.uniform(0.9, 1.1, n_sgen),
                   bus_zone=zone, name=f"rand{n_bus}")


def _general_case():
    net = _random_tree_net(23, 4, seed=11)
    rng = np.random.default_rng(2)
    T = 3 * 480 + 1
    prof = ProfileDesc(pv=rng.uniform(0.1, 0.5, (T, net.n_sgen)), load_p=rng.uniform(0.0, 0.3, (T, net.n_load)),
                       load_q=rng.uniform(0.0, 0.1, (T, net.n_load)), steps_per_hour=20, n_days=3)
    return net, prof


def _overload_case():
    """case33 with a profile whose rows 60..459 carry a demand the feeder cannot serve: the divergence branch of step
    (:188-196) and, for sampled starts inside the window, the retry loop of reset (:108-133)."""
    net, prof = cases.case33(), cases.make_profiles("case33", n_days=4)
    lp = prof.load_p.copy(); lp[60:460] *= 60.0
    return net, ProfileDesc(pv=prof.pv, load_p=lp, load_q=prof.load_q, steps_per_hour=20, n_days=prof.n_days)


def _case(name):
    return cases.make_case(name), cases.make_profiles(name, n_days=4)


_FULL = [("init",)] + [("step", True)] * 4 + [("reset",)] + [("step", True)] * 2 + [("manual", 2, 11, 7)] + \
        [("step", False)] * 3
_SHORT = [("init",)] + [("step", True)] * 3

SCENARIOS = {}


def _add(name, build, args, env_ids, ops, per_env_manual=None):
    assert ops[0] == ("init",)          # the reference's constructor always performs the first reset (:85)
    SCENARIOS[name] = dict(name=name, build=build, args=args, env_ids=list(env_ids), ops=list(ops),
                           per_env_manual=per_env_manual)


for _b in ("l1", "l2", "bowl", "bump", "courant_beltrami"):
    _add(f"case33_{_b}", lambda: _case("case33"), dict(voltage_barrier_type=_b, action_scale=0.8, seed=5), (0, 7), _FULL)
_add("case141_l1", lambda: _case("case141"), dict(voltage_barrier_type="l1", action_scale=0.6, seed=5), (0, 3), _SHORT)
_add("case322_bowl", lambda: _case("case322"), dict(voltage_barrier_type="bowl", action_scale=0.8, seed=5), (0, 2), _SHORT)
_add("case322_l2", lambda: _case("case322"), dict(voltage_barrier_type="l2", action_scale=0.8, seed=6), (1,),
     [("init",), ("step", True), ("manual", 1, 13, 4), ("step", False)])
_add("general_line_weight", _general_case,
     dict(voltage_barrier_type="l1", line_weight=0.7, q_weight=None, action_scale=0.5, action_bias=0.1, seed=9), (0, 1, 4),
     _FULL[:8] + [("manual", 1, 9, 3)] + [("step", False)] * 2)
_add("case33_state_space", lambda: _case("case33"),
     dict(voltage_barrier_type="bowl", action_scale=0.8, seed=8, state_space=["pv", "vm_pu", "demand"], reset_action=False,
          voltage_weight=2.5, q_weight=0.3, v_upper=1.03, v_lower=0.97, episode_limit=6), (0, 5),
     [("init",)] + [("step", True)] * 5)          # steps reaches episode_limit: terminated without divergence
# obs history (:303-315): every get_obs() call stacks the last `history` frames (zero frames first); the fixtures hold the
# stacked rows, the batched engine / the oracle restatement are compared on the newest frame
_add("case33_history", lambda: _case("case33"), dict(voltage_barrier_type="l1", action_scale=0.8, seed=12, history=3), (0,),
     [("init",)] + [("step", True)] * 3 + [("reset",), ("step", True)])
_add("case33_reset_keep", lambda: _case("case33"), dict(voltage_barrier_type="l2", action_scale=0.8, seed=14), (0, 2),
     [("init",), ("step", True), ("reset_keep",), ("step", True), ("step", True)])
# manual starts at rows 55..58 (day 0, hour 2, interval 15 + k): the overload begins at row 60
_add("case33_divergence", _overload_case, dict(voltage_barrier_type="l1", action_scale=0.8, seed=7), (0, 1, 2, 3),
     [("init",), ("manual", 0, 2, 15)] + [("step", False)] * 7, per_env_manual=lambda k: (0, 2, 15 + (k % 4)))


def action_stream(name, n_steps, n_env, n_agents, low, high):
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    return rng.uniform(low, high, (n_steps, n_env, n_agents))


def fixture_path(root, name):
    import os
    return os.path.join(root, "tests", "golden", f"ref_env_{name}.npz")


def digest(a):
    """SHA-256 of an array's float64 values: exact equality against a fixture without storing the array."""
    import hashlib
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float64).tobytes()).hexdigest()


def n_steps_of(sc):
    return sum(1 for op in sc["ops"] if op[0] == "step")


def manual_of(sc, op, k):
    """(day, hour, interval) of a manual reset for the k-th env of the scenario."""
    return sc["per_env_manual"](k) if sc["per_env_manual"] is not None else tuple(op[1:4])
