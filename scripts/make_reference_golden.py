#!/usr/bin/env python
"""Writes tests/golden/ref_env_*.npz: trajectories produced by the REFERENCE's own env code
(/root/reference/environments/var_voltage_control/voltage_control_env.py, unmodified, imported at run time) for the
scenarios of oracle/ref_scenarios.py. Only runs where /root/reference exists (this container); pandapower is substituted
as described in oracle/ref_harness.py (the Newton-Raphson behind pp.runpp is oracle/pandapower_nr.py - these fixtures pin
the ENV LOGIC, the literature KATs and scripts/pin_with_pandapower.py pin the power flow).

    python scripts/make_reference_golden.py [scenario ... | records]

``records`` writes tests/golden/ref_env_records.npz (see :func:`records`).
"""
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_harness as H            # noqa: E402
from oracle import ref_scenarios as S          # noqa: E402


def main():
    names = sys.argv[1:] or list(S.SCENARIOS) + ["records"]
    for name in names:
        if name == "records":
            path = S.fixture_path(ROOT, "records")
            np.savez_compressed(path, **records())
            print(f"records: {os.path.getsize(path) / 1024:.1f} kB")
            continue
        sc = S.SCENARIOS[name]
        res = record(sc)
        path = S.fixture_path(ROOT, name)
        np.savez_compressed(path, **res)
        print(f"{name}: {os.path.getsize(path) / 1024:.1f} kB, {res['reward'].shape[0]} steps x {len(sc['env_ids'])} envs")


def record(sc, view_rows=True):
    """Runs the reference env for every env id of the scenario. Arrays: obs [n_ops, E, n_agents, obs_dim],
    state [n_ops, E, state_dim] (one snapshot after every operation), reward / term [n_steps, E], info [n_steps, E, 11],
    alive [n_steps, E] (0 once an env has terminated: the reference would be reset by its caller), start [n_resets, E, 3]
    = (day, hour, interval) the reference used, actions [n_steps, E, n_agents]."""
    net, prof = sc["build"]()
    ids = sc["env_ids"]
    E, n_steps = len(ids), S.n_steps_of(sc)
    obs, state, start = [], [], []
    reward, term = np.zeros((n_steps, E)), np.zeros((n_steps, E), np.uint8)
    info, alive = np.zeros((n_steps, E, 11)), np.ones((n_steps, E), np.uint8)
    with tempfile.TemporaryDirectory() as d:
        H.write_reference_data(d, net, prof)
        runs = [H.ReferenceRun(d, net, sc["args"], env_id=e, view_rows=view_rows) for e in ids]
        lo, hi = runs[0].env.action_space.low, runs[0].env.action_space.high
        acts = S.action_stream(sc["name"], n_steps, E, net.n_sgen, lo, hi)
        dead = [False] * E
        t = 0
        for k_op, op in enumerate(sc["ops"]):
            o_all, s_all = [], []
            for k, r in enumerate(runs):
                if op[0] == "init":
                    o, s = r.initial()
                elif op[0] == "reset":
                    o, s = r.reset()
                elif op[0] == "manual":
                    o, s = r.manual_reset(*S.manual_of(sc, op, k))
                elif op[0] == "reset_keep":
                    o, s = r.reset_keep_time()
                elif dead[k]:
                    alive[t, k] = 0
                    o, s = obs[-1][k], state[-1][k]
                else:
                    reward[t, k], tm, info[t, k], o, s = r.step(acts[t, k], add_noise=op[1])
                    term[t, k] = tm
                    dead[k] = tm
                o_all.append(o); s_all.append(s)
            if op[0] == "step":
                t += 1
            else:
                start.append([r.start[0] for r in runs])
                dead = [False] * E
            obs.append(np.array(o_all)); state.append(np.array(s_all))
    return dict(env_ids=np.array(ids), ops=np.array(json.dumps(sc["ops"])), actions=acts, obs=np.array(obs),
                state=np.array(state), reward=reward, term=term, info=info, alive=alive,
                start=np.array(start, np.int64).reshape(len(start), E, 3))


RERUN = ["case33_bowl", "general_line_weight", "case33_divergence", "case33_state_space", "case33_history", "case33_reset_keep"]
RERUN_KEYS = ("obs", "state", "reward", "term", "info", "alive", "start", "actions")


def records():
    """What the reference itself did in three situations that the trajectories above do not cover:
    * csv_*: its CSV readers (voltage_control_env.py:407-438) on case33 profiles (3 days, pv_scale 1.3, demand_scale 0.7):
      digests of the three tables, the std / s_max vectors, time_delta and the day span;
    * pinned_* / cow_*: one reset + one step of case33_bowl env 0 with the zone table's rows as views (the pandas the
      reference pins) and as copies (copy-on-write pandas): obs, state, reward;
    * decentralised_error: the exception its constructor raises for mode="decentralised";
    * rerun_<scenario>_<key>: digests of a second run of the reference on six of the scenarios."""
    from mapdn_b200 import cases
    out = {}
    net, prof = cases.make_case("case33"), cases.make_profiles("case33", n_days=3)
    with tempfile.TemporaryDirectory() as d:
        H.write_reference_data(d, net, prof)
        env = H.ReferenceRun(d, net, dict(pv_scale=1.3, demand_scale=0.7, seed=0), env_id=0).env
        out.update(csv_pv=S.digest(env.pv_data.values), csv_load_p=S.digest(env.active_demand_data.values),
                   csv_load_q=S.digest(env.reactive_demand_data.values), csv_pv_std=np.asarray(env.pv_std, np.float64),
                   csv_s_max=np.asarray(env.s_max, np.float64),
                   csv_load_p_std=np.asarray(env.active_demand_std, np.float64), csv_time_delta=env.time_delta,
                   csv_n_days=(env.pv_data.index[-1] - env.pv_data.index[0]).days)
        try:
            H.ReferenceRun(d, net, dict(mode="decentralised", seed=0), env_id=0)
            out["decentralised_error"] = "none"
        except Exception as e:      # noqa: BLE001
            out["decentralised_error"] = f"{type(e).__name__}: {e}"
    sc = dict(S.SCENARIOS["case33_bowl"], ops=[("init",), ("step", True)], env_ids=[0])
    for tag, view in (("pinned", True), ("cow", False)):
        r = record(sc, view_rows=view)
        out.update({f"{tag}_obs": r["obs"], f"{tag}_state": r["state"], f"{tag}_reward": r["reward"]})
    out["pandas_ops"] = np.array(json.dumps(sc["ops"]))
    for name in RERUN:                                  # digests of a fresh run, to hold the committed fixtures to
        res = record(S.SCENARIOS[name])
        out.update({f"rerun_{name}_{key}": S.digest(res[key]) for key in RERUN_KEYS})
    return {k: np.array(v) for k, v in out.items()}


if __name__ == "__main__":
    main()
