"""Golden trajectories produced by the REFERENCE's own env code (tests/golden/ref_env_*.npz, written by
scripts/make_reference_golden.py from /root/reference/environments/var_voltage_control/voltage_control_env.py with the
pandapower import substituted - oracle/ref_harness.py says exactly what is real and what is not).

* CPU: the oracle restatement (oracle/voltage_control_ref.py) reproduces them (1e-11);
* CPU: a re-run of the reference reproduced the committed fixtures, ingest reads CSV files as the reference's readers
  did, the product follows the reference's get_obs under the pandas it pins, and the reference's decentralised mode
  failed (tests/golden/ref_env_records.npz);
* ``-m gpu``: the CUDA path through the C-ABI reproduces them at the parity tolerances of the other GPU tests
  (reward / info / obs 1e-9, state 1e-8).

Every scenario covers reset (sampled start, noise, random reset action), noisy steps, a second episode, manual_reset and
noise-free steps; all five barriers; case33 / 141 / 322; a general net with transformers, shunts, scaling and the
line_weight reward; a reduced state_space with non-default weights / limits / episode_limit; the divergence branch."""
import json

import numpy as np
import pytest

from conftest import ROOT
from oracle import ref_scenarios as S

NAMES = list(S.SCENARIOS)


def _load(name):
    g = np.load(S.fixture_path(ROOT, name))
    return g, [tuple(op) for op in json.loads(str(g["ops"]))]


def test_fixtures_match_the_scenario_table():
    for name in NAMES:
        g, ops = _load(name)
        sc = S.SCENARIOS[name]
        assert ops == [tuple(op) for op in sc["ops"]] and g["env_ids"].tolist() == sc["env_ids"]
        net, _ = sc["build"]()
        lo = -sc["args"]["action_scale"] + sc["args"].get("action_bias", 0.0)
        hi = sc["args"]["action_scale"] + sc["args"].get("action_bias", 0.0)
        acts = S.action_stream(name, S.n_steps_of(sc), len(sc["env_ids"]), net.n_sgen, lo, hi)
        assert np.array_equal(acts, g["actions"])
        assert g["obs"].shape[:3] == (len(ops), len(sc["env_ids"]), net.n_sgen)
        assert g["obs"].shape[3] == sc["args"].get("history", 1) * net.obs_dim or "state_space" in sc["args"]


@pytest.mark.parametrize("name", NAMES)
def test_oracle_reproduces_the_reference_trajectories(name):
    from oracle.voltage_control_ref import INFO_KEYS, VoltageControlOracle
    g, ops = _load(name)
    sc = S.SCENARIOS[name]
    net, prof = sc["build"]()
    for k, e in enumerate(sc["env_ids"]):
        o = VoltageControlOracle(net, prof, sc["args"], env_id=e)
        t = n_reset = 0
        for k_op, op in enumerate(ops):
            if op[0] == "step":
                if g["alive"][t, k]:
                    r, term, info = o.step(g["actions"][t, k], add_noise=op[1])
                    assert abs(r - g["reward"][t, k]) < 1e-11 and term == bool(g["term"][t, k])
                    assert np.abs(np.array([info[q] for q in INFO_KEYS]) - g["info"][t, k]).max() < 1e-11
                    obs, st = np.array(o.get_obs()), o.get_state()
                else:
                    obs = None
                t += 1
            else:
                if op[0] == "manual":
                    obs, st = o.reset(start=S.manual_of(sc, op, k), add_noise=False)
                elif op[0] == "reset_keep":                      # reset(reset_time=False): the previous start, noise on
                    obs, st = o.reset(start=tuple(int(x) for x in g["start"][n_reset - 1, k]), add_noise=True)
                else:
                    obs, st = o.reset()
                day, hour, interval = g["start"][n_reset, k]
                assert o.start == interval + hour * prof.steps_per_hour + day * 24 * prof.steps_per_hour
                n_reset += 1
                obs = np.array(obs)
            if obs is not None:
                assert np.abs(obs - g["obs"][k_op, k][:, -obs.shape[1]:]).max() < 1e-11     # history > 1: the newest frame
                assert np.abs(st - g["state"][k_op, k]).max() < 1e-9        # va_degree: 1e-11 rad x 57.3


def _records():
    return np.load(S.fixture_path(ROOT, "records"))


@pytest.mark.parametrize("name", ["case33_bowl", "general_line_weight", "case33_divergence", "case33_state_space", "case33_history",
                                  "case33_reset_keep"])
def test_reference_rerun_reproduces_the_committed_fixture(name):
    """A second run of the reference (digests recorded by scripts/make_reference_golden.py) produced exactly the committed
    fixture: the script and the fixtures cannot drift apart."""
    ref = _records()
    g, _ = _load(name)
    for key in ("obs", "state", "reward", "term", "info", "alive", "start", "actions"):
        assert S.digest(g[key]) == str(ref[f"rerun_{name}_{key}"]), key


def test_reference_csv_loading_equals_ingest(tmp_path):
    """The reference's own CSV readers (voltage_control_env.py:407-438) and mapdn_b200.ingest.load_profiles read the same
    files to the same arrays, statistics and action bounds (pv_scale / demand_scale applied)."""
    from mapdn_b200 import cases, ingest
    from oracle import ref_harness as H
    ref = _records()
    net, prof = cases.make_case("case33"), cases.make_profiles("case33", n_days=3)
    H.write_reference_data(str(tmp_path), net, prof)
    got = ingest.load_profiles(str(tmp_path), pv_scale=1.3, demand_scale=0.7)
    assert S.digest(got.pv) == ref["csv_pv"] and S.digest(got.load_p) == ref["csv_load_p"]
    assert S.digest(got.load_q) == ref["csv_load_q"]
    assert np.allclose(ref["csv_pv_std"], got.pv_std, rtol=0, atol=1e-15) and np.allclose(ref["csv_s_max"], got.s_max, rtol=0, atol=1e-15)
    assert np.allclose(ref["csv_load_p_std"], got.load_p_std, rtol=0, atol=1e-15)
    assert got.steps_per_hour == 60 // int(ref["csv_time_delta"])
    assert got.n_days == int(ref["csv_n_days"])


def test_reference_get_obs_depends_on_the_pandas_version():
    """voltage_control_env.py:239-244 adds every PV's p/q to its bus row of the zone table through a chained
    ``.loc[bus]["p_mw"] += pv``. With the pandas the reference pins (1.1.3) the row is a view and the write lands; with
    copy-on-write pandas (>= 3) it is lost. The product (and every fixture) follows the pinned behaviour; this test keeps
    the difference on record: only the "demand" entries of the PV buses change, by exactly the PV's p and q."""
    from oracle.voltage_control_ref import VoltageControlOracle
    ref = _records()
    sc = S.SCENARIOS["case33_bowl"]
    assert json.loads(str(ref["pandas_ops"])) == [["init"], ["step", True]]
    pinned = {k: ref[f"pinned_{k}"] for k in ("obs", "state", "reward")}
    cow = {k: ref[f"cow_{k}"] for k in ("obs", "state", "reward")}
    assert np.array_equal(pinned["reward"], cow["reward"]) and np.array_equal(pinned["state"], cow["state"])
    net, prof = sc["build"]()
    d = pinned["obs"][1, 0] - cow["obs"][1, 0]                 # [n_agents, obs_dim] after the step
    pv, q = pinned["state"][1, 0][2 * net.n_bus:2 * net.n_bus + net.n_sgen], pinned["state"][1, 0][2 * net.n_bus + net.n_sgen:2 * net.n_bus + 2 * net.n_sgen]
    for a in range(net.n_sgen):
        zb = net.zone_buses(a)
        exp = np.zeros(pinned["obs"].shape[-1])
        for j in range(net.n_sgen):
            if net.sgen_zone[j] == net.sgen_zone[a]:
                kk = int(np.nonzero(zb == net.sgen_bus[j])[0][0])
                exp[kk] += pv[j]
                exp[len(zb) + kk] += q[j]
        assert np.abs(d[a] - exp).max() < 1e-12
    assert np.abs(d).max() > 1e-3
    # the product's env logic reproduces the pinned behaviour, not the copy-on-write one
    lo = -sc["args"]["action_scale"] + sc["args"].get("action_bias", 0.0)
    hi = sc["args"]["action_scale"] + sc["args"].get("action_bias", 0.0)
    acts = S.action_stream(sc["name"], 1, 1, net.n_sgen, lo, hi)
    o = VoltageControlOracle(net, prof, sc["args"], env_id=0)
    o.reset()
    assert np.abs(np.array(o.get_obs()) - pinned["obs"][0, 0]).max() < 1e-11
    r, _, _ = o.step(acts[0, 0], add_noise=True)
    assert abs(r - pinned["reward"][0, 0]) < 1e-11
    assert np.abs(np.array(o.get_obs()) - pinned["obs"][1, 0]).max() < 1e-11


# ------------------------------------------------------------------ CUDA path ------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_cuda_path_reproduces_the_reference_trajectories(name):
    import torch
    from mapdn_b200.env import BatchedVoltageControl
    g, ops = _load(name)
    sc = S.SCENARIOS[name]
    net, prof = sc["build"]()
    ids = sc["env_ids"]
    B = max(ids) + 1
    env = BatchedVoltageControl(net, prof, sc["args"], batch=B)
    spd = prof.steps_per_hour
    t = n_reset = 0
    for k_op, op in enumerate(ops):
        if op[0] == "step":
            a = np.zeros((B, net.n_sgen))
            a[ids] = g["actions"][t]
            r, term, info = env.step(torch.tensor(a, device=env.device), add_noise=op[1])
            st = env.get_state()
            torch.cuda.synchronize()
            live = np.nonzero(g["alive"][t])[0]
            sel = [ids[k] for k in live]
            if live.size:
                assert np.abs(r[sel].cpu().numpy() - g["reward"][t, live]).max() < 1e-9
                assert np.array_equal(term[sel].cpu().numpy(), g["term"][t, live])
                assert np.abs(info[sel].cpu().numpy() - g["info"][t, live]).max() < 1e-9
            t += 1
            if live.size == 0:          # every env of the scenario has terminated (the reference's caller would reset)
                continue
        else:
            if op[0] in ("manual", "reset_keep"):
                start = np.zeros((B, 3), np.int32)
                for k, e in enumerate(ids):
                    start[e] = S.manual_of(sc, op, k) if op[0] == "manual" else g["start"][n_reset - 1, k]
                env.reset(torch.tensor(start, device=env.device), add_noise=(op[0] == "reset_keep"))
            else:
                env.reset()
            st = env.get_state()
            torch.cuda.synchronize()
            rows = env.get_field("start_row")[ids, 0].cpu().numpy()
            s = g["start"][n_reset]
            assert np.array_equal(rows, s[:, 2] + s[:, 1] * spd + s[:, 0] * 24 * spd)
            n_reset += 1
            live = np.arange(len(ids))
            sel = ids
        assert np.abs(env.obs[sel].cpu().numpy() - g["obs"][k_op, live][..., -env.obs_size:]).max() < 1e-9   # newest frame
        assert np.abs(st[sel].cpu().numpy() - g["state"][k_op, live]).max() < 1e-8
    env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n in NAMES if S.SCENARIOS[n]["env_ids"][0] == 0 and not n.startswith("case322")])
def test_drop_in_class_reproduces_the_reference_trajectories(name):
    """The same replay through ``mapdn_b200.VoltageControl`` - the class a user of the reference switches to (same
    constructor argument, method names, NumPy shapes, info keys): it is env id 0 of the batched engine."""
    from mapdn_b200.env import INFO_KEYS, VoltageControl
    g, ops = _load(name)
    sc = S.SCENARIOS[name]
    net, prof = sc["build"]()
    env = VoltageControl(dict(sc["args"], net=net, profiles=prof))          # resets like the reference's __init__ (:85)
    nb, ng = net.n_bus, net.n_sgen
    t = 0
    for k_op, op in enumerate(ops):
        if op[0] == "step":
            if not g["alive"][t, 0]:
                break
            reward, terminated, info = env.step(g["actions"][t, 0], add_noise=op[1])
            assert abs(reward - g["reward"][t, 0]) < 1e-9 and terminated == bool(g["term"][t, 0])
            assert list(info) == list(INFO_KEYS)
            assert np.abs(np.array([info[q] for q in INFO_KEYS]) - g["info"][t, 0]).max() < 1e-9
            t += 1
            obs, state = env.get_obs(), env.get_state()
        elif op[0] == "init":
            obs, state = env.get_obs(), env.get_state()
        elif op[0] == "reset":
            obs, state = env.reset()
        elif op[0] == "reset_keep":
            obs, state = env.reset(reset_time=False)
        else:
            obs, state = env.manual_reset(*S.manual_of(sc, op, 0))
        if op[0] != "step":
            d, h, i = g["start"][sum(1 for o in ops[:k_op] if o[0] != "step"), 0]
            assert (env._episode_start_day, env._episode_start_hour, env._episode_start_interval) == (d, h, i)
            assert env.steps == 1 and env.sum_rewards == 0
        assert isinstance(obs, list) and len(obs) == ng and obs[0].shape == (env.get_obs_size(),) == (g["obs"].shape[-1],)
        assert np.abs(np.array(obs) - g["obs"][k_op, 0]).max() < 1e-9
        assert state.shape == (env.get_state_size(),) and np.abs(state - g["state"][k_op, 0]).max() < 1e-8
        if "state_space" not in sc["args"]:          # default layout: [p_bus | q_bus | pv | q | vm | va_degree] (:213-230)
            ref = g["state"][k_op, 0]
            assert np.abs(env._get_res_bus_active() - ref[:nb]).max() < 1e-9
            assert np.abs(env._get_res_bus_reactive() - ref[nb:2 * nb]).max() < 1e-9
            assert np.abs(env._get_sgen_active() - ref[2 * nb:2 * nb + ng]).max() < 1e-9
            assert np.abs(env._get_sgen_reactive() - ref[2 * nb + ng:2 * nb + 2 * ng]).max() < 1e-9
            assert np.abs(env._get_res_bus_v() - ref[2 * nb + 2 * ng:3 * nb + 2 * ng]).max() < 1e-9
    info_env = env.get_env_info()
    assert info_env["n_agents"] == ng and info_env["obs_shape"] == g["obs"].shape[-1] and info_env["state_shape"] == g["state"].shape[-1]
    env.close()


def test_reference_decentralised_mode_is_broken_upstream():
    """`mode="decentralised"` cannot even construct the reference env: `get_obs` indexes `clusters["sgen0"]`
    (voltage_control_env.py:239), a key that only the distributed branch of `_get_clusters_info` creates. The product
    therefore raises NotImplementedError for that mode instead of inventing semantics."""
    assert str(_records()["decentralised_error"]) == "KeyError: 'sgen0'"
