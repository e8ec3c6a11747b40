"""Launch geometries on the H100, at the sizes the benchmark runs.

Benchmark-size parity: case33 x 4096 (Bowl), case141 x 2048 (L1), case322 x 1024 and x 512 (L2) - the planner's own
geometries, including case141's and case322 x 1024's two rounds of a persistent grid and case322's plan 3 (cold tables,
loads staged in the node records) - run a sampled noisy reset and two noisy steps with tester records, and EVERY env is
compared with the oracle (tests/geometry_cases.py; the oracle runs over a process pool).

The matrix on the device: forced plans 0-3, helper warps 1 and 4, small and default envs per CTA for case141 x 2048 and
case322 x 1024, each needing at least two rounds, must give bit-identical outputs (and so match the oracle too).

The record instantiation's own persistent grid (max_blocks_record) never needs more rounds than the plain step's at the
planner's geometries: for G <= 32 it holds 165-166 registers instead of 130-134 (168 vs 136 allocated, 5376 vs 4352 per
warp), so a CTA of W warps fits floor(12.19 / W) times instead of floor(15.06 / W) by registers - fewer only for W = 2, 3,
5 or 7. The planner picks a CTA size that finishes the batch in one round of <= 132 CTAs whenever that fits (1 CTA per SM
suffices for both grids). Where it plans 2-3 rounds its CTAs take >= 115 KB of shared memory (one per SM for both grids).
Beyond that it falls back to its default CTA (case33: 4 warps, case141: 6), where both grids hold 3 / 2 CTAs per SM.
Replaying the planner for every 7th batch size up to 20 000 (case33, case141) found no batch where the record grid needs
more rounds. For G = 64 / 128 both instantiations sit at the 96-register cap of __launch_bounds__(640).
"""
import time

import numpy as np
import pytest
import torch

import geometry_cases as GC
from mapdn_b200 import cases
from mapdn_b200.env import BatchedVoltageControl

pytestmark = pytest.mark.gpu
OVERRIDES = ("MAPDN_PLAN", "MAPDN_EPB", "MAPDN_HELPERS")
SMEM_PER_SM = 233472          # H100: 228 KB of shared memory per SM, 1 KB of it reserved per CTA
T_STEPS = 2
_ORACLE = {}


def _setup(name, barrier, batch):
    net, prof = cases.make_case(name), cases.make_profiles(name, n_days=4)
    scale = cases.SCENARIOS[name]["action_scale"]
    args = dict(voltage_barrier_type=barrier, action_scale=scale, seed=11)
    return net, prof, args, GC.actions(batch, net.n_sgen, scale, T_STEPS, seed=batch)


def _oracle(name, barrier, batch):
    key = (name, barrier, batch)
    if key not in _ORACLE:
        net, prof, args, acts = _setup(name, barrier, batch)
        t0 = time.time()
        _ORACLE[key] = GC.oracle_trajectory(net, prof, args, 100, acts, procs=GC.default_procs())
        print(f"\n[oracle] {name} x {batch}: {time.time() - t0:.1f} s on {GC.default_procs()} processes")
    return _ORACLE[key]


def _device_run(monkeypatch, name, barrier, batch, geom):
    for k in OVERRIDES:
        monkeypatch.delenv(k, raising=False)
    for k, v in geom.items():
        monkeypatch.setenv(k, str(v))
    net, prof, args, acts = _setup(name, barrier, batch)
    env = BatchedVoltageControl(net, prof, args, batch=batch, env_id_offset=100)
    try:
        dev = env.device
        R = env.record_len
        rec = torch.full((batch, T_STEPS + 1, R), float("nan"), dtype=torch.float64, device=dev)
        out = {k: [] for k in ("obs", "state", "iters", "reward", "term", "info")}
        fields = {k: [] for k in GC.FIELDS}

        def snap():
            out["obs"].append(env.obs.cpu().numpy().copy()); out["state"].append(env.get_state().cpu().numpy().copy())
            for k in GC.FIELDS:
                fields[k].append(env.get_field(k).cpu().numpy())
            out["iters"].append(fields["nr_iters"][-1][:, 0].astype(np.int64))
        env.reset_ok.fill_(7)
        env.reset()
        reset_ok = env.reset_ok.cpu().numpy().copy()
        env.record(rec[:, 0])
        snap()
        for t in range(T_STEPS):
            r, tm, info = env.step(torch.tensor(acts[t], device=dev), record=rec[:, t + 1])
            out["reward"].append(r.cpu().numpy().copy()); out["term"].append(tm.cpu().numpy().copy())
            out["info"].append(info.cpu().numpy().copy())
            snap()
        traj = {k: np.array(v) for k, v in out.items()}
        traj["rec"] = rec.transpose(0, 1).cpu().numpy().copy()
        traj["fields"] = {k: np.array(v) for k, v in fields.items()}
        traj["reset_ok"] = reset_ok
        return env.dims, traj
    finally:
        env.close()


def _min_rounds(batch, dims):
    """Rounds of the persistent loop at the least: CTAs per SM cannot exceed what shared memory allows."""
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    per_sm = SMEM_PER_SM // (dims["smem_bytes"] + 1024)
    needed = -(-batch // dims["envs_per_block"])
    return -(-needed // (per_sm * n_sm))


def _check_oracle(name, barrier, batch, traj):
    assert np.all(traj["reset_ok"] == 1)
    diffs = GC.assert_matches_oracle(traj, _oracle(name, barrier, batch))
    print(f"[parity] {name} x {batch}: largest differences " + ", ".join(f"{k} {v:.1e}" for k, v in diffs.items()))


BENCH = [("case33", "bowl", 4096, (8, 32, 184064)), ("case141", "l1", 2048, (32, 8, 204896)),
         ("case322", "l2", 1024, (64, 4, 229328)), ("case322", "l2", 512, (64, 4, 229328))]


@pytest.mark.parametrize("name,barrier,batch,geometry", BENCH)
def test_benchmark_size_batches_match_the_oracle_env_by_env(monkeypatch, name, barrier, batch, geometry):
    t0 = time.time()
    dims, traj = _device_run(monkeypatch, name, barrier, batch, {})
    assert (dims["lanes_per_env"], dims["envs_per_block"], dims["smem_bytes"]) == geometry
    if name != "case33" and batch > 512:
        assert _min_rounds(batch, dims) >= 2
    _check_oracle(name, barrier, batch, traj)
    print(f"[time] {name} x {batch}: {time.time() - t0:.1f} s")


# forced plans at a CTA size every plan holds, helper warps 1 and 4, one env per CTA
MATRIX = {
    ("case141", "l1", 2048): [dict(MAPDN_PLAN=k, MAPDN_EPB=4, MAPDN_HELPERS=h) for k, h in zip(range(4), (1, 4, 1, 4))]
    + [dict(MAPDN_EPB=1, MAPDN_HELPERS=1), dict(MAPDN_HELPERS=4)],
    ("case322", "l2", 1024): [dict(MAPDN_PLAN=k, MAPDN_EPB=3, MAPDN_HELPERS=h) for k, h in zip(range(4), (4, 1, 4, 1))]
    + [dict(MAPDN_EPB=1, MAPDN_HELPERS=1), dict(MAPDN_HELPERS=1)],
}


@pytest.mark.parametrize("config", sorted(MATRIX))
def test_forced_geometries_are_bit_identical_on_the_device(monkeypatch, config):
    name, barrier, batch = config
    _, ref = _device_run(monkeypatch, name, barrier, batch, {})
    _check_oracle(name, barrier, batch, ref)
    smem = {}
    for geom in MATRIX[config]:
        dims, traj = _device_run(monkeypatch, name, barrier, batch, geom)
        assert _min_rounds(batch, dims) >= 2, (geom, dims)
        if "MAPDN_EPB" in geom:
            assert dims["envs_per_block"] == geom["MAPDN_EPB"], (geom, dims)
        if "MAPDN_PLAN" in geom:
            smem[geom["MAPDN_PLAN"]] = dims["smem_bytes"]
        GC.assert_bit_identical(ref, traj, str(geom))
    # the four plans were all in effect (two independent savings: the once-per-step tables, the staged loads)
    assert smem[0] - smem[1] == smem[2] - smem[3] > 0 and smem[0] - smem[2] == smem[1] - smem[3] > 0, smem


@pytest.mark.parametrize("which", ["case141_meshed", "mesh256"])
def test_meshed_dense_fallback_beyond_one_row_per_lane(which):
    """The dense fallback at 2 npq = 280 (case141 with four tie lines: solve and noisy steps, every env against the
    oracle) and at its limit of 256 PQ buses (2 npq = 512: solve against the oracle's Newton-Raphson)."""
    from oracle.pandapower_nr import PandapowerEquivalent
    if which == "mesh256":
        net = GC.meshed_chain(256)
        B, rng = 8, np.random.default_rng(0)
        pl = rng.uniform(0.0, 0.004, (B, net.n_load)); ql = 0.3 * pl
        pv = rng.uniform(0.0, 0.2, (B, 2)); qv = rng.uniform(-0.05, 0.05, (B, 2))
        env = BatchedVoltageControl(net, None, dict(voltage_barrier_type="l1"), batch=1)
        assert env.dims["lanes_per_env"] == 32
        out = {k: v.cpu().numpy() for k, v in env.solve(pl, ql, pv, qv).items()}
        env.close()
        pf = PandapowerEquivalent(net)
        for e in range(B):
            r = pf.runpp(pl[e], ql[e], pv[e], qv[e])
            assert r.converged and out["converged"][e] == 1 and out["iterations"][e] == r.iterations
            assert np.abs(out["vm"][e] - r.vm_pu).max() < GC.TOL and np.abs(out["pl"][e] - r.pl_mw).max() < GC.TOL
        return
    net = GC.with_ties(cases.make_case("case141"), [(10, 60), (30, 100), (50, 130), (80, 140)], which)
    prof = cases.make_profiles("case141", n_days=4)
    B, scale = 64, cases.SCENARIOS["case141"]["action_scale"]
    args = dict(voltage_barrier_type="l1", action_scale=scale, seed=3)
    acts = GC.actions(B, net.n_sgen, scale, T_STEPS, seed=1)
    env = BatchedVoltageControl(net, prof, args, batch=B, env_id_offset=100)
    assert env.dims["lanes_per_env"] == 32
    obs = [env.reset()[0].cpu().numpy().copy()]
    rew, info = [], []
    for t in range(T_STEPS):
        r, _, i = env.step(torch.tensor(acts[t], device=env.device))
        rew.append(r.cpu().numpy().copy()); info.append(i.cpu().numpy().copy()); obs.append(env.obs.cpu().numpy().copy())
    vm = env.get_field("vm").cpu().numpy()
    env.close()
    want = GC.oracle_trajectory(net, prof, args, 100, acts, procs=GC.default_procs())
    assert np.abs(np.array(obs) - want["obs"]).max() < GC.TOL and np.abs(np.array(rew) - want["reward"]).max() < GC.TOL
    assert np.abs(np.array(info) - want["info"]).max() < GC.TOL and np.abs(vm - want["vm"][-1]).max() < GC.TOL
