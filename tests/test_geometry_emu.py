"""CPU tier: the launch geometries of mapdn_create (shared-memory plan, envs per CTA, helper warps, lanes per env and the
rounds of the persistent grid) on the kernel source compiled for the CPU SIMT emulation (tests/emu).

MAPDN_EMU_SMS shrinks the emulated SM count, so a handful of envs runs the planner's benchmark choices (case33 x 4096:
32 envs per CTA; case141 x 2048: 8 envs per CTA and 2 rounds; case322 x 1024: plan 3 - cold tables, loads staged in the
node records - 4 envs per CTA and 2 rounds) and multi-round launches whose last round has idle groups. The overrides
MAPDN_PLAN / MAPDN_EPB / MAPDN_HELPERS force the other plans, CTA sizes and helper counts.

Every geometry asserts that it was in effect (lanes, envs per CTA, shared memory and the grid of every launch), and every
output - reward, terminated, info, obs, state, every get_field field, the tester record rows, Newton iteration counts,
reset_ok, solve and droop - must be bit-identical across the geometries of a net: only addresses may change with the
geometry, never arithmetic. The first geometry of each net is also compared with the oracle env by env, so all of them are.
"""
import os
import sys

import numpy as np
import pytest

import geometry_cases as GC
from conftest import ROOT, random_tree_net
from mapdn_b200 import cases
from mapdn_b200.network import NetDesc, ProfileDesc

sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
from emu_record import EmuRecordEnv                                 # noqa: E402
from oracle.pandapower_nr import PandapowerEquivalent               # noqa: E402
from oracle.voltage_control_ref import INFO_KEYS, VoltageControlOracle   # noqa: E402
from test_emu_kernel import _oracle_droop                           # noqa: E402

OVERRIDES = ("MAPDN_PLAN", "MAPDN_EPB", "MAPDN_HELPERS", "MAPDN_EMU_SMS")


def _random_profile(net, seed, pv_hi, load_hi):
    rng = np.random.default_rng(seed)
    T = 3 * 24 * 20 + 1
    lp = rng.uniform(0.2 * load_hi, load_hi, (T, net.n_load))
    return ProfileDesc(pv=rng.uniform(0, pv_hi, (T, net.n_sgen)), load_p=lp, load_q=lp * rng.uniform(0.2, 0.5, (T, net.n_load)),
                       steps_per_hour=20)


def _hub_net():
    """Six-child hub plus a second hub: the > 2 children path of the sweeps."""
    rng = np.random.default_rng(5)
    f, t, nxt = [0], [1], 2
    for _ in range(6):
        f += [1, nxt, nxt + 1]; t += [nxt, nxt + 1, nxt + 2]; nxt += 3
    for _ in range(4):
        f.append(4); t.append(nxt); nxt += 1
    n = nxt
    return NetDesc(base_mva=1.0, n_bus=n, slack_bus=0, slack_vm=1.0, br_from=f, br_to=t, br_r=rng.uniform(0.002, 0.01, n - 1),
                   br_x=rng.uniform(0.002, 0.01, n - 1), load_bus=np.arange(1, n), sgen_bus=[3, 10, n - 1], sgen_zone=[1, 2, 2],
                   bus_zone=[0] + [1] * 9 + [2] * (n - 10), name="hub")


def _net(name):
    if name == "case141_meshed":   # 2 npq = 280: several rows and columns per lane in the pivot search, update, back substitution
        net = GC.with_ties(cases.make_case("case141"), [(10, 60), (30, 100), (50, 130), (80, 140)], name)
        return net, cases.make_profiles("case141", n_days=3), cases.SCENARIOS["case141"]["action_scale"]
    if name == "general":        # taps, line charging, shunts, scaling, parallel and open branches, slack != 0
        net = random_tree_net(23, 4, seed=11)
        return net, _random_profile(net, 1, 0.5, 0.3), 0.8
    if name == "hub":
        net = _hub_net()
        return net, _random_profile(net, 2, 0.3, 0.05), 0.8
    return cases.make_case(name), cases.make_profiles(name, n_days=3), cases.SCENARIOS[name]["action_scale"]


def _rounds(batch, epb, grid):
    needed = -(-batch // epb)
    return -(-needed // grid)


def _set_geometry(monkeypatch, geom):
    for k in OVERRIDES:
        monkeypatch.delenv(k, raising=False)
    for k, v in geom.items():
        if k in OVERRIDES:
            monkeypatch.setenv(k, str(v))


def _solve_inputs(net, prof, batch, seed):
    rng = np.random.default_rng(seed)
    rows = rng.integers(0, prof.n_rows, batch)
    pv = np.minimum(prof.pv[rows] * rng.uniform(0.5, 1.5, (batch, net.n_sgen)), prof.s_max)     # droop: p <= s_rated
    q = rng.uniform(-0.3, 0.3, (batch, net.n_sgen)) * np.maximum(pv, 0.05 * prof.s_max)
    return prof.load_p[rows], prof.load_q[rows], pv, q


def run_geometry(monkeypatch, name, lanes, batch, geom, n_steps=2, seed=5, droop=True):
    """One trajectory on one geometry; returns (dims, grids, trajectory, solve, droop) - all of it, for the comparisons."""
    net, prof, scale = _net(name)
    _set_geometry(monkeypatch, geom)
    args = dict(voltage_barrier_type="bowl", action_scale=scale, seed=seed)
    env = EmuRecordEnv(net, prof, args, batch=batch, lanes_per_env=lanes, env_id_offset=100)
    try:
        acts = GC.actions(batch, net.n_sgen, scale, n_steps, seed)
        _, R = env.record_layout()
        rec = np.full((batch, n_steps + 1, R), np.nan)
        out = {k: [] for k in ("obs", "state", "iters", "reward", "term", "info")}
        fields = {k: [] for k in GC.FIELDS}
        grids = []

        def snap():
            out["obs"].append(env.obs.copy()); out["state"].append(env.get_state().copy())
            for k in GC.FIELDS:
                fields[k].append(env.get_field(k))
            out["iters"].append(fields["nr_iters"][-1][:, 0].astype(np.int64))
        env.reset_ok[:] = 7
        env.reset()
        grids.append(env.last_grid())
        reset_ok = env.reset_ok.copy()
        env.record(rec[:, 0])
        snap()
        for t in range(n_steps):
            r, tm, info = env.step_record(acts[t], rec[:, t + 1])
            grids.append(env.last_grid())
            out["reward"].append(r.copy()); out["term"].append(tm.copy()); out["info"].append(info.copy())
            snap()
        traj = {k: np.array(v) for k, v in out.items()}
        traj["rec"] = rec.transpose(1, 0, 2).copy()
        traj["fields"] = {k: np.array(v) for k, v in fields.items()}
        traj["reset_ok"] = reset_ok
        ins = _solve_inputs(net, prof, batch, seed)
        sol = env.solve(*ins)
        grids.append(env.last_grid())
        dr = None
        if droop:
            dr = env.droop(ins[0], ins[1], ins[2], prof.s_max)
            grids.append(env.last_grid())
        return dict(dims=env.dims, grids=grids, traj=traj, solve=sol, droop=dr, ins=ins, net=net, prof=prof, args=env.args,
                    acts=acts)
    finally:
        env.close()


def check_oracle(run):
    """Every env of the run against the oracle: the trajectory, the solve and the droop baseline."""
    net, prof, batch = run["net"], run["prof"], run["traj"]["reward"].shape[1]
    assert np.all(run["traj"]["reset_ok"] == 1)
    want = GC.oracle_trajectory(net, prof, run["args"], 100, run["acts"])
    GC.assert_matches_oracle(run["traj"], want)
    pf = PandapowerEquivalent(net)
    sol = run["solve"]
    for e in range(batch):
        r = pf.runpp(*[x[e] for x in run["ins"]])
        assert r.converged and sol["converged"][e] == 1 and sol["iterations"][e] == r.iterations
        assert np.abs(sol["vm"][e] - r.vm_pu).max() < GC.TOL and np.abs(sol["va_deg"][e] - r.va_degree).max() < 1e-8
        assert np.abs(sol["p_bus"][e] - r.p_mw).max() < 1e-8 and np.abs(sol["pl"][e] - r.pl_mw).max() < GC.TOL
    if run["droop"] is not None:
        dr = run["droop"]
        for e in range(batch):
            vm, q, loss, it = _oracle_droop(net, *[x[e] for x in run["ins"][:3]], prof.s_max)
            assert dr["iterations"][e] == it and np.abs(dr["vm"][e] - vm).max() < 1e-8
            assert np.abs(dr["q"][e] - q).max() < 1e-8 and abs(dr["loss"][e] - loss) < 1e-8


def check_identical(a, b, label):
    GC.assert_bit_identical(a["traj"], b["traj"], label)
    GC.assert_bit_identical(a["solve"], b["solve"], label + " solve")
    if a["droop"] is not None:
        GC.assert_bit_identical(a["droop"], b["droop"], label + " droop")


# Per net and lane count: a batch and geometries (overrides + emulated SM count) with what each must produce -
# (envs per CTA, shared memory per CTA, CTAs of every launch, rounds of the persistent loop). None: the planner's choice.
# The four plans of a net at one CTA size differ in two independent amounts (the once-per-step tables, the staged loads),
# which is the witness that a forced plan was not silently dropped (see _assert_plans).
def _plans(sms, epb, helpers=(1, 4, 1, 4)):
    return [dict(MAPDN_EMU_SMS=sms, MAPDN_PLAN=k, MAPDN_EPB=epb, MAPDN_HELPERS=h) for k, h in zip(range(4), helpers)]


MATRIX = {
    # G = 8 sub-warp groups. 132 SMs: 5 CTAs of 8 in one round; 1 SM: the planner's 20 per CTA, case33 x 4096's 32 per
    # CTA and 184 064 B, the four plans at 16, the smallest unit (4): two rounds, the last one ragged
    "case33_G8": dict(net="case33", lanes=0, batch=36, geoms=[
        (dict(), (8, 8, 50432, 5, 1)),
        (dict(MAPDN_EMU_SMS=1), (8, 20, 117248, 1, 2)),
        (dict(MAPDN_EMU_SMS=1, MAPDN_EPB=32), (8, 32, 184064, 1, 2)),
        *zip(_plans(1, 16), [(8, 16, 94976, 2, 2), (8, 16, 86784, 2, 2), (8, 16, 92704, 2, 2), (8, 16, 84512, 2, 2)]),
        (dict(MAPDN_EMU_SMS=1, MAPDN_EPB=4, MAPDN_HELPERS=4), (8, 4, 28160, 5, 2)),
    ]),
    # G = 32, one SM: the planner's 7 per CTA in 3 rounds (the last holds 6 envs: an idle group), case141 x 2048's 8 per
    # CTA and 204 896 B, the four plans at 4 (a 2-CTA grid whose third round leaves one CTA idle), one env per CTA
    "case141_G32": dict(net="case141", lanes=0, batch=20, geoms=[
        (dict(MAPDN_EMU_SMS=1), (32, 7, 182560, 1, 3)),
        (dict(MAPDN_EMU_SMS=1, MAPDN_EPB=8, MAPDN_HELPERS=4), (32, 8, 204896, 1, 3)),
        *zip(_plans(1, 4), [(32, 4, 115552, 2, 3), (32, 4, 110176, 2, 3), (32, 4, 104304, 2, 3), (32, 4, 98928, 2, 3)]),
        (dict(MAPDN_EMU_SMS=1, MAPDN_EPB=1, MAPDN_HELPERS=1), (32, 1, 48544, 4, 5)),
    ]),
    # G = 64 (two-warp groups, named barriers), two SMs: case322 x 1024's plan 3 at 4 per CTA (229 328 B) in 3 rounds
    # (round 3: one env in CTA 0, CTA 1 idle), the planner's 3 per CTA, the four plans at 3, one env per CTA
    "case322_G64": dict(net="case322", lanes=0, batch=17, droop=False, geoms=[
        (dict(MAPDN_EMU_SMS=2, MAPDN_PLAN=3, MAPDN_EPB=4), (64, 4, 229328, 2, 3)),
        (dict(MAPDN_EMU_SMS=2), (64, 3, 220544, 2, 3)),
        *zip(_plans(2, 3), [(64, 3, 220544, 2, 3), (64, 3, 204368, 2, 3), (64, 3, 197904, 2, 3), (64, 3, 181728, 2, 3)]),
        (dict(MAPDN_EMU_SMS=2, MAPDN_EPB=1, MAPDN_HELPERS=1), (64, 1, 114560, 4, 5)),
    ]),
    # G = 128 (four-warp groups), one SM: the planner's 3 per CTA in 4 rounds (the last holds one env), the four plans
    # at 2, one env per CTA in 10 rounds
    "case322_G128": dict(net="case322", lanes=128, batch=10, droop=False, geoms=[
        (dict(MAPDN_EMU_SMS=1), (128, 3, 220208, 1, 4)),
        *zip(_plans(1, 2), [(128, 2, 183232, 1, 5), (128, 2, 172448, 1, 5), (128, 2, 160592, 1, 5), (128, 2, 149808, 1, 5)]),
        (dict(MAPDN_EMU_SMS=1, MAPDN_EPB=1, MAPDN_HELPERS=4), (128, 1, 130080, 1, 10)),
    ]),
    "general_G8": dict(net="general", lanes=0, batch=12, geoms=[
        (dict(MAPDN_EMU_SMS=1), (8, 12, 51648, 1, 1)),
        *zip(_plans(1, 4), [(8, 4, 19776, 3, 1), (8, 4, 18112, 3, 1), (8, 4, 18416, 3, 1), (8, 4, 16752, 3, 1)]),
    ]),
    "general_G32": dict(net="general", lanes=32, batch=12, geoms=[
        (dict(MAPDN_EMU_SMS=1), (32, 6, 30176, 2, 1)),
        (dict(MAPDN_EMU_SMS=1, MAPDN_PLAN=1, MAPDN_EPB=5, MAPDN_HELPERS=4), (32, 5, 24112, 3, 1)),
    ]),
    "hub_G8": dict(net="hub", lanes=0, batch=12, geoms=[
        (dict(MAPDN_EMU_SMS=1), (8, 12, 52640, 1, 1)),
        *zip(_plans(1, 4), [(8, 4, 20128, 3, 1), (8, 4, 18656, 3, 1), (8, 4, 18576, 3, 1), (8, 4, 17104, 3, 1)]),
    ]),
}


def _assert_plans(spec, smem_of):
    """Forced plans 0..3 at one CTA size: hot vs cold tables and scratch vs record staging are two independent savings,
    smem(0) - smem(1) = smem(2) - smem(3) > 0 and smem(0) - smem(2) = smem(1) - smem(3) > 0, so every plan was in effect."""
    plans = {}
    for geom, _ in spec["geoms"]:
        if "MAPDN_PLAN" in geom:
            plans.setdefault(geom["MAPDN_EPB"], {})[geom["MAPDN_PLAN"]] = smem_of[id(geom)]
    for s in plans.values():
        if sorted(s) != [0, 1, 2, 3]:
            continue
        assert s[0] - s[1] == s[2] - s[3] > 0 and s[0] - s[2] == s[1] - s[3] > 0, s


@pytest.mark.parametrize("group", sorted(MATRIX))
def test_geometry_matrix_is_bit_identical_and_matches_the_oracle(monkeypatch, group):
    spec = MATRIX[group]
    ref, smem_of = None, {}
    for geom, want in spec["geoms"]:
        run = run_geometry(monkeypatch, spec["net"], spec["lanes"], spec["batch"], geom, droop=spec.get("droop", True))
        d = run["dims"]
        got = (d["lanes_per_env"], d["envs_per_block"], d["smem_bytes"], run["grids"][0],
               _rounds(spec["batch"], d["envs_per_block"], run["grids"][0]))
        assert got == want, (geom, got, want)
        assert all(g == want[3] for g in run["grids"]), (geom, run["grids"])     # reset, steps, solve, droop
        smem_of[id(geom)] = d["smem_bytes"]
        if ref is None:
            check_oracle(run)
            ref = run
        else:
            check_identical(ref, run, str(geom))
    _assert_plans(spec, smem_of)


def _overload(name):
    """The named case with a profile whose rows 60..459 carry a demand the feeder cannot serve."""
    net, prof = cases.make_case(name), cases.make_profiles(name, n_days=3)
    lp = prof.load_p.copy(); lp[60:460] *= 60.0
    return net, ProfileDesc(pv=prof.pv, load_p=lp, load_q=prof.load_q, steps_per_hour=prof.steps_per_hour, n_days=prof.n_days)


@pytest.mark.parametrize("geom,want", [(dict(MAPDN_EMU_SMS=1), (32, 7, 182560, 1, 2)),
                                       (dict(MAPDN_EMU_SMS=1, MAPDN_PLAN=3, MAPDN_EPB=4, MAPDN_HELPERS=4), (32, 4, 98928, 2, 2))])
def test_diverging_and_never_converging_envs_in_later_rounds(monkeypatch, geom, want):
    """case141 x 14 on one emulated SM. Env 11 (round 2) walks into rows the feeder cannot serve and its second step
    diverges; env 13 (the last env, in the ragged last CTA) then gets a masked reset into those rows whose draws all
    diverge: reset_ok reports it for env 13 only, the other envs are untouched bit for bit and env 13 keeps its power
    flow results. Every other env matches the oracle throughout (env 13 until its failed reset: the reference retries
    such a reset for ever), and both geometries give the same bits, env 13 included."""
    net, prof = _overload("case141")
    B, scale = 14, cases.SCENARIOS["case141"]["action_scale"]
    args = dict(voltage_barrier_type="l1", action_scale=scale, seed=9)
    start = np.array([[1, e % 24, (3 * e) % 20] for e in range(B)], np.int32)       # day 1: clear of the overload
    start[11] = (0, 2, 18)                         # row 58: the reset solves row 59, step 1 loads row 60, step 2 diverges
    _set_geometry(monkeypatch, geom)
    env = EmuRecordEnv(net, prof, args, batch=B, env_id_offset=100)
    d = env.dims
    ors = [VoltageControlOracle(net, prof, env.args, env_id=100 + e) for e in range(B)]
    acts = GC.actions(B, net.n_sgen, scale, 4, seed=2)
    trace = []

    live = list(range(B))

    def compare(label):
        st = env.get_state()
        for e in live:
            o = ors[e]
            assert np.abs(np.array(o.get_obs()) - env.obs[e]).max() < GC.TOL, (label, e)
            assert np.abs(o.get_state() - st[e]).max() < GC.TOL_STATE, (label, e)
        trace.append((env.obs.copy(), st.copy(), np.concatenate([env.get_field(k) for k in GC.FIELDS], axis=1)))

    env.reset(start)
    grid = env.last_grid()
    assert (d["lanes_per_env"], d["envs_per_block"], d["smem_bytes"], grid, _rounds(B, d["envs_per_block"], grid)) == want
    assert -(-12 // d["envs_per_block"]) > grid                     # env 11 runs in round 2
    for e, o in enumerate(ors):
        o.reset(tuple(int(x) for x in start[e]))
    compare("reset")
    destroyed = np.zeros(B, bool)
    for t in range(4):
        if t == 2:
            mask = np.zeros(B, np.uint8); mask[13] = 1
            st2 = start.copy(); st2[13] = (0, 5, 0)                  # row 100: every draw diverges
            before = {k: env.get_field(k) for k in GC.FIELDS}
            b_obs, b_state = env.obs.copy(), env.get_state().copy()
            env.reset_ok[:] = 7
            env.reset(st2, mask=mask)
            assert env.reset_ok[13] == 0 and np.all(env.reset_ok[:13] == 7)
            assert np.array_equal(env.obs[:13], b_obs[:13]) and np.array_equal(env.get_state()[:13], b_state[:13])
            for k in GC.FIELDS:
                after = env.get_field(k)
                assert np.array_equal(after[:13], before[k][:13]), k
                if k in ("vm", "va_deg", "p_bus", "q_bus", "line_loss"):
                    assert np.array_equal(after[13], before[k][13]), k
            live.remove(13)
        r, term, info = env.step(acts[t])
        it = env.get_field("nr_iters")[:, 0]
        trace.append((r.copy(), term.copy(), info.copy()))
        for e in live:
            o = ors[e]
            ro, to, io = o.step(acts[t, e])
            destroyed[e] |= io["destroy"] == 1.0
            assert abs(ro - r[e]) < GC.TOL and to == bool(term[e]), (t, e)
            assert np.abs(np.array([io[k] for k in INFO_KEYS]) - info[e]).max() < GC.TOL, (t, e)
            assert it[e] == (o.g.res.iterations if io["destroy"] == 0.0 else 10), (t, e)
        compare(f"step {t}")
    assert destroyed.tolist() == [e == 11 for e in range(B)]
    env.close()
    key = "awkward"
    if key in _TRACES:
        for a, b in zip(_TRACES[key], trace):
            for x, y in zip(a, b):
                assert np.array_equal(x, y)
    else:
        _TRACES[key] = trace


_TRACES = {}


def test_meshed_case141_dense_fallback_matches_the_oracle(monkeypatch):
    """case141 with four tie lines (2 npq = 280, several rows / columns per lane in every pass of the dense LU) on one
    emulated SM: reset, noisy steps with records, solve and droop, env by env against the oracle's Newton-Raphson."""
    run = run_geometry(monkeypatch, "case141_meshed", 0, 2, dict(MAPDN_EMU_SMS=1))
    d = run["dims"]
    assert d["lanes_per_env"] == 32 and run["grids"][0] * d["envs_per_block"] >= 2
    check_oracle(run)


def test_meshed_net_size_limit_of_the_dense_fallback(monkeypatch):
    """256 PQ buses are accepted (one warp per env, 2 npq = 512); 257 are refused at create with MAPDN_ERR_TOPOLOGY (3)."""
    _set_geometry(monkeypatch, dict(MAPDN_EMU_SMS=1))
    env = EmuRecordEnv(GC.meshed_chain(256), None, dict(voltage_barrier_type="l1"), batch=1)
    assert env.dims["lanes_per_env"] == 32 and env.dims["n_bus"] == 257
    env.close()
    with pytest.raises(RuntimeError, match=r"mapdn status 3: .*more than 256 PQ buses"):
        EmuRecordEnv(GC.meshed_chain(257), None, dict(voltage_barrier_type="l1"), batch=1)


@pytest.mark.parametrize("lanes,cap", [(32, 8), (64, 8), (128, 4)])
def test_envs_per_block_override_is_capped(monkeypatch, lanes, cap):
    """MAPDN_EPB cannot exceed the solver threads the planner's own search allows (256 for G <= 32, 512 above: the
    kernel's launch bounds and the named-barrier ids 3 + group): a small net whose shared memory would allow more."""
    net, prof, _ = _net("hub")
    _set_geometry(monkeypatch, dict(MAPDN_EPB=64))
    env = EmuRecordEnv(net, prof, None, batch=64, lanes_per_env=lanes)
    assert env.dims["lanes_per_env"] == lanes and env.dims["envs_per_block"] == cap
    env.close()
