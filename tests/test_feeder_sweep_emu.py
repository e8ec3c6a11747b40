"""CPU tier of the feeder sweep: the kernel source on the CPU emulation solves generated feeders (tests/feeder_cases.py)
at every lane count, and every env is held to the extended-precision Newton reference (oracle/mp_newton.py).

Two fp64 implementations of the same Newton iteration legitimately drift apart where the iteration is badly conditioned
(near the nose, impedances over decades), so "close to the fp64 oracle" cannot say which of the two is wrong. Against
the mp reference the kernel must be as accurate as the oracle itself: |V - V_mp| <= C_ORACLE * |V_oracle - V_mp| + 1e-12,
besides the absolute bound. Results need not be bit-identical across lane counts: the schedules change the order in
which children are accumulated."""
import multiprocessing as mp
import os
import sys

import numpy as np
import pytest

from conftest import ROOT, random_tree_net
import feeder_cases as FC
from mapdn_b200 import cases
from mapdn_b200.network import NetDesc
from oracle.mp_newton import MpNewton
from oracle.pandapower_nr import PandapowerEquivalent, make_ybus

sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
from emu_env import make_env, nan_filled_outputs                    # noqa: E402,F401  (autouse fixture)

from feeder_cases import LANES, TOL_NR, check_env, refusal_bytes   # noqa: E402

UNSUPPORTED = 4

NETS = FC.catalogue("emu")
MESHED = FC.meshed_catalogue()


def _solve(env, *inputs):
    return {k: v.numpy() for k, v in env.solve(*inputs).items()}


def _reference(item):
    name, net = item
    pf = PandapowerEquivalent(net)
    inp = FC.loadings(net, seed=len(name), pf=pf)
    B = inp[0].shape[0]
    m = MpNewton(net)
    return name, inp, [m.run(*(a[k] for a in inp)) for k in range(B)], [pf.runpp(*(a[k] for a in inp)) for k in range(B)]


@pytest.fixture(scope="module")
def references():
    """{name: (inputs, mp results, fp64 oracle results)} for every generated net, computed over a fork pool."""
    items = list(NETS.items()) + list(MESHED.items())
    with mp.get_context("fork").Pool(max(1, min(8, os.cpu_count() or 1))) as pool:
        out = pool.map(_reference, items, chunksize=1)
    return {name: rest for name, *rest in [(o[0], o[1], o[2], o[3]) for o in out]}


@pytest.mark.parametrize("name", sorted(NETS))
def test_generated_feeder_matches_mp_newton_at_every_lane_count(name, references):
    net = NETS[name]
    inp, rmp, ror = references[name]
    live = [k for k in range(len(rmp)) if not rmp[k].ambiguous(TOL_NR)]
    for lanes in LANES:
        try:
            env = make_env(net, None, dict(voltage_barrier_type="l1"), batch=1, lanes_per_env=lanes)
        except RuntimeError as ex:       # an explicit lane count may not fit; the default always must
            need, _, avail = refusal_bytes(str(ex))
            assert lanes != 0 and need > avail, (name, lanes)
            continue
        try:
            out = _solve(env, *inp)
        finally:
            env.close()
        for k in live:
            check_env(out, k, rmp[k], ror[k], (name, lanes, FC.LOADINGS[k]))


@pytest.mark.parametrize("name", sorted(MESHED))
def test_generated_meshed_feeder_matches_mp_newton(name, references):
    """The dense fallback (one warp per env whatever lanes_per_env asks)."""
    net = MESHED[name]
    inp, rmp, ror = references[name]
    env = make_env(net, None, dict(voltage_barrier_type="l1"), batch=1)
    assert env.dims["lanes_per_env"] == 32
    out = _solve(env, *inp)
    env.close()
    for k in range(len(rmp)):
        if not rmp[k].ambiguous(TOL_NR):
            check_env(out, k, rmp[k], ror[k], (name, FC.LOADINGS[k]))


def test_generated_cases_span_the_loading_range_and_are_rarely_ambiguous(references):
    """The generator places the envs where they test something: near-nose envs need 6+ Newton iterations, envs beyond
    the nose do not converge, and at most 1 % of the cases sit on the convergence threshold."""
    rs = [r for _, rmp, _ in references.values() for r in rmp]
    n_amb = sum(r.ambiguous(TOL_NR) for r in rs)
    assert n_amb <= 0.01 * len(rs), (n_amb, len(rs))
    assert sum(r.converged and r.iterations >= 6 for r in rs) >= 0.2 * len(rs)
    assert sum(not r.converged for r in rs) >= 0.05 * len(rs)


@pytest.mark.parametrize("name", ["random40", "decades4", "hub4", "forest12"])
def test_device_ybus_with_phase_shifters_matches_makeYbus(name):
    """ybus_branch_kernel / ybus_diag_kernel with shifters: Ybus is asymmetric, and Y[i,j] vs Y[j,i] must land right."""
    net = NETS[name]
    assert np.any(net.br_shift != 0)
    env = make_env(net, None, dict(voltage_barrier_type="l1"), batch=1)
    Y, Yo = env.ybus_dense(), make_ybus(net)[0].toarray()
    env.close()
    assert np.abs(Yo - Yo.T).max() > 1e-3 * np.abs(Yo).max()
    assert np.abs(Y - Yo).max() <= 1e-12 * np.abs(Yo).max()
    Ym = MpNewton(net).ybus_dense()
    assert np.abs(Yo - Ym).max() <= 1e-12 * np.abs(Ym).max()


def test_mp_newton_matches_the_fp64_oracle_on_the_golden_nets():
    """The mp reference against the fp64 oracle where both are well conditioned: same iteration counts, differences at
    fp64 rounding level."""
    nets = dict(case33=cases.case33(), case141=cases.case141(), case322=cases.case322(),
                baran_wu=cases.baran_wu_nominal()[0], rand23=random_tree_net(23, 4, seed=11))
    for name, net in nets.items():
        g = np.load(os.path.join(ROOT, "tests", "golden", f"solve_{name}.npz"))
        m, pf = MpNewton(net), PandapowerEquivalent(net)
        for k in range(min(len(g["iterations"]), 2 if net.n_bus > 100 else 4)):
            args = (g["p_load"][k], g["q_load"][k], g["p_pv"][k], g["q"][k])
            r, o = m.run(*args), pf.runpp(*args)
            assert r.converged == o.converged and r.iterations == o.iterations == g["iterations"][k], name
            assert np.abs(MpNewton.complex_V(r) - o.V).max() < 1e-12, name
            assert np.abs(r.p_mw - o.p_mw).max() < 1e-9 and np.abs(r.pl_mw - o.pl_mw).max() < 1e-11, name
            assert len(r.iterates) == r.iterations + 1 and len(r.norms) == r.iterations + 1 and r.norms[-1] < TOL_NR


# ---- the planner: lane counts and refusals ----

def _default_lanes(npq):
    return 8 if npq <= 64 else (32 if npq <= 256 else 64)


def test_default_lane_count_of_accepted_nets_is_unchanged():
    from oracle import ref_scenarios as S
    nets = [cases.make_case(c) for c in ("case33", "case141", "case322")] + [random_tree_net(23, 4, seed=11)]
    nets += [S.SCENARIOS[s]["build"]()[0] for s in sorted(S.SCENARIOS)]
    for net in nets:
        env = make_env(net, None, dict(voltage_barrier_type="l1"), batch=4)
        assert env.dims["lanes_per_env"] == _default_lanes(net.n_bus - 1), net.name
        env.close()


def _chain(n, seed=0):
    return FC.feeder(FC.chain(n), seed=seed, shift=True, name=f"chain{n}")


def test_default_lane_count_falls_back_for_a_deep_feeder():
    """A 400-bus chain does not fit in shared memory at the default 64 lanes (the schedules grow as depth x lanes); with
    lanes_per_env = 0 the planner takes the first lane count that fits, and the solve matches the mp reference."""
    n = 400
    rng = np.random.default_rng(4)
    net = NetDesc(base_mva=1.0, n_bus=n, slack_bus=0, slack_vm=1.0, br_from=np.arange(n - 1), br_to=np.arange(1, n),
                  br_r=rng.uniform(1e-4, 4e-4, n - 1), br_x=rng.uniform(1e-4, 4e-4, n - 1), load_bus=np.arange(1, n),
                  sgen_bus=[n - 1, n // 2], sgen_zone=[1, 1], bus_zone=[0] + [1] * (n - 1), name="chain400")
    with pytest.raises(RuntimeError, match="too large"):
        make_env(net, None, None, batch=1, lanes_per_env=64).close()
    env = make_env(net, None, dict(voltage_barrier_type="l1"), batch=1, lanes_per_env=0)
    assert env.dims["lanes_per_env"] in (4, 8, 16, 32)
    pl = rng.uniform(0.0, 2e-3, (2, net.n_load)) * np.array([[1.0], [4.0]])
    inp = (pl, 0.3 * pl, np.full((2, net.n_sgen), 1e-3), np.zeros((2, net.n_sgen)))
    out = _solve(env, *inp)
    env.close()
    m, pf = MpNewton(net), PandapowerEquivalent(net)
    for k in range(2):
        args = tuple(a[k] for a in inp)
        r = m.run(*args)
        assert r.converged and not r.ambiguous(TOL_NR)
        check_env(out, k, r, pf.runpp(*args), ("chain400", k))


@pytest.mark.parametrize("lanes", [0, 8])
def test_refusal_states_the_bytes_the_smallest_plan_needs(lanes):
    """A net no plan fits: the message names a byte count above the opt-in limit it was refused against."""
    n = 400 if lanes else 1700
    with pytest.raises(RuntimeError) as ex:
        make_env(_chain(n), None, None, batch=1, lanes_per_env=lanes)
    msg = str(ex.value)
    assert f"mapdn status {UNSUPPORTED}" in msg
    need, at, avail = refusal_bytes(msg)
    assert need > avail and avail == 232448 and (lanes == 0 or at == lanes)


@pytest.mark.parametrize("lanes", LANES)
def test_a_bus_with_258_children_is_refused(lanes):
    net = FC.feeder(FC.hub(258), seed=5, name="hub258")
    with pytest.raises(RuntimeError, match=f"mapdn status {UNSUPPORTED}: a bus with more than 257 children"):
        make_env(net, None, None, batch=1, lanes_per_env=lanes)
