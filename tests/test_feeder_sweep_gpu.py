"""GPU tier of the feeder sweep: the generated feeders of tests/feeder_cases.py (more families, larger nets, larger
batches than the CPU tier) through ``BatchedVoltageControl`` on the sm_90a build, at every lane count.

* every env against the fp64 oracle: same converged flag and iteration count, voltages to 1e-9; where the two disagree the
  extended-precision reference decides, and only a convergence test that lies on the tolerance may excuse it;
* a fixed sample of envs against the extended-precision reference, with the bounds of the CPU tier;
* one env step (reward, info, observations, voltages) on a shifted net and on a near-nose net against the oracle env.

Nets that must be refused are refused by mapdn_create before any solve launch."""
import multiprocessing as mp
import os

import numpy as np
import pytest
import torch

import feeder_cases as FC
from mapdn_b200.network import ProfileDesc
from oracle.mp_newton import MpNewton
from oracle.pandapower_nr import PandapowerEquivalent
from feeder_cases import LANES, TOL_NR, check_env, refusal_bytes

pytestmark = pytest.mark.gpu

NETS = FC.catalogue("gpu")
FRACTIONS = tuple(np.round(np.linspace(-0.5, 1.05, 32), 4)) + FC.LOADINGS      # 38 envs per net
MP_SAMPLE = tuple(range(len(FRACTIONS) - len(FC.LOADINGS), len(FRACTIONS)))     # the CPU tier's loadings
V_ORACLE = 1e-9


def _reference(item):
    name, net = item
    pf = PandapowerEquivalent(net)
    inp = FC.loadings(net, seed=len(name) + 1000, fractions=FRACTIONS, pf=pf)
    return name, inp, [pf.runpp(*(a[k] for a in inp)) for k in range(len(FRACTIONS))]


def _mp_env(job):
    net, args = job
    return MpNewton(net).run(*args)


def _procs():
    return max(1, min(32, os.cpu_count() or 1))


@pytest.fixture(scope="module")
def references():
    with mp.get_context("fork").Pool(_procs()) as pool:
        out = pool.map(_reference, list(NETS.items()), chunksize=1)
        refs = {name: (inp, ror) for name, inp, ror in out}
        jobs = [(name, k) for name in sorted(NETS) for k in MP_SAMPLE]
        rmp = pool.map(_mp_env, [(NETS[n], tuple(a[k] for a in refs[n][0])) for n, k in jobs], chunksize=1)
    return refs, dict(zip(jobs, rmp))


def _solve(net, inp, lanes):
    from mapdn_b200._capi import MapdnError
    from mapdn_b200.env import BatchedVoltageControl
    try:
        env = BatchedVoltageControl(net, None, dict(voltage_barrier_type="l1"), batch=1, lanes_per_env=lanes)
    except MapdnError as ex:            # an explicit lane count may not fit; the default always must
        need, _, avail = refusal_bytes(str(ex))
        assert lanes != 0 and need > avail, (net.name, lanes)
        return None
    out = env.solve(*inp)
    torch.cuda.synchronize()
    env.close()
    return {k: v.cpu().numpy() for k, v in out.items()}


@pytest.mark.parametrize("name", sorted(NETS))
def test_generated_feeder_on_the_h100_matches_the_oracles(name, references):
    refs, rmp = references
    net = NETS[name]
    inp, ror = refs[name]
    for lanes in LANES:
        out = _solve(net, inp, lanes)
        if out is None:
            continue
        for k, r in enumerate(ror):
            where = (name, lanes, FRACTIONS[k])
            agree = bool(out["converged"][k]) == r.converged and int(out["iterations"][k]) == r.iterations
            if not agree:                # only a convergence test on the tolerance may tell two correct solvers apart
                r_mp = _mp_env((net, tuple(a[k] for a in inp)))
                assert r_mp.ambiguous(TOL_NR), (where, int(out["iterations"][k]), r.iterations, r_mp.norms)
                continue
            if r.converged:
                V = out["vm"][k] * np.exp(1j * np.deg2rad(out["va_deg"][k]))
                assert np.abs(V - r.V).max() < V_ORACLE, where
        for k in MP_SAMPLE:
            if not rmp[name, k].ambiguous(TOL_NR):
                check_env(out, k, rmp[name, k], ror[k], (name, lanes, FRACTIONS[k]))


def test_a_bus_with_258_children_is_refused_on_the_device_build():
    from mapdn_b200._capi import MapdnError
    from mapdn_b200.env import BatchedVoltageControl
    net = FC.feeder(FC.hub(258), seed=5, name="hub258")
    for lanes in LANES:
        with pytest.raises(MapdnError, match="more than 257 children"):
            BatchedVoltageControl(net, None, None, batch=1, lanes_per_env=lanes)


def _profiles(net, seed, scale):
    """Three days of 3-minute rows: the injection pattern of the feeder under a daily load curve and a PV bell, with the
    evening peak at ``scale`` times the pattern."""
    pl, ql, ps, _ = (a for a in FC.loadings(net, seed, fractions=(1.0,)))
    spd, n_days = 480, 3
    T = n_days * spd + 1
    tod = (np.arange(T) % spd) / spd * 24.0
    curve = 0.4 + 0.6 * np.exp(-0.5 * ((tod - 19.0) / 3.0) ** 2)
    bell = np.clip(np.sin((tod - 6.0) / 12.0 * np.pi), 0.0, None)
    return ProfileDesc(pv=bell[:, None] * (4.0 * scale * ps[0])[None, :], load_p=scale * curve[:, None] * pl[0][None, :],
                       load_q=scale * curve[:, None] * ql[0][None, :], steps_per_hour=20, n_days=n_days)


@pytest.mark.parametrize("name,scale", [("random200", 0.5), ("levels_g64", 0.96)])
def test_env_step_on_generated_feeders_matches_the_oracle_env(name, scale):
    """reset + noisy steps through the step kernel, a shifted net at half the nose loading and a net near the nose,
    against VoltageControlOracle env by env."""
    from mapdn_b200.env import BatchedVoltageControl
    from oracle.voltage_control_ref import INFO_KEYS, VoltageControlOracle
    net = NETS[name]
    prof = _profiles(net, seed=len(name) + 1000, scale=scale)
    B = 8
    env = BatchedVoltageControl(net, prof, dict(voltage_barrier_type="l1", seed=3), batch=B)
    ors = [VoltageControlOracle(net, prof, env.args, env_id=i) for i in range(B)]
    obs, _ = env.reset()
    for i, o in enumerate(ors):
        oo, _ = o.reset()
        assert np.abs(np.array(oo) - obs[i].cpu().numpy()).max() < 1e-9
    rng = np.random.default_rng(0)
    for _ in range(3):
        a = rng.uniform(-0.8, 0.8, (B, net.n_sgen))
        r, term, info = env.step(torch.tensor(a, device=env.device))
        torch.cuda.synchronize()
        vm = env.get_field("vm").cpu().numpy()
        for i, o in enumerate(ors):
            ro, to, io = o.step(a[i])
            assert abs(ro - r[i].item()) < 1e-9 and to == bool(term[i].item()), (name, i)
            assert max(abs(io[k] - info[i, j].item()) for j, k in enumerate(INFO_KEYS)) < 1e-9, (name, i)
            assert np.abs(o.g.res.vm_pu - vm[i]).max() < 1e-9, (name, i)
            assert np.abs(np.array(o.get_obs()) - env.obs[i].cpu().numpy()).max() < 1e-9, (name, i)
    env.close()
