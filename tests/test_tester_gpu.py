"""Tester records on the H100: mapdn_step_record / mapdn_record against mapdn_get_field, and BatchedPolicyTester on the
CUDA env against the reference's PGTester (tests/golden/ref_tester.npz, see tests/test_tester_cpu.py)."""
import json

import numpy as np
import pytest
import torch

import tester_cases as TC
from mapdn_b200 import cases
from mapdn_b200.env import BatchedVoltageControl
from mapdn_b200.marl_runner import BatchedPolicyTester

pytestmark = pytest.mark.gpu
FIELDS = ("p_sgen", "q_sgen", "p_bus", "q_bus", "vm", "line_loss")


def _fields(env):
    return torch.cat([env.get_field(k) for k in FIELDS], dim=1)


@pytest.mark.parametrize("name,batch", [("case33", 4096), ("case141", 2048), ("case322", 1024)])
def test_fused_rows_equal_get_field_bit_for_bit(name, batch):
    """The BASELINE batch sizes; the step with records is the step without them (reward, terminated, info, obs)."""
    net, prof = cases.make_case(name), cases.make_profiles(name, n_days=3)
    args = dict(voltage_barrier_type="bowl", action_scale=cases.SCENARIOS[name]["action_scale"], seed=7)
    plain, fused = (BatchedVoltageControl(net, prof, args, batch=batch) for _ in range(2))
    R, T = fused.record_len, 3
    buf = torch.full((batch, T + 1, R + 1), float("nan"), dtype=torch.float64, device=fused.device)
    for e in (plain, fused):
        e.reset(check=True)
    fused.record(buf[:, 0, :R])
    assert torch.equal(buf[:, 0, :R], _fields(fused))
    g = torch.Generator(device=fused.device).manual_seed(3)
    for t in range(T):
        a = (torch.rand(batch, net.n_sgen, generator=g, device=fused.device, dtype=torch.float64) * 2 - 1) * args["action_scale"]
        r0, t0, i0 = [x.clone() for x in plain.step(a)]
        n0 = fused.launch_count
        r1, t1, i1 = fused.step(a, record=buf[:, t + 1, :R])
        assert fused.launch_count == n0 + 1
        if fused.dims["lanes_per_env"] <= 32:
            assert torch.equal(r0, r1) and torch.equal(t0, t1) and torch.equal(i0, i1) and torch.equal(plain.obs, fused.obs)
        else:
            # multi-warp groups: ptxas allocates the record instantiation differently (it spills more), and the Newton
            # iterates of the two separately compiled kernels round differently (measured: <= 4e-11 p.u. / MW, reward
            # <= 6e-14). The rows are the fused kernel's own results, bit for bit (below).
            assert torch.equal(t0, t1) and float((r0 - r1).abs().max()) < 1e-9 and float((i0 - i1).abs().max()) < 1e-9
            assert float((plain.obs - fused.obs).abs().max()) < 1e-9
        assert torch.equal(buf[:, t + 1, :R], _fields(fused)), t
        assert torch.equal(fused.record(torch.empty(batch, R, dtype=torch.float64, device=fused.device)), buf[:, t + 1, :R])
    assert bool(torch.isnan(buf[:, :, R]).all())
    plain.close(); fused.close()


def _gpu_tester(g, name, batch=None):
    case = json.loads(str(g["cases"]))[name]
    net, prof = TC.build(case)
    env = BatchedVoltageControl(net, prof, case["env_args"], batch=batch or case["batch"])
    return case, env, BatchedPolicyTester(env, TC.ReplayPolicy(g, name, case))


@pytest.mark.parametrize("name", ["rnn_day", "mlp_days", "diverge"])
def test_cuda_tester_reproduces_the_reference_records(name):
    g = np.load(TC.GOLDEN)
    case, env, tester = _gpu_tester(g, name)
    n0 = env.launch_count
    records, lengths = tester.test_run(case["days"], hour=case["hour"], interval=case["interval"])
    chunks = -(-len(case["days"]) // env.batch)
    assert env.launch_count - n0 == chunks * (case["max_steps"] + 2)     # per chunk: reset, record, one launch per step
    want_len = g[f"{name}/lengths"]
    assert lengths.tolist() == want_len.tolist()
    for i, w in enumerate(np.split(g[f"{name}/records"], np.cumsum(want_len)[:-1])):
        got = records[i].cpu().numpy()
        assert np.abs(got[:len(w)] - w).max() < 1e-9, i
    assert tester.net.checked == int(want_len.sum() - len(want_len))
    env.close()


def test_cuda_batch_run_reproduces_the_reference_statistics():
    from mapdn_b200._capi import INFO_KEYS
    g = np.load(TC.GOLDEN)
    case, env, tester = _gpu_tester(g, "batch")
    stat = tester.test_batch_run(case["episodes"])
    for k, key in enumerate(INFO_KEYS):
        m, s2 = stat["mean_test_" + key]
        assert abs(m - g["batch/stat"][k, 0]) < 1e-9 and abs(s2 - g["batch/stat"][k, 1]) < 1e-9, key
    env.close()


def test_day_in_a_batch_of_many_days_equals_a_batch_of_one():
    """Day d's record does not depend on the other days of its launch (the reset action is drawn for env 0, episode 1
    in both runs)."""
    from types import SimpleNamespace
    net, prof = cases.make_case("case33"), cases.make_profiles("case33", n_days=6)
    args = dict(voltage_barrier_type="l1", action_scale=0.8, episode_limit=480, reset_action=False, seed=1)

    class Policy:                               # a deterministic policy of the observation (same interface as the models)
        def __init__(self, n):
            self.args = SimpleNamespace(max_steps=40, action_scale=0.8, action_bias=0.0)
            self.policy_dicts = [SimpleNamespace(init_hidden=lambda: torch.zeros(1, n, 4))]

        def get_actions(self, state, status, exploration, actions_avail, target, last_hid):
            a = torch.tanh(state.sum(dim=2, keepdim=True) - state.mean(dim=(1, 2), keepdim=True)) * 0.5
            return a, None, None, None, last_hid + 1.0
    days = [4, 0, 3, 1, 2]
    many_env = BatchedVoltageControl(net, prof, args, batch=len(days))
    many, n_many = BatchedPolicyTester(many_env, Policy(net.n_sgen)).test_run(days)
    for k in (0, 3):
        one_env = BatchedVoltageControl(net, prof, args, batch=1)
        one, n_one = BatchedPolicyTester(one_env, Policy(net.n_sgen)).test_run([days[k]])
        assert int(n_one[0]) == int(n_many[k]) == 41
        assert torch.equal(one[0], many[k])
        one_env.close()
    many_env.close()
