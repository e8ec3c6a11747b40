"""GPU tier of the auto-reset step (BatchedVoltageControl.step_autoreset / mapdn_step_autoreset).

At the benchmark batch sizes, an env that calls step_autoreset (A) and one that calls step, then reset(mask = terminated)
(B) give the same step outputs, the same first observation of every new episode and the same env state: bit for bit up to
32 lanes per env, within 1e-10 at 64 / 128 lanes with identical iteration counts, terminated flags and reset outcomes.
Episodes run out of phase and one env diverges. The batched runner and rollout on the real env must give bit-identical
results to the same loops on a proxy that hides step_autoreset (the step + masked reset path), the rollout over two run()
calls with an episode boundary on the last step of the first."""
import pytest
import torch

from mapdn_b200 import cases
from mapdn_b200.env import BatchedVoltageControl
from mapdn_b200.marl_runner import BatchedMarlRunner, DeviceTransitionBuffer
from mapdn_b200.rollout import BatchedRollout, DeviceReplayBuffer
from geometry_cases import FIELDS, overloaded_case
from test_history_gpu import _Recorder

pytestmark = pytest.mark.gpu


def _same(a, b, exact, what):
    if exact:
        assert torch.equal(a.nan_to_num(7.0), b.nan_to_num(7.0)) and torch.equal(a.isnan(), b.isnan()), what
    else:
        assert a.shape == b.shape and torch.equal(a.isnan(), b.isnan()), what
        d = (a.nan_to_num(0.0) - b.nan_to_num(0.0)).abs()
        assert d.numel() == 0 or float(d.max()) <= 1e-10, (what, float(d.max()))


@pytest.mark.parametrize("H", [1, 3])
@pytest.mark.parametrize("name,batch", [("case33", 4096), ("case141", 2048), ("case322", 1024), ("case322", 512)])
def test_benchmark_sizes_autoreset_equals_step_then_reset(name, batch, H):
    net, prof = overloaded_case(name)
    args = dict(voltage_barrier_type="l1", seed=7, action_scale=cases.SCENARIOS[name]["action_scale"], episode_limit=4,
                history=H)
    A = BatchedVoltageControl(net, prof, args, batch=batch)
    Bv = BatchedVoltageControl(net, prof, args, batch=batch)
    exact = A.dims["lanes_per_env"] <= 32
    dev, B, ng = A.device, batch, A.n_agents
    nan = float("nan")
    A.reset_obs = torch.full_like(A.obs, nan)
    A.reset_obs_stacked = torch.full_like(A.obs_stacked, nan) if H > 1 else A.reset_obs
    A.reset(); Bv.reset()
    gen = torch.Generator(device="cpu").manual_seed(1)
    scale = args["action_scale"]
    diverged = ended = 0
    for t in range(11):
        if t == 1:                              # every other env starts over (out of phase); env 3 from row 58, into the overload
            mask = (torch.arange(B, device=dev) % 2).to(torch.uint8)
            start = torch.tensor([[1, 5, 3]], dtype=torch.int32, device=dev).repeat(B, 1)
            start[3] = torch.tensor([0, 2, 18], dtype=torch.int32)
            A.reset(start, mask=mask); Bv.reset(start, mask=mask)
        a = ((torch.rand(B, ng, generator=gen, dtype=torch.float64) * 2 - 1) * scale).to(dev)
        A.reset_obs.fill_(nan); A.reset_obs_stacked.fill_(nan); A.reset_ok.fill_(7)
        n0 = A.launch_count
        ra, ta, ia = A.step_autoreset(a)
        assert A.launch_count == n0 + 1
        rb, tb, ib = [x.clone() for x in Bv.step(a)]
        obs_b, stk_b = Bv.obs.clone(), Bv.obs_stacked.clone()
        Bv.reset_ok.fill_(7)
        Bv.reset(mask=tb, want_state=False)
        assert torch.equal(ta, tb), t
        _same(ra, rb, exact, (t, "reward")); _same(ia, ib, exact, (t, "info"))
        _same(A.obs, obs_b, exact, (t, "obs")); _same(A.obs_stacked, stk_b, exact, (t, "obs_stacked"))
        tm = tb.bool()
        _same(A.reset_obs[tm], Bv.obs[tm], exact, (t, "reset_obs"))
        assert bool(A.reset_obs[~tm].isnan().all()), t
        assert torch.equal(A.reset_ok, Bv.reset_ok), t
        if H > 1:
            _same(A.reset_obs_stacked[tm], Bv.obs_stacked[tm], exact, (t, "reset_obs_stacked"))
            assert bool(A.reset_obs_stacked[~tm].isnan().all()), t
            _same(A.get_obs_stacked(), Bv.get_obs_stacked(), exact, (t, "get_obs_stacked"))
        for k in FIELDS:
            if k in ("steps", "nr_iters", "start_row"):
                assert torch.equal(A.get_field(k), Bv.get_field(k)), (t, k)
            else:
                _same(A.get_field(k), Bv.get_field(k), exact, (t, k))
        _same(A.get_state(), Bv.get_state(), exact, (t, "state"))
        ended += int(tm.sum())
        diverged += int((ib[:, 10] == 1.0).sum())
    assert ended >= 2 * B and diverged > 0, (ended, diverged)
    A.close(); Bv.close()


class _NoAutoReset:
    """The env behind a wrapper that forwards attributes: the loops take the step + masked reset path."""

    def __init__(self, env):
        self.env = env

    def __getattr__(self, k):
        if k == "step_autoreset":
            raise AttributeError(k)
        return getattr(self.env, k)


def _env(H):
    net, prof = overloaded_case("case33", n_days=6)
    args = dict(voltage_barrier_type="l1", seed=4, action_scale=0.8, episode_limit=3, history=H)
    return BatchedVoltageControl(net, prof, args, batch=64)


@pytest.mark.parametrize("H", [1, 3])
def test_runner_and_rollout_bit_identical_with_autoreset(H):
    results = []
    for wrap in (lambda e: e, _NoAutoReset):
        env = _env(H)
        view = wrap(env)
        assert callable(getattr(type(view), "step_autoreset", None)) == (wrap is not _NoAutoReset)
        net = _Recorder(env.n_agents, env.obs_size, env.stacked_obs_size, env.device)
        net.args.max_steps = 8
        buf = DeviceTransitionBuffer(16, env.batch, env.n_agents, env.stacked_obs_size, 1, 8, env.device)
        stat = BatchedMarlRunner(view, net, buf).train_process({})
        runner = dict(stat=stat, inputs=torch.stack(net.inputs), data={k: v.clone() for k, v in buf.data.items()},
                      done=buf.data["done"].sum().item())
        rb = DeviceReplayBuffer(64 * 20, env.n_agents, env.obs_size, env.device)
        w = torch.randn(env.obs_size, 1, dtype=torch.float32, device=env.device, generator=torch.Generator(device=env.device).manual_seed(3))
        ro = BatchedRollout(view, lambda o: torch.tanh(o @ w).squeeze(-1), rb)
        # episodes of 3 steps from the reset end on the last step of the first call: the second call continues them
        first, obs = ro.run(2), ro.run(8)
        roll = dict(first=first, obs=obs, returns=ro.completed_episode_returns(), info_sum=ro.info_sum.clone(),
                    buf={k: getattr(rb, k).clone() for k in ("obs", "action", "reward", "next_obs", "done")})
        results.append((runner, roll))
        env.close()
    (r0, o0), (r1, o1) = results
    assert r0["done"] > 0 and o0["returns"].numel() > 64          # episodes ended inside both loops
    assert r0["stat"] == r1["stat"]
    assert torch.equal(r0["inputs"], r1["inputs"])
    for k in r0["data"]:
        assert torch.equal(r0["data"][k], r1["data"][k]), k
    assert torch.equal(o0["first"], o1["first"]) and torch.equal(o0["obs"], o1["obs"])
    assert torch.equal(o0["returns"], o1["returns"])
    assert torch.equal(o0["info_sum"], o1["info_sum"])
    for k in o0["buf"]:
        assert torch.equal(o0["buf"][k], o1["buf"][k]), k
