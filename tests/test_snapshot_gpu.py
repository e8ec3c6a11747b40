"""GPU tier of env state snapshots (BatchedVoltageControl.snapshot / restore / fork, mapdn_snapshot / mapdn_restore).

At the benchmark batch sizes, with and without observation history: restoring a snapshot replays the following noisy
auto-reset steps bit for bit (episode ends, a diverged power flow, the ring wrap), a fork gives every copy the source's
first step, and one handle restored as two shards continues bit for bit. A checkpoint file restores into a fresh handle,
and BatchedRollout / BatchedMarlRunner resumed from a checkpoint equal the uninterrupted runs."""
import os

import pytest
import torch

from mapdn_b200 import cases
from mapdn_b200.env import BatchedVoltageControl, EnvSnapshot
from mapdn_b200.marl_runner import BatchedMarlRunner, DeviceTransitionBuffer, attach
from mapdn_b200.rollout import BatchedRollout, DeviceReplayBuffer
from geometry_cases import FIELDS, overloaded_case

pytestmark = pytest.mark.gpu


def _eq(a, b, what):
    assert a.shape == b.shape and torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(7.0), b.nan_to_num(7.0)), what


def _step(env, a):
    """step_autoreset; returns copies of every output (the reset rows of the other envs are not written: masked)."""
    r, t, i = env.step_autoreset(a)
    m = t.bool()
    out = dict(reward=r.clone(), term=t.clone(), info=i.clone(), obs=env.obs.clone(), reset_ok=torch.where(m, env.reset_ok, 7),
               reset_obs=torch.where(m[:, None, None], env.reset_obs, 0.0))
    if env.history > 1:
        out.update(obs_stacked=env.obs_stacked.clone(),
                   reset_obs_stacked=torch.where(m[:, None, None], env.reset_obs_stacked, 0.0))
    return out


def _getters(env):
    d = {k: env.get_field(k) for k in FIELDS}
    d.update(obs=env.get_obs().clone(), state=env.get_state().clone(), stacked=env.get_obs_stacked().clone())
    return d


def _env(name, batch, H, offset=0, **kw):
    net, prof = overloaded_case(name)
    args = dict(voltage_barrier_type="l1", seed=7, action_scale=cases.SCENARIOS[name]["action_scale"], episode_limit=4,
                history=H)
    return BatchedVoltageControl(net, prof, args, batch=batch, env_id_offset=offset, **kw)


def _start(env, diverge_env=1):
    """Sampled reset, env `diverge_env` restarted at row 58: its second step runs into the overload."""
    env.reset()
    start = torch.tensor([[1, 5, 3]], dtype=torch.int32, device=env.device).repeat(env.batch, 1)
    start[diverge_env] = torch.tensor([0, 2, 18], dtype=torch.int32)
    mask = torch.zeros(env.batch, dtype=torch.uint8, device=env.device); mask[diverge_env] = 1
    env.reset(start, mask=mask)


@pytest.mark.parametrize("H", [1, 3])
@pytest.mark.parametrize("name,batch", [("case33", 4096), ("case141", 2048), ("case322", 1024), ("case322", 512)])
def test_replay_fork_and_reshard_at_benchmark_sizes(name, batch, H):
    env = _env(name, batch, H)
    B, ng, dev = batch, env.n_agents, env.device
    g = torch.Generator(device=dev).manual_seed(3)
    scale = cases.SCENARIOS[name]["action_scale"]
    act = lambda: ((torch.rand(B, ng, generator=g, device=dev, dtype=torch.float64) * 2 - 1) * scale).contiguous()
    _start(env)
    _step(env, act())
    # replay: M steps from a snapshot, restore, the same M actions again
    snap = env.snapshot()
    assert snap.data.shape == (B, env.snapshot_layout[-1]) and torch.equal(snap.env_ids, torch.arange(B))
    before = _getters(env)
    acts = [act() for _ in range(6)]
    first = [_step(env, a) for a in acts]
    assert sum(int(o["term"].sum()) for o in first) >= B and sum(int((o["info"][:, 10] == 1).sum()) for o in first) > 0
    after = _getters(env)
    n0 = env.launch_count
    slots = env.restore(snap)
    assert torch.equal(slots, torch.arange(B)) and env.launch_count == n0 + 3 + (H > 1)     # restore + obs/state/stacked
    for k, v in _getters(env).items():
        _eq(v, before[k], ("restored", k))
    for t, a in enumerate(acts):
        for k, v in _step(env, a).items():
            _eq(v, first[t][k], ("replay", t, k))
    for k, v in _getters(env).items():
        _eq(v, after[k], ("end of the replay", k))
    # resharding: the snapshot into two handles of B / 2 (global ids 0.. and B / 2..), both continue like the whole
    halves = [_env(name, B // 2, H, offset=o) for o in (0, B // 2)]
    for h in halves:
        h.reset()
        assert torch.equal(h.restore(snap), torch.arange(B // 2))
    env.restore(snap)
    for t, a in enumerate(acts[:4]):
        want = _step(env, a)
        got = [_step(h, a[i * (B // 2):(i + 1) * (B // 2)].contiguous()) for i, h in enumerate(halves)]
        for k in want:
            _eq(torch.cat([x[k] for x in got]), want[k], ("shards", t, k))
    for h in halves:
        h.close()
    # fork: env 5 into every slot; the first step gives the source's reward, info and voltages everywhere
    src = 5
    row = env.snapshot([src])
    a = acts[0][src:src + 1].repeat(B, 1).contiguous()
    env.fork([src] * B, torch.arange(B))
    r, _, info = [x.clone() for x in env.step(a)]                       # a plain step: res_vm is this step's power flow
    vm = env.get_field("vm")
    env.restore(row, [src])
    r_src, _, i_src = env.step(a)
    assert torch.equal(r, r_src[src].expand(B)) and torch.equal(info, i_src[src].expand(B, -1))
    assert torch.equal(vm, env.get_field("vm")[src].expand(B, -1))
    env.close()


def test_checkpoint_file_into_a_fresh_handle(tmp_path):
    env = _env("case33", 512, 3)
    _start(env)
    a = torch.rand(512, env.n_agents, dtype=torch.float64, device=env.device) - 0.5
    _step(env, a)
    path = os.path.join(tmp_path, "env.pt")
    torch.save(dict(env=env.snapshot().state_dict()), path)
    fresh = _env("case33", 512, 3)
    assert fresh.fingerprint == env.fingerprint
    fresh.restore(EnvSnapshot.from_state_dict(torch.load(path, weights_only=True)["env"]))
    want = _getters(env)
    for k, v in _getters(fresh).items():
        _eq(v, want[k], k)
    for _ in range(5):
        a = torch.rand(512, env.n_agents, dtype=torch.float64, device=env.device) - 0.5
        x, y = _step(env, a), _step(fresh, a)
        for k in x:
            _eq(y[k], x[k], k)
    other = BatchedVoltageControl(cases.make_case("case33"), cases.make_profiles("case33", n_days=4), dict(seed=7, history=3),
                                  batch=512)
    with pytest.raises(ValueError, match="another net"):
        other.restore(EnvSnapshot.from_state_dict(torch.load(path, weights_only=True)["env"]))
    env.close(); fresh.close(); other.close()


def _rollout():
    env = _env("case33", 1024, 1)
    w = torch.linspace(-1, 1, env.obs_size, device=env.device, dtype=torch.float32)
    buf = DeviceReplayBuffer(4 * 1024, env.n_agents, env.obs_size, env.device)
    return env, buf, BatchedRollout(env, lambda o: torch.tanh(o @ w), buf, keep_returns=2048)


def test_rollout_resumes_from_a_checkpoint(tmp_path):
    n1, n2 = 3, 6
    env, buf, ro = _rollout()
    ref = ro.run(n1 + n2)
    env2, buf2, ro2 = _rollout()
    ro2.run(n1)
    path = os.path.join(tmp_path, "ro.pt")
    torch.save(ro2.state_dict(), path)
    env2.close()
    env3, buf3, ro3 = _rollout()
    ro3.load_state_dict(torch.load(path, weights_only=True))
    assert torch.equal(ro3._obs, ro2._obs)                             # re-gathered == the kept observation
    out = ro3.run(n2)
    assert torch.equal(out, ref)
    assert int(ro._ret_n) > 1024 and torch.equal(ro3.completed_episode_returns(), ro.completed_episode_returns())
    assert torch.equal(ro3.episode_return, ro.episode_return) and torch.equal(ro3.info_sum, ro.info_sum)
    for k in ("obs", "action", "reward", "next_obs", "done"):
        assert torch.equal(getattr(buf3, k), getattr(buf, k)), k
    assert (buf3.head, buf3.count) == (buf.head, buf.count)
    env.close(); env3.close()


def _runner():
    from test_gpu_round2 import _TinyActorCritic
    net, prof = cases.make_case("case33"), cases.make_profiles("case33", n_days=4)
    env = BatchedVoltageControl(net, prof, dict(voltage_barrier_type="bowl", seed=3, episode_limit=6), batch=256)
    torch.manual_seed(0)
    model = attach(_TinyActorCritic(env.n_agents, env.obs_size, 32, env.device))
    buf = DeviceTransitionBuffer(16, 256, env.n_agents, env.obs_size, 1, 32, env.device)
    return env, BatchedMarlRunner(env, model, buf)


def test_marl_runner_resumes_from_a_checkpoint(tmp_path):
    env, runner = _runner()
    runner.train_process({})
    torch.manual_seed(11)
    want = runner.train_process({})
    env2, r2 = _runner()
    r2.train_process({})
    path = os.path.join(tmp_path, "runner.pt")
    torch.save(r2.state_dict(), path)
    env2.close()
    env3, r3 = _runner()
    r3.load_state_dict(torch.load(path, weights_only=True))
    torch.manual_seed(11)
    got = r3.train_process({})
    assert got == want
    assert (r3.steps, r3.episodes) == (runner.steps, runner.episodes)
    assert (r3.buffer.head, r3.buffer.count) == (runner.buffer.head, runner.buffer.count)
    for k, v in runner.buffer.data.items():
        assert torch.equal(r3.buffer.data[k], v), k
    assert torch.equal(env3.get_field("start_row"), env.get_field("start_row"))    # the sampled starts follow the episode counters
    env.close(); env3.close()
