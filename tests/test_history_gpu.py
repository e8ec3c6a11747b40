"""GPU tier of the observation history (reference get_obs :303-315): the reference's own stacked rows through
BatchedVoltageControl, the stacked rows of the benchmark batch sizes against the stacking rule and the standalone gather
(bit for bit), history as a pure side output, and the batched runner / tester feeding the learner the stacked frames."""
import json
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from conftest import ROOT
from geometry_cases import FIELDS
from mapdn_b200 import cases
from mapdn_b200.env import BatchedVoltageControl
from mapdn_b200.marl_runner import BatchedMarlRunner, BatchedPolicyTester
from oracle import ref_scenarios as S

pytestmark = pytest.mark.gpu


def stacking_rule(frames, H):
    """frames: [B] lists of the frames [n_agents, obs_dim] since each env's last reset -> [B, n_agents, H * obs_dim]."""
    B = len(frames)
    out = torch.zeros(B, frames[0][0].shape[0], H * frames[0][0].shape[1], dtype=torch.float64, device=frames[0][0].device)
    od = frames[0][0].shape[1]
    for b in range(B):
        for k, f in enumerate(frames[b][-H:][::-1]):
            out[b, :, (H - 1 - k) * od:(H - k) * od] = f
    return out


def test_reference_history_fixture_full_stacked_rows():
    """The reference's stacked rows (frames per reset / step: test_history_emu.reference_rows_one_frame_per_transition)."""
    from test_history_emu import reference_rows_one_frame_per_transition
    g = np.load(S.fixture_path(ROOT, "case33_history"))
    ops = [tuple(op) for op in json.loads(str(g["ops"]))]
    sc = S.SCENARIOS["case33_history"]
    net, prof = sc["build"]()
    env = BatchedVoltageControl(net, prof, sc["args"], batch=1)
    H = sc["args"]["history"]
    assert env.history == H and env.stacked_obs_size == H * env.obs_size == g["obs"].shape[-1]
    assert env.get_env_info()["obs_shape"] == env.obs_size
    want = reference_rows_one_frame_per_transition(g, ops, H, env.obs_size)
    t = 0
    for k_op, op in enumerate(ops):
        if op[0] == "step":
            env.step(torch.tensor(g["actions"][t], device=env.device), add_noise=op[1])
            t += 1
        else:
            env.reset()
        fused = env.obs_stacked[0].cpu().numpy()
        assert np.abs(fused - want[k_op]).max() < 1e-9, (k_op, op)
        assert np.array_equal(env.get_obs_stacked()[0].cpu().numpy(), fused)
    env.close()


@pytest.mark.parametrize("name,batch", [("case33", 4096), ("case141", 2048), ("case322", 1024)])
def test_benchmark_sizes_stacked_rows_and_pure_side_output(name, batch):
    H = 3
    net, prof = cases.make_case(name), cases.make_profiles(name, n_days=4)
    args = dict(voltage_barrier_type="l1", seed=7, action_scale=cases.SCENARIOS[name]["action_scale"])
    plain = BatchedVoltageControl(net, prof, args, batch=batch)
    hist = BatchedVoltageControl(net, prof, dict(args, history=H), batch=batch)
    exact = hist.dims["lanes_per_env"] <= 32
    dev, B, ng = hist.device, batch, hist.n_agents

    def same(a, b, what):
        if exact:
            assert torch.equal(a, b), what
        else:
            assert a.shape == b.shape and float((a - b).abs().max()) <= 1e-10, (what, float((a - b).abs().max()))

    plain.reset(); hist.reset()
    same(plain.obs, hist.obs, "reset obs")
    frames = [[hist.obs[b].clone()] for b in range(B)]
    assert torch.equal(hist.obs_stacked, stacking_rule(frames, H))
    gen = torch.Generator(device="cpu").manual_seed(1)
    rec0 = torch.full((B, plain.record_len), float("nan"), dtype=torch.float64, device=dev)
    rec1 = rec0.clone()
    scale = args["action_scale"]
    for t in range(H + 4):
        if t == H + 2:                                   # mid-episode masked reset of every 8th env
            mask = (torch.arange(B, device=dev) % 8 == 3).to(torch.uint8)
            plain.reset(mask=mask); hist.reset(mask=mask)
            same(plain.obs, hist.obs, "masked reset obs")
            for b in torch.nonzero(mask).flatten().tolist():
                frames[b] = [hist.obs[b].clone()]
            assert torch.equal(hist.obs_stacked, stacking_rule(frames, H))
        a = ((torch.rand(B, ng, generator=gen, dtype=torch.float64) * 2 - 1) * scale).to(dev)
        r0, t0, i0 = [x.clone() for x in plain.step(a, record=rec0)]
        r1, t1, i1 = hist.step(a, record=rec1)
        same(r0, r1, "reward"); assert torch.equal(t0, t1); same(i0, i1, "info")
        same(plain.obs, hist.obs, "obs"); same(rec0, rec1, "record")
        for b in range(B):
            frames[b].append(hist.obs[b].clone())
        want = stacking_rule(frames, H)
        assert torch.equal(hist.obs_stacked, want), t
        assert torch.equal(hist.get_obs_stacked(), want), t
    for k in FIELDS:
        same(plain.get_field(k), hist.get_field(k), k)
    same(plain.get_state(), hist.get_state(), "state")
    plain.close(); hist.close()


class _Recorder:
    """A tiny actor-critic with the reference Model's interface that records every learner input. Its action depends
    on the newest frame only, so runs with and without history take the same actions."""

    def __init__(self, n, obs_dim, width, device):
        torch.manual_seed(0)
        self.args = SimpleNamespace(max_steps=6, action_scale=0.8, action_bias=0.0, hid_size=8, num_eval_episodes=4)
        self.n, self.od, self.width = n, obs_dim, width
        self.w = torch.randn(obs_dim, 1, device=device) * 0.05
        self.q = torch.nn.Linear((width + 1) * n, 1).to(device)
        self.policy_dicts = [SimpleNamespace(init_hidden=lambda: torch.zeros(1, n, 8, device=device))]
        self.inputs = []

    def get_actions(self, state, status, exploration, actions_avail, target=False, last_hid=None):
        assert state.shape[-1] == self.width
        self.inputs.append(state.clone())
        act = torch.tanh(state[..., -self.od:] @ self.w)
        return act, act, torch.zeros_like(act), act, last_hid

    def value(self, obs, act):
        B = obs.shape[0]
        return self.q(torch.cat([obs.reshape(B, -1), act.reshape(B, -1)], dim=-1)).view(B, 1, 1).expand(-1, self.n, -1)


def _history_pair(B, **kw):
    net, prof = cases.make_case("case33"), cases.make_profiles("case33", n_days=6)
    args = dict(voltage_barrier_type="l1", seed=4, action_scale=0.8, **kw)
    return (BatchedVoltageControl(net, prof, args, batch=B), BatchedVoltageControl(net, prof, dict(args, history=3), batch=B))


class _StackedView:
    """Wraps an env with history: every reset / step also appends the stacked rows the env holds afterwards."""

    def __init__(self, env):
        self.env, self.seen = env, []

    def __getattr__(self, k):
        return getattr(self.env, k)

    def reset(self, *a, **kw):
        out = self.env.reset(*a, **kw)
        self.seen.append(self.env.get_obs_stacked().to(torch.float32))
        return out

    def step(self, *a, **kw):
        out = self.env.step(*a, **kw)
        self.seen.append(self.env.get_obs_stacked().to(torch.float32))
        return out


def test_runner_and_tester_feed_the_stacked_frames():
    B = 16
    one, three = _history_pair(B, episode_limit=4)
    view = _StackedView(three)
    net = _Recorder(three.n_agents, three.obs_size, three.stacked_obs_size, three.device)
    runner = BatchedMarlRunner(view, net)
    runner.train_process({})
    # train_process: state (initial), next state per step (two get_actions per step), state after the masked resets
    assert len(net.inputs) == 2 * net.args.max_steps
    seen = view.seen
    assert torch.equal(net.inputs[0], seen[0])
    for t in range(net.args.max_steps):
        nxt = seen[1 + 2 * t]                              # after step t
        assert torch.equal(net.inputs[1 + 2 * t], nxt)      # next_state
        if t + 1 < net.args.max_steps:
            after_reset = seen[2 + 2 * t]                  # the masked reset of the envs that terminated
            assert torch.equal(net.inputs[2 + 2 * t], after_reset), t
    assert net.inputs[0].shape == (B, three.n_agents, 3 * three.obs_size)
    net.inputs.clear(); view.seen.clear()
    runner.evaluation({}, num_eval_episodes=B)
    assert all(torch.equal(x, s) for x, s in zip(net.inputs, view.seen))
    one.close(); three.close()
    # the tester on fresh envs (the reset action is drawn per episode): the same policy on history = 1 and history = 3
    # envs writes the same records
    one, three = _history_pair(B, episode_limit=4)
    recs = []
    for env in (one, three):
        pol = _Recorder(env.n_agents, env.obs_size, env.stacked_obs_size, env.device)
        rec, n = BatchedPolicyTester(env, pol).test_run([0, 1, 2, 3])
        recs.append((rec, n))
        if env is three:
            assert all(x.shape[-1] == 3 * env.obs_size for x in pol.inputs)
    assert torch.equal(recs[0][1], recs[1][1]) and torch.equal(recs[0][0].nan_to_num(7.0), recs[1][0].nan_to_num(7.0))
    one.close(); three.close()
