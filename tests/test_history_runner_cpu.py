"""BatchedMarlRunner and BatchedPolicyTester hand the learner the stacked frames of an env with observation history
(``history > 1``: ``env.obs_stacked``, reference get_obs :303-315) - after the first reset, after every step, after the
masked reset of the envs that ended, in evaluation and in both tester runs. CPU stand-ins only."""
from types import SimpleNamespace

import torch

from mapdn_b200.marl_runner import BatchedMarlRunner, BatchedPolicyTester

B, N, OD, H = 4, 3, 5, 3


class HistoryEnv:
    """CPU stand-in with the surface of a BatchedVoltageControl with history: ``obs`` holds the newest frame and
    ``obs_stacked`` the last H frames (a fresh random frame per reset / step, stacked per env)."""

    def __init__(self, episode_limit=3, seed=0):
        self.batch, self.n_agents, self.n_actions, self.obs_size = B, N, 1, OD
        self.history, self.stacked_obs_size, self.device = H, H * OD, torch.device("cpu")
        self.g = torch.Generator().manual_seed(seed)
        self.obs = torch.zeros(B, N, OD, dtype=torch.float64)
        self.obs_stacked = torch.zeros(B, N, H * OD, dtype=torch.float64)
        self.t = torch.zeros(B, dtype=torch.int64)
        self.episode_limit = episode_limit
        self.record_len = 2

    def _frame(self, m):
        new = torch.rand(B, N, OD, generator=self.g, dtype=torch.float64)
        self.obs = torch.where(m[:, None, None], new, self.obs)
        shifted = torch.cat([self.obs_stacked[:, :, OD:], self.obs], dim=2)
        self.obs_stacked = torch.where(m[:, None, None], shifted, self.obs_stacked)

    def reset(self, start=None, mask=None, want_state=True, **kw):
        m = torch.ones(B, dtype=torch.bool) if mask is None else mask.bool()
        self.obs_stacked = torch.where(m[:, None, None], torch.zeros_like(self.obs_stacked), self.obs_stacked)
        self._frame(m)
        self.t = torch.where(m, torch.ones_like(self.t), self.t)
        return self.obs, None

    def step(self, a, add_noise=True, record=None):
        self._frame(torch.ones(B, dtype=torch.bool))
        self.t += 1
        if record is not None:
            record.fill_(1.0)
        done = (self.t >= self.episode_limit).to(torch.uint8)
        return -a.abs().mean(dim=1), done, torch.zeros(B, 11, dtype=torch.float64)

    def record(self, out):
        return out.fill_(0.0)


class Learner:
    """Records every input of get_actions / value."""

    def __init__(self):
        self.args = SimpleNamespace(max_steps=5, action_scale=0.8, action_bias=0.0, hid_size=2, num_eval_episodes=B)
        self.policy_dicts = [SimpleNamespace(init_hidden=lambda: torch.zeros(1, N, 2))]
        self.inputs, self.values = [], []

    def get_actions(self, state, status, exploration, actions_avail, target=False, last_hid=None):
        self.inputs.append(state.clone())
        act = torch.tanh(state.sum(dim=2, keepdim=True))
        return act, act, torch.zeros_like(act), act, last_hid

    def value(self, obs, act):
        self.values.append(obs.clone())
        return obs.sum(dim=2, keepdim=True)


class Watch:
    """Forwards to the env and keeps the stacked rows it holds after every reset / step."""

    def __init__(self, env):
        self.env, self.seen = env, []

    def __getattr__(self, k):
        return getattr(self.env, k)

    def reset(self, *a, **kw):
        out = self.env.reset(*a, **kw)
        self.seen.append(self.env.obs_stacked.to(torch.float32))
        return out

    def step(self, *a, **kw):
        out = self.env.step(*a, **kw)
        self.seen.append(self.env.obs_stacked.to(torch.float32))
        return out


def test_train_process_and_evaluation_feed_the_stacked_frames():
    env, net = Watch(HistoryEnv()), Learner()
    BatchedMarlRunner(env, net).train_process({})
    T = net.args.max_steps
    assert len(net.inputs) == 2 * T and all(x.shape == (B, N, H * OD) for x in net.inputs)
    assert torch.equal(net.inputs[0], env.seen[0])                               # initial state
    for t in range(T):
        assert torch.equal(net.inputs[2 * t + 1], env.seen[2 * t + 1])          # next_state
        assert torch.equal(net.values[2 * t + 1], env.seen[2 * t + 1])
        if t + 1 < T:                                                            # state after the masked reset
            assert torch.equal(net.inputs[2 * t + 2], env.seen[2 * t + 2])
    # episode_limit 3: the envs ended after their second step, and the rows after the masked reset start a new episode
    fresh = env.seen[4]
    assert float(fresh[:, :, :(H - 1) * OD].abs().max()) == 0.0 and float(env.seen[3][:, :, :OD].abs().min()) > 0.0
    net.inputs.clear(); env.seen.clear()
    BatchedMarlRunner(env, net).evaluation({})
    assert len(net.inputs) == T and all(torch.equal(x, s) for x, s in zip(net.inputs, env.seen))


def test_tester_runs_feed_the_stacked_frames():
    env, net = Watch(HistoryEnv(episode_limit=10)), Learner()
    tester = BatchedPolicyTester(env, net)
    tester.test_run([0, 1, 2, 3])
    assert len(net.inputs) == net.args.max_steps and all(torch.equal(x, s) for x, s in zip(net.inputs, env.seen))
    assert net.inputs[0].shape == (B, N, H * OD)
    net.inputs.clear(); env.seen.clear()
    tester.test_batch_run(num_episodes=B)
    assert len(net.inputs) == net.args.max_steps and all(torch.equal(x, s) for x, s in zip(net.inputs, env.seen))


def test_envs_without_history_still_feed_obs():
    env, net = Watch(HistoryEnv()), Learner()
    env.env.history = 1
    BatchedMarlRunner(env, net).train_process({})
    assert all(x.shape == (B, N, OD) for x in net.inputs)
