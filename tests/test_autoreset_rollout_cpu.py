"""BatchedRollout over successive run() calls, with and without auto-reset, on a CPU stand-in env.

The stand-in draws its observations from one generator in the same order on both paths, so the step + masked reset loop
and the auto-reset loop must give bit-identical observations, buffer and episode returns, also when an episode ends on the
last step of one run() call and the next call continues it."""
import torch

from mapdn_b200.rollout import BatchedRollout, DeviceReplayBuffer


class _Env:
    """The surface of BatchedVoltageControl the rollout touches. The env state `x` is kept apart from the observation
    buffer `obs` (as the device state is from the observation rows); reset(mask) re-draws the masked envs' state."""

    def __init__(self, B=6, n_agents=2, obs_dim=3, episode_limit=3, seed=0):
        self.batch, self.n_agents, self.obs_size, self.episode_limit = B, n_agents, obs_dim, episode_limit
        self.device = torch.device("cpu")
        self.args = dict(action_scale=0.8, action_bias=0.0)
        self.g = torch.Generator().manual_seed(seed)
        self.x = torch.zeros(B, n_agents, obs_dim, dtype=torch.float64)
        self.obs = self.x.clone()
        self.info = torch.zeros(B, 11, dtype=torch.float64)
        self.t = torch.zeros(B, dtype=torch.int64)

    def reset(self, mask=None, want_state=True, **kw):
        m = torch.ones(self.batch, dtype=torch.bool) if mask is None else mask.bool()
        new = torch.rand(self.batch, self.n_agents, self.obs_size, generator=self.g, dtype=torch.float64)
        self.x = torch.where(m[:, None, None], new, self.x)
        self.obs = torch.where(m[:, None, None], self.x, self.obs)
        self.t = torch.where(m, torch.ones_like(self.t), self.t)
        return self.obs, None

    def step(self, a, add_noise=True):
        self.x = self.x * 0.5 + a[:, :, None] + torch.rand(self.x.shape, generator=self.g, dtype=torch.float64)
        self.obs = self.x.clone()
        self.t += 1
        done = (self.t >= self.episode_limit).to(torch.uint8)
        self.info = self.info + 1.0
        return -self.obs.abs().mean(dim=(1, 2)), done, self.info


class _AutoResetEnv(_Env):
    """The same env with step_autoreset: obs keeps the terminal observation, reset_obs gets the new episode's first."""

    def step_autoreset(self, a, add_noise=True):
        reward, done, info = self.step(a, add_noise)
        terminal = self.obs.clone()
        self.reset(mask=done)
        self.reset_obs, self.obs = self.obs, terminal
        return reward, done, info


def _rollout(env_cls, calls):
    env = env_cls()
    w = torch.tensor([[0.7], [-0.4], [0.2]], dtype=torch.float32)
    buf = DeviceReplayBuffer(64, env.n_agents, env.obs_size, env.device)
    ro = BatchedRollout(env, lambda o: torch.tanh(o @ w).squeeze(-1), buf)
    outs = [ro.run(n) for n in calls]
    return outs, ro, buf


def test_successive_runs_resume_the_episodes_with_and_without_autoreset():
    calls = (2, 4, 1, 3)              # from the reset, episodes of 3 steps end on the last step of the first call
    (o0, r0, b0), (o1, r1, b1) = _rollout(_Env, calls), _rollout(_AutoResetEnv, calls)
    assert int(r0._ret_n) > 0 and len(b0) == 6 * sum(calls)
    for x, y in zip(o0, o1):
        assert torch.equal(x, y)
    assert torch.equal(r0.completed_episode_returns(), r1.completed_episode_returns())
    assert torch.equal(r0.episode_return, r1.episode_return) and torch.equal(r0.info_sum, r1.info_sum)
    for k in ("obs", "action", "reward", "next_obs", "done"):
        assert torch.equal(getattr(b0, k), getattr(b1, k)), k

