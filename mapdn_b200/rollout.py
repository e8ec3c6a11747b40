"""Batched rollout adapter + device replay buffer (SURVEY §8 f2).

The reference collects experience one env at a time (``models/model.py:197-263``: ``view(1, n, obs)``,
``translate_action`` -> numpy -> ``env.step``) and stores transitions in Python lists
(``utilities/replay_buffer.py``). Here B envs step in lock-step on the GPU and transitions go into
a ring buffer in HBM, so a learner consumes B env-steps per Python iteration with no host copy.
"""
from __future__ import annotations

from typing import Callable, Optional

import torch

__all__ = ["translate_action", "DeviceReplayBuffer", "BatchedRollout"]


def translate_action(action: torch.Tensor, action_scale: float, action_bias: float) -> torch.Tensor:
    """Continuous branch of reference ``utilities/util.py:123-132``: clamp the policy output to
    [-1, 1] and map it affinely onto [bias - scale, bias + scale]. Returns fp64 (the env's dtype)."""
    cp = torch.clamp(action, min=-1.0, max=1.0)
    low, high = action_bias - action_scale, action_bias + action_scale
    return (0.5 * (cp + 1.0) * (high - low) + low).to(torch.float64)


class DeviceReplayBuffer:
    """Transition ring buffer on the GPU (reference ``TransReplayBuffer``, replay_buffer.py:7-30:
    FIFO of capacity ``size``, uniform sampling without replacement when possible)."""

    def __init__(self, size: int, n_agents: int, obs_dim: int, device, obs_dtype=torch.float32):
        self.size, self.device = int(size), device
        self.obs = torch.zeros(size, n_agents, obs_dim, dtype=obs_dtype, device=device)
        self.next_obs = torch.zeros_like(self.obs)
        self.action = torch.zeros(size, n_agents, dtype=torch.float32, device=device)
        self.reward = torch.zeros(size, dtype=torch.float32, device=device)
        self.done = torch.zeros(size, dtype=torch.bool, device=device)
        self.head, self.count = 0, 0

    def add_batch(self, obs, action, reward, next_obs, done):
        B = obs.shape[0]
        if B > self.size:
            raise ValueError(f"a batch of {B} transitions does not fit a buffer of {self.size} (duplicate ring indices)")
        idx = (self.head + torch.arange(B, device=self.device)) % self.size
        self.obs[idx] = obs.to(self.obs.dtype)
        self.next_obs[idx] = next_obs.to(self.obs.dtype)
        self.action[idx] = action.to(torch.float32)
        self.reward[idx] = reward.to(torch.float32)
        self.done[idx] = done.to(torch.bool)
        self.head = (self.head + B) % self.size
        self.count = min(self.size, self.count + B)

    def __len__(self):
        return self.count

    _FIELDS = ("obs", "next_obs", "action", "reward", "done")

    def state_dict(self) -> dict:
        return dict({k: getattr(self, k) for k in self._FIELDS}, head=self.head, count=self.count)

    def load_state_dict(self, d: dict):
        for k in self._FIELDS:
            if tuple(d[k].shape) != tuple(getattr(self, k).shape):
                raise ValueError(f"replay buffer {k}: checkpoint shape {tuple(d[k].shape)}, "
                                 f"buffer {tuple(getattr(self, k).shape)}")
            getattr(self, k).copy_(d[k])
        self.head, self.count = int(d["head"]), int(d["count"])

    def sample(self, batch_size: int, generator: Optional[torch.Generator] = None):
        n = min(batch_size, self.count)
        idx = torch.randperm(self.count, device=self.device, generator=generator)[:n]
        return dict(obs=self.obs[idx], action=self.action[idx], reward=self.reward[idx],
                    next_obs=self.next_obs[idx], done=self.done[idx])


class BatchedRollout:
    """Runs ``policy(obs[B, n_agents, obs_dim] fp32) -> raw actions [B, n_agents]`` on a
    :class:`~mapdn_b200.env.BatchedVoltageControl`, with the reference's action translation and
    episode handling (terminated envs are re-drawn on the device, no host sync). Successive :meth:`run` calls continue
    the same episodes: each starts from the observations the previous one returned."""

    def __init__(self, env, policy: Callable[[torch.Tensor], torch.Tensor], buffer: Optional[DeviceReplayBuffer] = None,
                 keep_returns: int = 1 << 16):
        self.env, self.policy, self.buffer = env, policy, buffer
        self.scale, self.bias = env.args["action_scale"], env.args["action_bias"]
        self.episode_return = torch.zeros(env.batch, dtype=torch.float64, device=env.device)
        # returns of finished episodes: a bounded ring on the device (the last `keep_returns`) + running sum / count
        self.keep_returns = max(int(keep_returns), env.batch)
        self._ret_ring = torch.zeros(self.keep_returns, dtype=torch.float64, device=env.device)
        self._ret_n = torch.zeros((), dtype=torch.int64, device=env.device)          # episodes finished so far
        self._ret_sum = torch.zeros((), dtype=torch.float64, device=env.device)
        self.info_sum = torch.zeros(env.batch, len(env.info[0]), dtype=torch.float64, device=env.device)
        self._started = False
        # the observation every env's next step acts on. With auto-reset the env's own `obs` holds the terminal observation
        # of an env that just ended (its new episode's first one is in `reset_obs`), so the rollout keeps its own.
        self._obs = None

    @torch.no_grad()
    def run(self, n_steps: int, add_noise: bool = True):
        env = self.env
        if not self._started:
            env.reset()
            self._started = True
            self._obs = env.obs.clone()
        obs = self._obs
        # an env whose class has auto-reset re-draws the envs that terminate inside the step launch; the others (and
        # wrappers that forward attributes, which may hook step / reset) get a masked reset
        autoreset = callable(getattr(type(env), "step_autoreset", None))
        step = env.step_autoreset if autoreset else env.step
        for _ in range(n_steps):
            raw = self.policy(obs.to(torch.float32))
            act = translate_action(raw.reshape(env.batch, env.n_agents), self.scale, self.bias).contiguous()
            reward, done, info = step(act, add_noise=add_noise)
            next_obs = env.obs.clone()
            if self.buffer is not None:
                self.buffer.add_batch(obs, raw.reshape(env.batch, env.n_agents), reward, next_obs, done)
            self.episode_return += reward
            self.info_sum += info
            d = done.to(torch.int64)                    # finished episodes -> ring slots, no host sync
            slot = (self._ret_n + torch.cumsum(d, 0) - 1) % self.keep_returns
            slot = torch.where(d.bool(), slot, torch.full_like(slot, self.keep_returns))      # dropped by the scatter
            pad = torch.cat([self._ret_ring, self._ret_ring.new_zeros(1)])
            pad[slot] = self.episode_return
            self._ret_ring = pad[:-1]
            self._ret_sum += (self.episode_return * d).sum()
            self._ret_n += d.sum()
            self.episode_return = torch.where(done.bool(), torch.zeros_like(self.episode_return), self.episode_return)
            if not autoreset:
                env.reset(mask=done, want_state=False)                  # masked, stream-ordered: only terminated envs are re-drawn
            obs = torch.where(done.bool()[:, None, None], env.reset_obs if autoreset else env.obs, next_obs)
        self._obs = obs
        return obs.clone()

    def state_dict(self) -> dict:
        """What a later :meth:`run` continues from: the env's state (:meth:`env.snapshot`, all envs), the running
        episode returns, the finished-episode statistics and the replay buffer. Tensors and plain values only
        (``torch.save`` / ``torch.load(weights_only=True)``); the policy is the caller's."""
        d = dict(env=self.env.snapshot().state_dict(), episode_return=self.episode_return, ret_ring=self._ret_ring,
                 ret_n=self._ret_n, ret_sum=self._ret_sum, info_sum=self.info_sum, started=self._started)
        if self.buffer is not None:
            d["buffer"] = self.buffer.state_dict()
        return d

    def load_state_dict(self, d: dict):
        """Restores a :meth:`state_dict` into this rollout and its env (one with the same fingerprint; any
        ``env_id_offset`` that covers the envs). The observation the next step acts on is gathered again from the restored
        env state (``env.get_obs()``), not stored."""
        from .env import EnvSnapshot
        self.env.restore(EnvSnapshot.from_state_dict(d["env"]))
        dev = self.episode_return.device
        for name, key in (("episode_return", "episode_return"), ("_ret_n", "ret_n"), ("_ret_sum", "ret_sum"),
                          ("info_sum", "info_sum")):
            setattr(self, name, d[key].to(dev).clone())
        self._ret_ring = d["ret_ring"].to(dev).clone()
        self.keep_returns = int(self._ret_ring.numel())
        self._started = bool(d["started"])
        self._obs = self.env.get_obs().clone() if self._started else None
        if self.buffer is not None and "buffer" in d:
            self.buffer.load_state_dict(d["buffer"])

    def completed_episode_returns(self) -> torch.Tensor:
        """Returns of the episodes that ended so far - the last ``keep_returns`` of them (one host sync)."""
        n = int(self._ret_n)
        if n <= self.keep_returns:
            return self._ret_ring[:n].clone()
        h = n % self.keep_returns
        return torch.cat([self._ret_ring[h:], self._ret_ring[:h]])

    def mean_episode_return(self) -> float:
        """Mean return over ALL finished episodes (one host sync)."""
        n = int(self._ret_n)
        return float(self._ret_sum) / n if n else float("nan")
