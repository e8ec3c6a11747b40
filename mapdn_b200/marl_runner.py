"""Batched counterpart of the reference's experience collection (SURVEY §8 f2).

The reference learners (``models/*.py`` + ``utilities/trainer.py``) collect experience through
``Model.train_process`` / ``Model.evaluation`` (reference ``models/model.py:197-302``): ONE env, ``view(1, n, obs)``,
``translate_action`` -> NumPy -> ``env.step`` -> per-transition ``Transition`` tuples of NumPy arrays in a Python-list
replay buffer (``utilities/replay_buffer.py:5-58``), unpacked again into tensors by ``Model.unpack_data`` (``:304-321``).

Here B envs step in lock-step on the GPU and nothing leaves the device:

* :class:`DeviceTransitionBuffer` - ring of lock-step transitions in HBM holding exactly the twelve fields of the
  reference's ``Transition`` namedtuple (``model.py:18``) in the shapes ``unpack_data`` produces for a batch;
  ``get_batch`` draws windows of consecutive transitions like ``TransReplayBuffer.get_truncated_episodes_batch``.
* :func:`attach` - points a reference model's ``unpack_data`` at those device batches, so the reference's own
  ``get_loss`` / ``PGTrainer.*_transition_process`` code runs unchanged on them.
* :class:`BatchedMarlRunner` - ``train_process`` / ``evaluation`` with the reference's sequencing: action -> value ->
  ``translate_action`` -> ``step`` -> next obs -> next action / value -> transition with ``last_step = done or
  t == max_steps - 1`` (``:225``) -> ``mean_train_*`` averaged over the collected steps (``:243-261``); envs that
  terminate early are re-drawn on the device (masked reset) and their hidden state is zeroed.

The model object only needs the reference's interface: ``get_actions(state, status, exploration, actions_avail, target,
last_hid)``, ``value(obs, act)``, ``policy_dicts[0].init_hidden()`` and an ``args`` with ``max_steps, action_scale,
action_bias, hid_size``.
"""
from __future__ import annotations

from typing import Callable, Optional

import torch

from ._capi import INFO_KEYS
from .rollout import translate_action

__all__ = ["TRANSITION_FIELDS", "DeviceBatch", "DeviceTransitionBuffer", "attach", "BatchedMarlRunner",
           "BatchedPolicyTester"]

# reference models/model.py:18
TRANSITION_FIELDS = ("state", "action", "log_prob_a", "value", "next_value", "reward", "next_state", "done",
                     "last_step", "action_avail", "last_hid", "hid")


class _Sized:
    """``len(batch.state)`` is how the reference's ``get_loss`` reads the batch size (e.g. maddpg.py:96)."""

    def __init__(self, t):
        self.t = t

    def __len__(self):
        return int(self.t.shape[0])


class DeviceBatch:
    """A batch of T transitions on the device, fields shaped as ``Model.unpack_data`` returns them
    (``state [T,n,obs]``, ``action/log_prob_a [T,n,a]``, ``value/next_value [T,n,1]``, ``reward [T,n]``,
    ``done/last_step [T,1]``, ``action_avail [T,n,a]``, ``last_hid/hid [T,n,h]``)."""

    def __init__(self, fields: dict):
        self._f = fields
        self.state = _Sized(fields["state"])

    def __len__(self):
        return len(self.state)

    def unpacked(self, net=None):
        f = self._f
        reward = f["reward"]
        if net is not None and getattr(net.args, "reward_normalisation", False):
            reward = net.batchnorm(reward)                            # model.py:319-320
        return (f["state"], f["action"], f["log_prob_a"], f["value"], f["next_value"], reward, f["next_state"],
                f["done"], f["last_step"], f["action_avail"], f["last_hid"], f["hid"])


def attach(net):
    """Route ``net.unpack_data`` to device batches (instances of :class:`DeviceBatch`); anything else still goes through
    the reference implementation."""
    ref_unpack = net.unpack_data

    def unpack(batch):
        return batch.unpacked(net) if isinstance(batch, DeviceBatch) else ref_unpack(batch)
    net.unpack_data = unpack
    return net


class DeviceTransitionBuffer:
    """FIFO of lock-step transitions ``[capacity_steps, B, ...]`` (reference ``TransReplayBuffer``, capacity counted in
    transitions = ``capacity_steps * B``)."""

    def __init__(self, capacity_steps: int, batch: int, n_agents: int, obs_dim: int, act_dim: int, hid_dim: int,
                 device, dtype=torch.float32):
        S, B, n = int(capacity_steps), int(batch), int(n_agents)
        z = lambda *shape: torch.zeros(S, B, *shape, dtype=dtype, device=device)
        self.data = dict(state=z(n, obs_dim), action=z(n, act_dim), log_prob_a=z(n, act_dim), value=z(n, 1),
                         next_value=z(n, 1), reward=z(n), next_state=z(n, obs_dim), done=z(1), last_step=z(1),
                         action_avail=z(n, act_dim), last_hid=z(n, hid_dim), hid=z(n, hid_dim))
        self.S, self.B, self.device = S, B, device
        self.head, self.count = 0, 0

    def __len__(self):
        return self.count * self.B

    def clear(self):
        self.head = self.count = 0

    def state_dict(self) -> dict:
        return dict(data=dict(self.data), head=self.head, count=self.count)

    def load_state_dict(self, d: dict):
        """The fields of a :meth:`state_dict` (``value`` / ``next_value`` take the checkpoint's width)."""
        for k in TRANSITION_FIELDS:
            v = d["data"][k]
            if tuple(v.shape[:2]) != (self.S, self.B):
                raise ValueError(f"transition buffer {k}: checkpoint shape {tuple(v.shape)}, buffer [{self.S}, {self.B}, ...]")
            self.data[k] = v.to(self.device, self.data[k].dtype).clone()
        self.head, self.count = int(d["head"]), int(d["count"])

    def add(self, **fields):
        """One lock-step: every field ``[B, ...]``. The width of ``value`` / ``next_value`` is the learner's business (one
        Q per agent for most of the reference's algorithms, two for MATD3's twin critics, ``sample_size`` coalition
        values for SQDDPG): the two arrays are re-shaped to what the first lock-step delivers."""
        for k in ("value", "next_value"):
            v = fields[k].reshape(self.B, self.data[k].shape[2], -1)
            if v.shape[2] != self.data[k].shape[3]:
                if self.count:
                    raise ValueError(f"{k}: width changed from {self.data[k].shape[3]} to {v.shape[2]}")
                self.data[k] = torch.zeros(self.S, self.B, v.shape[1], v.shape[2], dtype=self.data[k].dtype, device=self.device)
        for k in TRANSITION_FIELDS:
            self.data[k][self.head].copy_(fields[k].reshape(self.data[k][self.head].shape))
        self.head = (self.head + 1) % self.S
        self.count = min(self.S, self.count + 1)

    def _time_index(self, start, length):
        # logical step 0 = the oldest stored lock-step
        first = (self.head - self.count) % self.S
        return (first + start + torch.arange(length, device=self.device)) % self.S

    def get_batch(self, batch_size: int, n_windows: int = 1, generator: Optional[torch.Generator] = None) -> DeviceBatch:
        """``n_windows`` windows of ``batch_size`` consecutive transitions of one env each (reference
        ``get_truncated_episodes_batch``: a random contiguous chunk of the FIFO), concatenated."""
        L = min(int(batch_size), self.count)
        if L < 1:
            raise ValueError("empty buffer")
        starts = torch.randint(0, self.count - L + 1, (n_windows,), device=self.device, generator=generator)
        envs = torch.randint(0, self.B, (n_windows,), device=self.device, generator=generator)
        first = (self.head - self.count) % self.S
        t_idx = (first + starts[:, None] + torch.arange(L, device=self.device)[None, :]) % self.S      # [W, L]
        e_idx = envs[:, None].expand(-1, L)
        out = {k: v[t_idx, e_idx].reshape((n_windows * L,) + tuple(v.shape[2:])) for k, v in self.data.items()}
        return DeviceBatch(out)

    def latest(self, n_steps: int = 1) -> DeviceBatch:
        """The last ``n_steps`` lock-steps of every env (on-policy learners use the fresh transitions, model.py:66)."""
        n = min(int(n_steps), self.count)
        t_idx = self._time_index(self.count - n, n)
        out = {k: v[t_idx].reshape((n * self.B,) + tuple(v.shape[2:])) for k, v in self.data.items()}
        return DeviceBatch(out)


def learner_obs(env) -> torch.Tensor:
    """What the learner consumes after a reset or step: the stacked frames ``[B, n_agents, history * obs_dim]`` of an env
    with observation history (``history > 1``, reference :303-315), else the observations ``env.obs``."""
    return env.obs_stacked if getattr(env, "history", 1) > 1 else env.obs


def learner_reset_obs(env) -> torch.Tensor:
    """:func:`learner_obs` of the new episodes that ``env.step_autoreset`` started (rows of the terminated envs)."""
    return env.reset_obs_stacked if getattr(env, "history", 1) > 1 else env.reset_obs


class BatchedMarlRunner:
    """``Model.train_process`` / ``Model.evaluation`` over B lock-step envs (see module docstring).

    ``update_fn(runner, stat)`` (optional) is called after every lock-step - the place of the reference's
    ``transition_update`` (model.py:40-70); ``runner.steps`` counts env transitions like ``trainer.steps``."""

    def __init__(self, env, net, buffer: Optional[DeviceTransitionBuffer] = None,
                 update_fn: Optional[Callable] = None):
        self.env, self.net, self.buffer, self.update_fn = env, net, buffer, update_fn
        self.args = net.args
        self.steps, self.episodes = 0, 0
        self._avail = torch.ones(env.batch, env.n_agents, env.n_actions, device=env.device)

    def _init_hidden(self):
        h = self.net.policy_dicts[0].init_hidden()                   # [1, n, hid]
        return h.expand(self.env.batch, -1, -1).contiguous()

    def _translate(self, action):
        a = action.detach().reshape(self.env.batch, self.env.n_agents)
        return translate_action(a, self.args.action_scale, self.args.action_bias).contiguous()

    def train_process(self, stat: dict) -> dict:
        env, net, args = self.env, self.net, self.args
        B = env.batch
        env.reset()
        state = learner_obs(env).to(torch.float32).clone()
        last_hid = self._init_hidden()
        info_sum = torch.zeros(len(INFO_KEYS), dtype=torch.float64, device=env.device)
        reward_sum = torch.zeros((), dtype=torch.float64, device=env.device)
        n_steps = 0
        # an env whose class has auto-reset re-draws the envs that terminate inside the step launch; the others (and
        # wrappers that forward attributes, which may hook step / reset) get a masked reset
        autoreset = callable(getattr(type(env), "step_autoreset", None))
        step = env.step_autoreset if autoreset else env.step
        for t in range(args.max_steps):
            action, action_pol, log_prob_a, _, hid = net.get_actions(state, status="train", exploration=True,
                                                                     actions_avail=self._avail, target=False,
                                                                     last_hid=last_hid)
            value = net.value(state, action_pol)
            reward, done, info = step(self._translate(action))
            next_state = learner_obs(env).to(torch.float32).clone()
            _, next_action_pol, _, _, _ = net.get_actions(next_state, status="train", exploration=True,
                                                          actions_avail=self._avail, target=False, last_hid=hid)
            next_value = net.value(next_state, next_action_pol)
            done_f = done.to(torch.float32).view(B, 1)
            last = torch.ones_like(done_f) if t == args.max_steps - 1 else done_f       # model.py:225
            if self.buffer is not None:
                lp = log_prob_a if log_prob_a is not None else torch.zeros_like(action_pol)
                self.buffer.add(state=state, action=action_pol.detach(), log_prob_a=lp.detach(), value=value.detach(),
                                next_value=next_value.detach(), reward=reward.to(torch.float32)[:, None].expand(-1, env.n_agents),
                                next_state=next_state, done=done_f, last_step=last, action_avail=self._avail,
                                last_hid=last_hid.detach(), hid=hid.detach())
            info_sum += info.sum(dim=0)
            reward_sum += reward.sum()
            n_steps += 1
            self.steps += B
            if self.update_fn is not None:
                self.update_fn(self, stat)
            # envs that ended early (divergence) start a new episode right away; the others carry on
            if not autoreset:
                env.reset(mask=done, want_state=False)
            first = learner_reset_obs(env) if autoreset else learner_obs(env)
            keep = (1.0 - done_f)[:, :, None]
            state = torch.where(done.bool()[:, None, None], first.to(torch.float32), next_state)
            last_hid = hid.detach() * keep
        self.episodes += B
        denom = float(n_steps * B)
        stat["mean_train_reward"] = float(reward_sum) / denom                        # one host sync per call
        for k, v in zip(INFO_KEYS, (info_sum / denom).tolist()):
            stat["mean_train_" + k] = v
        return stat

    def state_dict(self) -> dict:
        """What the next :meth:`train_process` depends on besides the model: the env's state (its per-env episode counters
        key the sampled starts of the next reset), the counters ``steps`` / ``episodes`` and the transition buffer.
        Tensors and plain values only; learner weights, optimiser state and the torch RNG are the caller's, as in the
        reference's ``train.py``."""
        d = dict(env=self.env.snapshot().state_dict(), steps=self.steps, episodes=self.episodes)
        if self.buffer is not None:
            d["buffer"] = self.buffer.state_dict()
        return d

    def load_state_dict(self, d: dict):
        from .env import EnvSnapshot
        self.env.restore(EnvSnapshot.from_state_dict(d["env"]))
        self.steps, self.episodes = int(d["steps"]), int(d["episodes"])
        if self.buffer is not None and "buffer" in d:
            self.buffer.load_state_dict(d["buffer"])

    @torch.no_grad()
    def evaluation(self, stat: dict, num_eval_episodes: Optional[int] = None) -> dict:
        """``num_eval_episodes`` rounds of one episode per env, greedy actions (model.py:265-302); a terminated env
        stops contributing to its episode's means."""
        env, net, args = self.env, self.net, self.args
        B = env.batch
        rounds = max(1, -(-int(num_eval_episodes or args.num_eval_episodes) // B))
        tot = torch.zeros(len(INFO_KEYS) + 1, dtype=torch.float64, device=env.device)
        for _ in range(rounds):
            env.reset()
            state = learner_obs(env).to(torch.float32).clone()
            last_hid = self._init_hidden()
            alive = torch.ones(B, dtype=torch.float64, device=env.device)
            acc = torch.zeros(B, len(INFO_KEYS) + 1, dtype=torch.float64, device=env.device)
            cnt = torch.zeros(B, dtype=torch.float64, device=env.device)
            for t in range(args.max_steps):
                action, _, _, _, hid = net.get_actions(state, status="test", exploration=False,
                                                       actions_avail=self._avail, target=False, last_hid=last_hid)
                reward, done, info = env.step(self._translate(action))
                acc += alive[:, None] * torch.cat([reward[:, None], info], dim=1)
                cnt += alive
                alive = alive * (1.0 - done.to(torch.float64))
                state, last_hid = learner_obs(env).to(torch.float32).clone(), hid
            tot += (acc / cnt[:, None]).mean(dim=0)
        tot = (tot / rounds).tolist()
        stat["mean_test_reward"] = tot[0]
        for k, v in zip(INFO_KEYS, tot[1:]):
            stat["mean_test_" + k] = v
        return stat


class BatchedPolicyTester:
    """The reference's ``PGTester`` (``utilities/tester.py``) over B lock-step envs: ``run`` becomes :meth:`test_run`
    (one env per test day, the six tester getters written by the step kernel itself) and ``batch_run`` becomes
    :meth:`test_batch_run` (B episodes at a time, statistics pooled on the device). Same model interface as
    :class:`BatchedMarlRunner`, whose hidden-state and ``translate_action`` helpers it uses. Needs an env with the record
    surface of ``BatchedVoltageControl`` (``record_slices``, ``record_len``, ``record(out)``, ``step(..., record=)``)."""

    def __init__(self, env, net):
        self.env, self.net, self.args = env, net, net.args
        self._runner = BatchedMarlRunner(env, net)
        self.records, self.lengths = None, None

    def _act(self, state, last_hid):
        action, _, _, _, hid = self.net.get_actions(state, status="test", exploration=False, actions_avail=self._runner._avail,
                                                    target=False, last_hid=last_hid)
        return self._runner._translate(action), hid

    @torch.no_grad()
    def test_run(self, days, hour: int = 23, interval: int = 2):
        """``PGTester.run(day, hour, interval)`` for every day of ``days`` (tester.py:19-63): ``manual_reset`` (noise-free
        start, reset action drawn as in the reference), then noise-free steps of the policy with its hidden state
        carried, until ``done or t == max_steps - 1``. Returns ``records [n_days, max_steps + 1, record_len]`` (fp64, on
        the env's device; rows past an env's end are NaN) and ``lengths [n_days]`` (rows of each day's record). More days
        than the env's batch run in chunks of B. :meth:`records_for_day` gives one day in the reference's structure."""
        env, T = self.env, int(self.args.max_steps)
        days = [int(d) for d in days]
        B, R, dev = env.batch, env.record_len, env.device
        nan = float("nan")
        records = torch.full((len(days), T + 1, R), nan, dtype=torch.float64, device=dev)
        lengths = torch.zeros(len(days), dtype=torch.int64, device=dev)
        for c0 in range(0, len(days), B):
            chunk = days[c0:c0 + B]
            n = len(chunk)
            # a short last chunk repeats its first day in the spare envs (their rows are dropped)
            start = torch.tensor([[d, hour, interval] for d in chunk + chunk[:1] * (B - n)], dtype=torch.int32, device=dev)
            buf = records[c0:c0 + n] if n == B else torch.full((B, T + 1, R), nan, dtype=torch.float64, device=dev)
            env.reset(start, add_noise=False, check=True)                                     # tester.py:21
            env.record(buf[:, 0])                                                             # :34-39
            state = learner_obs(env).to(torch.float32).clone()
            last_hid = self._runner._init_hidden()
            alive = torch.ones(B, dtype=torch.bool, device=dev)
            length = torch.ones(B, dtype=torch.int64, device=dev)
            for t in range(T):
                actions, hid = self._act(state, last_hid)
                _, done, _ = env.step(actions, add_noise=False, record=buf[:, t + 1])           # :48-55
                length += alive
                alive &= done == 0                                                            # :49, :61
                state, last_hid = learner_obs(env).to(torch.float32).clone(), hid
            rows = torch.arange(T + 1, device=dev)[None, :, None]
            buf.masked_fill_(rows >= length[:, None, None], nan)
            if n < B:
                records[c0:c0 + n] = buf[:n]
            lengths[c0:c0 + n] = length[:n]
        self.records, self.lengths = records, lengths
        return records, lengths

    def records_for_day(self, i: int) -> dict:
        """Day ``i`` of the last :meth:`test_run` as ``PGTester.run`` returns it: a dict of six lists of 1-D arrays (one
        per reset / step), keys in the tester's order - pickling it gives the file ``test.py`` writes."""
        n = int(self.lengths[i])
        rows = self.records[i, :n].cpu().numpy()
        return {k: [rows[t, o:o + w].copy() for t in range(n)] for k, (o, w) in self.env.record_slices.items()}

    @torch.no_grad()
    def test_batch_run(self, num_episodes: int = 100) -> dict:
        """``PGTester.batch_run(num_episodes)`` (tester.py:65-99): sampled resets with noise (as ``reset()``), noise-free
        steps, every info key pooled over every step of every episode up to its ``done_``, reported as
        ``{"mean_test_<key>": (mean, 2 * std)}`` (``np.mean`` / population ``np.std``). Episode ``e`` runs on env
        ``e % B`` in round ``e // B``; the statistics are combined on the device, one host read at the end."""
        env, T = self.env, int(self.args.max_steps)
        B, dev, K = env.batch, env.device, len(INFO_KEYS)
        num_episodes = int(num_episodes)
        n = torch.zeros((), dtype=torch.float64, device=dev)
        mean = torch.zeros(K, dtype=torch.float64, device=dev)
        m2 = torch.zeros(K, dtype=torch.float64, device=dev)
        vals = torch.zeros(T, B, K, dtype=torch.float64, device=dev)
        mask = torch.zeros(T, B, dtype=torch.float64, device=dev)
        for r0 in range(0, num_episodes, B):
            vals.zero_(); mask.zero_()
            env.reset(check=True)                                                             # tester.py:69
            state = learner_obs(env).to(torch.float32).clone()
            last_hid = self._runner._init_hidden()
            alive = torch.arange(B, device=dev) < num_episodes - r0                           # spare envs of the last round
            for t in range(T):
                actions, hid = self._act(state, last_hid)
                _, done, info = env.step(actions, add_noise=False)                            # :81
                vals[t] = info
                mask[t] = alive.to(torch.float64)                                             # :84-88
                alive &= done == 0                                                            # :82, :93
                state, last_hid = learner_obs(env).to(torch.float32).clone(), hid
            # this round's pooled statistics (two-pass), merged into the running ones (Chan et al.)
            nr = mask.sum()
            mr = (vals * mask[..., None]).sum(dim=(0, 1)) / nr
            m2r = (((vals - mr) ** 2) * mask[..., None]).sum(dim=(0, 1))
            tot = n + nr
            delta = mr - mean
            mean = mean + delta * (nr / tot)
            m2 = m2 + m2r + delta ** 2 * (n * nr / tot)
            n = tot
        std = torch.sqrt(m2 / n)
        out = torch.stack([mean, 2.0 * std], dim=1).tolist()                                # the one host read
        return {"mean_test_" + k: (v[0], v[1]) for k, v in zip(INFO_KEYS, out)}
