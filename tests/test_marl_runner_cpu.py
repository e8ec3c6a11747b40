"""The batched runner feeds the REFERENCE's own learner code (models/maddpg.py, utilities/trainer.py) unchanged.

The learners are not part of this repository: scripts/make_marl_golden.py ran these cases with them and recorded every
call of the runner (tests/golden/marl_replay.npz); :class:`ReplayNet` answers with the recorded outputs after checking the
runner asked the same, and updates check the batches handed to the trainer. The GPU leg with the real env and an in-repo
model of the same interface is tests/test_gpu_round2.py::test_marl_runner_on_device."""
import json
import os
import sys
from collections import namedtuple
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle.ref_scenarios import digest

REF = os.environ.get("MAPDN_REFERENCE_ROOT", "")      # only the recording script runs the reference
GOLDEN = os.path.join(ROOT, "tests", "golden", "marl_replay.npz")
ALGS = ["iddpg", "maddpg", "matd3", "sqddpg", "facmaddpg", "mappo", "ippo", "coma"]
B, N, OD, T = 5, 3, 7, 6                     # stand-in env: batch, agents, obs dim, max_steps


def dig(t):
    return digest(t.detach().cpu().numpy())


class FakeBatchedEnv:
    """CPU stand-in with the surface of BatchedVoltageControl the runner touches."""

    def __init__(self, B, n_agents, obs_dim, episode_limit, seed=0):
        self.batch, self.n_agents, self.n_actions, self.obs_size = B, n_agents, 1, obs_dim
        self.device = torch.device("cpu")
        self.g = torch.Generator().manual_seed(seed)
        self.obs = torch.zeros(B, n_agents, obs_dim, dtype=torch.float64)
        self.t = torch.zeros(B, dtype=torch.int64)
        self.episode_limit = episode_limit
        self.actions_seen = []

    def reset(self, mask=None, want_state=True, **kw):
        m = torch.ones(self.batch, dtype=torch.bool) if mask is None else mask.bool()
        new = torch.rand(self.batch, self.n_agents, self.obs_size, generator=self.g, dtype=torch.float64)
        self.obs = torch.where(m[:, None, None], new, self.obs)
        self.t = torch.where(m, torch.ones_like(self.t), self.t)
        return self.obs, None

    def step(self, a):
        assert a.dtype == torch.float64 and tuple(a.shape) == (self.batch, self.n_agents)
        self.actions_seen.append(a.clone())
        self.obs = torch.rand(self.batch, self.n_agents, self.obs_size, generator=self.g, dtype=torch.float64)
        self.t += 1
        reward = -a.abs().mean(dim=1)
        done = (self.t >= self.episode_limit).to(torch.uint8)
        info = torch.arange(11, dtype=torch.float64)[None, :].repeat(self.batch, 1)
        return reward, done, info


def reference_on_path():
    """The reference imports its agents lazily (models/model.py:150-163) from namespace packages (no __init__.py); an
    unrelated `agents` distribution in site-packages would shadow them, so the reference's directories are registered
    as the packages for the duration of the test."""
    import types
    saved = {k: sys.modules.get(k) for k in ("agents", "critics", "models", "utilities")}
    for k in saved:
        for name in [m for m in sys.modules if m == k or m.startswith(k + ".")]:
            del sys.modules[name]
        pkg = types.ModuleType(k)
        pkg.__path__ = [os.path.join(REF, k)]
        sys.modules[k] = pkg
    sys.path.append(REF)
    yield
    sys.path.remove(REF)
    for k, v in saved.items():
        for name in [m for m in sys.modules if m == k or m.startswith(k + ".")]:
            del sys.modules[name]
        if v is not None:
            sys.modules[k] = v


def _reference_trainer(alg, n_agents, obs_dim, max_steps):
    import yaml
    from models.model_registry import Model as REGISTRY
    from utilities.trainer import PGTrainer
    d = yaml.safe_load(open(os.path.join(REF, "args", "default.yaml")))
    d.update(yaml.safe_load(open(os.path.join(REF, "args", "alg_args", alg + ".yaml")))["alg_args"])
    d.update(agent_num=n_agents, obs_size=obs_dim, action_dim=1, cuda=False, max_steps=max_steps, action_scale=0.8,
             action_bias=0.0, batch_size=8, hid_size=8)
    args = namedtuple("Args", d.keys())(**d)
    return args, PGTrainer(args, REGISTRY[alg], env=None, logger=None)


TRAIN_ENV = dict(voltage_barrier_type="bowl", action_scale=0.8, action_bias=0.0, seed=21)     # the train_process case


def oracle_env():
    from mapdn_b200 import cases
    net, prof = cases.make_case("case33"), cases.make_profiles("case33", n_days=4)
    return OracleBatchedEnv(net, prof, TRAIN_ENV, batch=1)


def batch_digests(batch):
    return [dig(x) for x in batch.unpacked()]


def window_generator(k):                       # seeded windows: the k-th update's batch is reproducible
    return torch.Generator().manual_seed(1000 + k)


ARG_KEYS = ("max_steps", "action_scale", "action_bias", "hid_size", "batch_size", "num_eval_episodes")


class ReplayNet:
    """Answers the runner's calls as the reference learner did when the case was recorded."""

    def __init__(self, g, case):
        self.g, self.case = g, case
        self.meta = json.loads(str(g[f"{case}/meta"]))
        self.args = SimpleNamespace(**self.meta["args"])
        init = torch.tensor(g[f"{case}/init_hidden"])
        self.policy_dicts = [SimpleNamespace(init_hidden=lambda: init.clone())]
        self.outputs = torch.tensor(g[f"{case}/outputs"])
        self.i = self.pos = 0

    def _answer(self, name, inputs, extra):
        c = self.meta["calls"][self.i]
        assert c["name"] == name and c["extra"] == extra, (self.i, name, c["name"])
        assert c["in"] == [dig(x) for x in inputs], f"call {self.i} ({name}): the runner passed other inputs"
        out = []
        for shape in c["out"]:
            n = 0 if shape is None else int(np.prod(shape))
            out.append(None if shape is None else self.outputs[self.pos:self.pos + n].reshape(shape).clone())
            self.pos += n
        self.i += 1
        return out

    def get_actions(self, state, status, exploration, actions_avail, target, last_hid):
        a, a_pol, lp, hid = self._answer("get_actions", [state, last_hid, actions_avail], [status, exploration, target])
        return a, a_pol, lp, None, hid

    def value(self, obs, act):
        return self._answer("value", [obs, act], [])[0]

    def finished(self):
        return self.i == len(self.meta["calls"]) and self.pos == len(self.outputs)


def _golden():
    return np.load(GOLDEN)


def _replay_on_stand_in(case):
    from mapdn_b200.marl_runner import BatchedMarlRunner, DeviceTransitionBuffer
    g = _golden()
    net = ReplayNet(g, case)
    env = FakeBatchedEnv(B, N, OD, episode_limit=4)
    buf = DeviceTransitionBuffer(32, B, N, OD, act_dim=1, hid_dim=net.args.hid_size, device=env.device)
    want = net.meta["update_batches"]
    updates = []

    def update(runner, stat):
        if len(runner.buffer) >= 2 * net.args.batch_size:
            k = len(updates)
            batch = runner.buffer.get_batch(net.args.batch_size, n_windows=2, generator=window_generator(k))
            updates.append(batch_digests(batch) == want[k])
    runner = BatchedMarlRunner(env, net, buf, update_fn=update)
    stat = runner.train_process({})
    assert len(updates) == len(want) and updates and all(updates)
    for k, v in net.meta["train_stat"].items():
        assert abs(stat[k] - v) < 1e-12, k
    ev = runner.evaluation({}, num_eval_episodes=B)
    assert dig(torch.stack(env.actions_seen)) == net.meta["actions_seen"]          # training and evaluation steps
    for k, v in net.meta["eval_stat"].items():
        assert abs(ev[k] - v) < 1e-12, k
    assert net.finished()
    return runner, env, buf, stat, ev


def test_reference_maddpg_learns_from_device_batches():
    runner, env, buf, stat, ev = _replay_on_stand_in("maddpg_learns")
    args, n, od = runner.args, N, OD
    assert runner.steps == T * B and buf.count == T
    # translate_action (utilities/util.py:123-132): every action the env saw lies inside [bias - scale, bias + scale]
    a = torch.stack(env.actions_seen)
    assert float(a.abs().max()) <= 0.8 + 1e-12
    # transition layout == what Model.unpack_data would have produced
    b = buf.latest(T)
    st, ac, lp, v, nv, rw, ns, dn, ls, av, lh, h = b.unpacked()
    assert st.shape == (T * B, n, od) and ac.shape == (T * B, n, 1) and v.shape == (T * B, n, 1) and rw.shape == (T * B, n)
    assert dn.shape == (T * B, 1) and ls.shape == (T * B, 1) and av.shape == (T * B, n, 1) and lh.shape == (T * B, n, args.hid_size)
    # done at the env's episode_limit (4 -> after 3 steps), last_step additionally at t = max_steps - 1 (model.py:225)
    dn, ls = dn.view(T, B), ls.view(T, B)
    assert bool((dn[2] == 1).all()) and bool((dn[[0, 1, 3, 4]] == 0).all())
    assert bool((ls[T - 1] == 1).all()) and bool((ls[2] == 1).all()) and float(ls.sum()) == float(dn.sum()) + B * (1 - int(dn[T - 1, 0]))
    # hidden state restarts at zero after a terminated episode
    assert float(lh.view(T, B, n, -1)[3].abs().max()) == 0.0 and float(lh.view(T, B, n, -1)[1].abs().max()) > 0.0
    # mean_train_* (model.py:243-261): info k is the constant k in the stand-in env
    assert abs(stat["mean_train_total_line_loss"] - 8.0) < 1e-12 and "mean_train_reward" in stat
    assert abs(ev["mean_test_destroy"] - 10.0) < 1e-12 and np.isfinite(ev["mean_test_reward"])


@pytest.mark.parametrize("alg", ["iddpg", "maddpg", "matd3", "sqddpg", "facmaddpg", "mappo", "ippo", "coma"])
def test_reference_algorithms_run_unchanged_on_device_batches(alg):
    """Eight of the ten algorithms of the reference's registry (models/model_registry.py) collect experience through the
    batched runner and run their own get_loss / optimiser steps on the device batches: deterministic and Gaussian
    policies, twin critics (MATD3: value width 2), coalition sampling (SQDDPG: value width sample_size), a mixer
    (FACMADDPG), PPO / COMA advantage code - replayed: the runner asks each learner what it asked then and hands its
    trainer the same batches. Not covered, for reasons upstream: IAC (`self.cuda_` is never set:
    models/iac.py:90 raises AttributeError with the reference's own env too) and MAAC (its value() returns a
    concatenation that is not [batch, n, k]-shaped, models/maac.py:47-66)."""
    runner, env, buf, stat, ev = _replay_on_stand_in(alg)
    assert runner.steps == T * B
    a = torch.stack(env.actions_seen)
    assert float(a.abs().max()) <= 0.8 + 1e-12                       # translate_action keeps the env's action range
    assert np.isfinite(ev["mean_test_reward"])


class OracleBatchedEnv:
    """CPU stand-in with the surface of BatchedVoltageControl the runner touches, backed by the oracle restatement of the
    env (one VoltageControlOracle per env id) - what the CUDA engine is held to by the parity tests."""

    def __init__(self, net, prof, env_args, batch):
        from oracle.voltage_control_ref import INFO_KEYS, VoltageControlOracle
        self.keys = INFO_KEYS
        self.envs = [VoltageControlOracle(net, prof, env_args, env_id=i) for i in range(batch)]
        self.batch, self.n_agents, self.n_actions = batch, net.n_sgen, 1
        self.device = torch.device("cpu")
        self.obs = None

    def _snap(self):
        self.obs = torch.tensor(np.array([np.array(e.get_obs()) for e in self.envs]))
        self.obs_size = self.obs.shape[-1]

    def reset(self, mask=None, want_state=True, **kw):
        for i, e in enumerate(self.envs):
            if mask is None or bool(mask[i]):
                e.reset()
        self._snap()
        return self.obs, None

    def step(self, a):
        out = [e.step(a[i].numpy()) for i, e in enumerate(self.envs)]
        self._snap()
        return (torch.tensor([o[0] for o in out]), torch.tensor([int(o[1]) for o in out], dtype=torch.uint8),
                torch.tensor([[o[2][k] for k in self.keys] for o in out]))


@pytest.mark.parametrize("alg", ["maddpg", "mappo"])
def test_runner_collects_what_the_reference_train_process_collects(alg):
    """End to end against the reference's OWN loop: `Model.train_process` (models/model.py:197-263) drives the reference's
    own env (oracle/ref_harness.py) with the reference's own learner; the batched runner drives the oracle-backed stand-in
    with a copy of the same learner (replayed). Every field of every transition (state, action, value,
    next_value, reward, next_state, done, last_step, last_hid, hid) and the mean_train_* statistics agree."""
    from mapdn_b200.marl_runner import BatchedMarlRunner, DeviceTransitionBuffer
    g = _golden()
    case = f"train_process_{alg}"
    net = ReplayNet(g, case)
    T = net.args.max_steps
    trans = [SimpleNamespace(**{f: g[f"{case}/ref_{f}"][t] for f in ("state", "next_state", "action", "value", "next_value",
                                                                   "reward", "done", "last_step", "last_hid", "hid")})
             for t in range(T)]                                                # the reference's own transitions
    stat_ref, ev_ref = net.meta["ref_train_stat"], net.meta["ref_eval_stat"]
    env = oracle_env()
    env.reset()                                                                # episode 1, like the reference's constructor
    buf = DeviceTransitionBuffer(T, 1, env.n_agents, env.obs_size, act_dim=1, hid_dim=net.args.hid_size, device=env.device)
    runner = BatchedMarlRunner(env, net, buf)
    stat = runner.train_process({})
    st, ac, lp, v, nv, rw, ns, dn, ls, av, lh, h = buf.latest(T).unpacked()
    tol = 2e-5                                                                 # the learner computes in fp32
    for t, tr in enumerate(trans):
        assert np.abs(np.array(tr.state) - st[t].numpy()).max() < tol and np.abs(np.array(tr.next_state) - ns[t].numpy()).max() < tol
        assert np.abs(tr.action.reshape(-1) - ac[t].numpy().reshape(-1)).max() < tol
        assert np.abs(tr.value.reshape(-1) - v[t].numpy().reshape(-1)).max() < 1e-4
        assert np.abs(tr.next_value.reshape(-1) - nv[t].numpy().reshape(-1)).max() < 1e-4
        assert np.abs(tr.reward - rw[t].numpy()).max() < tol
        assert float(tr.done) == float(dn[t]) and float(tr.last_step) == float(ls[t])
        assert np.abs(tr.last_hid.reshape(-1) - lh[t].numpy().reshape(-1)).max() < tol
        assert np.abs(tr.hid.reshape(-1) - h[t].numpy().reshape(-1)).max() < tol
    for k, v_ref in stat_ref.items():
        if k.startswith("mean_train_"):
            assert abs(stat[k] - v_ref) < 1e-5, k
    # Model.evaluation (models/model.py:265-302): greedy episodes, per-episode means averaged over the episodes
    ev = runner.evaluation({}, num_eval_episodes=2)
    assert len(ev_ref) == 12
    for k, v_ref in ev_ref.items():
        assert abs(ev[k] - v_ref) < 1e-5, k
    assert net.finished()
