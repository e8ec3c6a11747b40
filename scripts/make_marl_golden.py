#!/usr/bin/env python
"""Writes tests/golden/marl_replay.npz: the cases of tests/test_marl_runner_cpu.py run with the reference's own learners
(oracle/ref_harness.py: REFERENCE_ROOT), every call of the runner recorded in the format of its ReplayNet.

    MAPDN_REFERENCE_ROOT=<reference checkout> python scripts/make_marl_golden.py
"""
import copy
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_marl_runner_cpu as M     # noqa: E402
from oracle import ref_harness as H  # noqa: E402


class Recorder:
    """Forwards the runner's calls to a reference model and records them."""

    def __init__(self, net, out, case):
        self.net, self.out, self.case, self.calls, self.outputs = net, out, case, [], []
        self.args = net.args
        self.policy_dicts = net.policy_dicts
        out[f"{case}/init_hidden"] = net.policy_dicts[0].init_hidden().detach().numpy()

    def _log(self, name, inputs, extra, outs):
        self.calls.append({"name": name, "extra": extra, "in": [M.dig(x) for x in inputs],
                           "out": [None if o is None else list(o.shape) for o in outs]})
        self.outputs += [o.detach().numpy().astype(np.float32).reshape(-1) for o in outs if o is not None]

    def get_actions(self, state, status, exploration, actions_avail, target, last_hid):
        r = self.net.get_actions(state, status=status, exploration=exploration, actions_avail=actions_avail,
                                 target=target, last_hid=last_hid)
        self._log("get_actions", [state, last_hid, actions_avail], [status, exploration, target], [r[0], r[1], r[2], r[4]])
        return r

    def value(self, obs, act):
        v = self.net.value(obs, act)
        self._log("value", [obs, act], [], [v])
        return v

    def meta(self, **kw):
        self.out[f"{self.case}/outputs"] = np.concatenate(self.outputs)
        return dict(args={k: getattr(self.args, k) for k in M.ARG_KEYS}, calls=self.calls, **kw)


def record_stand_in(out, case, alg):
    from mapdn_b200._capi import INFO_KEYS
    from mapdn_b200.marl_runner import BatchedMarlRunner, DeviceTransitionBuffer, attach
    args, trainer = M._reference_trainer(alg, M.N, M.OD, max_steps=M.T)
    rec = Recorder(attach(trainer.behaviour_net), out, case)
    env = M.FakeBatchedEnv(M.B, M.N, M.OD, episode_limit=4)
    buf = DeviceTransitionBuffer(32, M.B, M.N, M.OD, act_dim=1, hid_dim=args.hid_size, device=env.device)
    batches, changed = [], []

    def update(runner, stat):
        if len(runner.buffer) >= 2 * args.batch_size:
            batch = runner.buffer.get_batch(args.batch_size, n_windows=2, generator=M.window_generator(len(batches)))
            batches.append(M.batch_digests(batch))
            w0 = [p.detach().clone() for p in trainer.behaviour_net.parameters()]
            trainer.value_transition_process(stat, batch)
            trainer.policy_transition_process(stat, batch)
            if args.mixer:
                trainer.mixer_transition_process(stat, batch)
            changed.append(any(not torch.equal(a, b) for a, b in zip(w0, trainer.behaviour_net.parameters())))
    runner = BatchedMarlRunner(env, rec, buf, update_fn=update)
    stat = runner.train_process({})
    assert batches and all(changed), case
    assert np.isfinite(stat["mean_train_value_loss"]) and np.isfinite(stat["mean_train_policy_loss"])
    ev = runner.evaluation({}, num_eval_episodes=M.B)
    out[f"{case}/meta"] = np.array(json.dumps(rec.meta(
        update_batches=batches, actions_seen=M.dig(torch.stack(env.actions_seen)),
        train_stat={k: stat[k] for k in ["mean_train_reward"] + ["mean_train_" + q for q in INFO_KEYS]},
        eval_stat={k: v for k, v in ev.items() if k.startswith("mean_test_")})))


def record_train_process(out, alg):
    import tempfile
    from mapdn_b200 import cases
    from mapdn_b200.marl_runner import BatchedMarlRunner, DeviceTransitionBuffer, attach
    case = f"train_process_{alg}"
    net, prof = cases.make_case("case33"), cases.make_profiles("case33", n_days=4)
    with tempfile.TemporaryDirectory() as d:
        H.write_reference_data(d, net, prof)
        ref = H.ReferenceRun(d, net, M.TRAIN_ENV, env_id=0)
        T = 5
        args, trainer = M._reference_trainer(alg, net.n_sgen, ref.env.get_obs_size(), max_steps=T)
        args = args._replace(replay_warmup=10 ** 9)            # collection only
        trainer.args = trainer.behaviour_net.args = args
        model_copy = copy.deepcopy(trainer.behaviour_net)

        def hooked(begin, fn):                                 # tells the harness which draws come next
            return lambda *a: (begin(), fn(*a))[1]
        trainer.env = ref.env
        ref.env.reset, ref.env.step = hooked(ref.draws.begin_reset, ref.env.reset), hooked(ref.draws.begin_step, ref.env.step)
        torch.manual_seed(5)
        stat_ref = {}
        with ref._ctx():
            trainer.behaviour_net.train_process(stat_ref, trainer)
        trans = trainer.replay_buffer.buffer
        assert len(trans) == T
        for f in ("state", "next_state", "action", "value", "next_value", "reward", "done", "last_step", "last_hid", "hid"):
            out[f"{case}/ref_{f}"] = np.array([np.asarray(getattr(tr, f), dtype=np.float64) for tr in trans])
        args = args._replace(num_eval_episodes=2)
        trainer.args = trainer.behaviour_net.args = model_copy.args = args
        ev_ref = {}
        with ref._ctx():
            trainer.behaviour_net.evaluation(ev_ref, trainer)
    env = M.oracle_env()
    env.reset()
    rec = Recorder(attach(model_copy), out, case)
    buf = DeviceTransitionBuffer(T, 1, net.n_sgen, env.obs_size, act_dim=1, hid_dim=args.hid_size, device=env.device)
    runner = BatchedMarlRunner(env, rec, buf)
    torch.manual_seed(5)
    runner.train_process({})
    runner.evaluation({}, num_eval_episodes=2)
    out[f"{case}/meta"] = np.array(json.dumps(rec.meta(
        ref_train_stat={k: v for k, v in stat_ref.items() if k.startswith("mean_train_")}, ref_eval_stat=ev_ref)))


def main():
    if not H.reference_available():
        raise SystemExit("set MAPDN_REFERENCE_ROOT to a checkout of Future-Power-Networks/MAPDN")
    next(M.reference_on_path())
    torch.manual_seed(0)
    out = {}
    record_stand_in(out, "maddpg_learns", "maddpg")
    for alg in M.ALGS:
        record_stand_in(out, alg, alg)
    for alg in ("maddpg", "mappo"):
        record_train_process(out, alg)
    np.savez_compressed(M.GOLDEN, **out)
    print(f"{M.GOLDEN}: {os.path.getsize(M.GOLDEN) / 1024:.1f} kB, {len(out)} arrays")


if __name__ == "__main__":
    main()
