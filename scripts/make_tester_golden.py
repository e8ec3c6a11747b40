#!/usr/bin/env python
"""Writes tests/golden/ref_tester.npz: the reference's own, unmodified ``PGTester`` (utilities/tester.py) driving the
reference's own env (oracle/ref_harness.py) with a reference MADDPG model of seeded weights.

    MAPDN_REFERENCE_ROOT=<reference checkout> python scripts/make_tester_golden.py

Every ``manual_reset`` / ``reset`` of the tester is given the device RNG's draws of the (env id, episode) that the batched
tester (mapdn_b200.marl_runner.BatchedPolicyTester) uses on a fresh env of batch B: day k of ``test_run`` runs on env
``k % B`` as its episode ``k // B + 1``, and episode e of ``test_batch_run`` on env ``e % B`` as its episode ``e // B + 1``.
Stored per case: the tester's records (rows concatenated, lengths per day), and for every policy call the actions and
hidden state the model returned plus the sum of the observation it was given (tests/test_tester_cpu.py replays them);
for ``batch_run`` also the per-step info values and the pooled statistics.
"""
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import tester_cases as TC            # noqa: E402
from oracle import ref_harness as H  # noqa: E402


def reference_model(case, n_agents, obs_dim):
    import yaml
    from models.model_registry import Model
    ref = H.REFERENCE_ROOT
    d = yaml.safe_load(open(os.path.join(ref, "args", "default.yaml")))
    d.update(yaml.safe_load(open(os.path.join(ref, "args", "alg_args", "maddpg.yaml")))["alg_args"])
    d.update(agent_num=n_agents, obs_size=obs_dim, action_dim=1, cuda=False, max_steps=case["max_steps"],
             action_scale=case["env_args"]["action_scale"], action_bias=case["env_args"]["action_bias"],
             hid_size=TC.HID, agent_type=case["agent_type"])
    from collections import namedtuple
    args = namedtuple("Args", d.keys())(**d)
    torch.manual_seed(case["weight_seed"])
    target = Model["maddpg"](args)
    return args, Model["maddpg"](args, target)


class Recorder:
    """Forwards the tester's policy calls to the reference model and records what they returned."""

    def __init__(self, net):
        self.net, self.args, self.policy_dicts = net, net.args, net.policy_dicts
        self.episode = []

    def get_actions(self, state, status, exploration, actions_avail, target, last_hid):
        r = self.net.get_actions(state, status=status, exploration=exploration, actions_avail=actions_avail, target=target,
                                 last_hid=last_hid)
        n = state.shape[1]
        self.episode.append((float(state.double().sum()), r[0].detach().numpy().reshape(n).astype(np.float32),
                             r[4].detach().numpy().reshape(n, -1).astype(np.float32)))
        return r

    def __getattr__(self, k):
        return getattr(self.net, k)


def record_case(out, name, case):
    from utilities.tester import PGTester
    net, prof = TC.build(case)
    with tempfile.TemporaryDirectory() as d:
        H.write_reference_data(d, net, prof)
        ref = H.ReferenceRun(d, net, case["env_args"], env_id=0)
        args, model = reference_model(case, net.n_sgen, ref.env.get_obs_size())
        rec = Recorder(model)
        model.eval()
        tester = PGTester(args, rec, ref.env)
        tester.behaviour_net = rec
        B = case["batch"]
        env, draws = ref.env, ref.draws
        counter = [0]

        def place():                                    # env id / episode of the next reset in the batched tester
            k = counter[0]
            counter[0] += 1
            draws.env_id, draws.episode = k % B, k // B
            draws.begin_reset()
            rec.episode = []
        orig_reset, orig_manual, orig_step = env.reset, env.manual_reset, env.step
        env.reset = lambda *a, **k: (place(), orig_reset(*a, **k))[1]
        env.manual_reset = lambda *a, **k: (place(), orig_manual(*a, **k))[1]
        env.step = lambda *a, **k: (draws.begin_step(), orig_step(*a, **k))[1]
        episodes, infos = [], []
        if case["kind"] == "run":
            rows = []
            for day in case["days"]:
                with ref._ctx():
                    r = tester.run(day, case["hour"], case["interval"])
                rows.append(np.concatenate([np.stack(r[k]) for k in TC.RECORD_KEYS], axis=1))
                episodes.append(rec.episode)
            out[f"{name}/records"] = np.concatenate(rows)
            out[f"{name}/lengths"] = np.array([len(x) for x in rows])
        else:
            seen = []
            step = env.step

            def step_and_log(*a, **k):
                res = step(*a, **k)
                seen.append([float(res[2][key]) for key in H.INFO_KEYS])
                return res
            env.step = step_and_log
            stat, prev = None, 0
            with ref._ctx():
                orig_reset2 = env.reset

                def reset_and_cut(*a, **k):             # closes the previous episode's records
                    nonlocal prev
                    if counter[0]:
                        episodes.append(rec.episode)
                        infos.append(seen[prev:])
                        prev = len(seen)
                    return orig_reset2(*a, **k)
                env.reset = reset_and_cut
                stat = tester.batch_run(case["episodes"])
            episodes.append(rec.episode)
            infos.append(seen[prev:])
            out[f"{name}/info"] = np.concatenate([np.array(x) for x in infos])
            out[f"{name}/info_lengths"] = np.array([len(x) for x in infos])
            out[f"{name}/stat"] = np.array([[stat["mean_test_" + k][0], stat["mean_test_" + k][1]] for k in H.INFO_KEYS])
    out[f"{name}/calls"] = np.array([len(e) for e in episodes])
    out[f"{name}/obs_sum"] = np.concatenate([np.array([c[0] for c in e]) for e in episodes])
    out[f"{name}/actions"] = np.concatenate([np.stack([c[1] for c in e]) for e in episodes])
    out[f"{name}/hid"] = np.concatenate([np.stack([c[2] for c in e]) for e in episodes])
    out[f"{name}/init_hidden"] = model.policy_dicts[0].init_hidden().detach().numpy().reshape(net.n_sgen, -1).astype(np.float32)


def main():
    if not H.reference_available():
        raise SystemExit("set MAPDN_REFERENCE_ROOT to a checkout of Future-Power-Networks/MAPDN")
    from test_marl_runner_cpu import reference_on_path
    next(reference_on_path())
    out = {}
    for name, case in TC.CASES.items():
        record_case(out, name, case)
    out["cases"] = np.array(json.dumps(TC.CASES))
    np.savez_compressed(TC.GOLDEN, **out)
    print(f"{TC.GOLDEN}: {os.path.getsize(TC.GOLDEN) / 1024:.1f} kB, {len(out)} arrays")


if __name__ == "__main__":
    main()
