"""The cases of tests/golden/ref_tester.npz (scripts/make_tester_golden.py runs them with the reference's PGTester) and the
two stand-ins the tester tests use: :class:`ReplayPolicy` answers the batched tester's policy calls with what the
reference model answered, and :class:`OracleRecordEnv` is the oracle restatement of the env (CPU) with the record
surface of BatchedVoltageControl. Imports neither the reference nor a GPU."""
import os
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_tester.npz")
HID = 8
RECORD_KEYS = ("pv_active", "pv_reactive", "bus_active", "bus_reactive", "bus_voltage", "line_loss")


def _env_args(episode_limit, seed=3):
    return dict(voltage_barrier_type="l1", action_scale=0.8, action_bias=0.0, episode_limit=episode_limit, seed=seed)


CASES = {
    # test.py's single-day test: episode_limit = max_steps = 480, agent_type rnn (args/default.yaml)
    "rnn_day": dict(kind="run", profile="case33", days=[1], hour=23, interval=2, max_steps=480, agent_type="rnn",
                    env_args=_env_args(480), batch=1, weight_seed=1),
    # three days on two envs: two chunks, MLP policy
    "mlp_days": dict(kind="run", profile="case33", days=[2, 0, 1], hour=23, interval=2, max_steps=10, agent_type="mlp",
                     env_args=_env_args(480), batch=2, weight_seed=2),
    # day 0 from 02:45 walks into rows the feeder cannot serve: its record ends early; day 1 runs to max_steps
    "diverge": dict(kind="run", profile="case33_overload", days=[0, 1], hour=2, interval=15, max_steps=20, agent_type="rnn",
                    env_args=_env_args(480), batch=2, weight_seed=3),
    # batch_run: 5 sampled episodes on 3 envs (two rounds), episodes end at episode_limit
    "batch": dict(kind="batch", profile="case33", episodes=5, max_steps=12, agent_type="rnn", env_args=_env_args(10, seed=4),
                  batch=3, weight_seed=4),
}


def build(case):
    from mapdn_b200 import cases
    from mapdn_b200.network import ProfileDesc
    net, prof = cases.make_case("case33"), cases.make_profiles("case33", n_days=4)
    if case["profile"] == "case33_overload":
        lp = prof.load_p.copy(); lp[60:460] *= 60.0
        prof = ProfileDesc(pv=prof.pv, load_p=lp, load_q=prof.load_q, steps_per_hour=20, n_days=prof.n_days)
    return net, prof


class ReplayPolicy:
    """The reference model's answers, per (episode, step), for the envs of the batched tester: env b of round r runs
    episode (or day) r * B + b. Checks that the tester hands over the right observation (its sum) and carries the hidden
    state it was given back (exactly)."""

    def __init__(self, g, name, case, obs_tol=1e-4):
        n_calls = g[f"{name}/calls"]
        cut = np.cumsum(n_calls)[:-1]
        self.acts = np.split(g[f"{name}/actions"], cut)
        self.hids = np.split(g[f"{name}/hid"], cut)
        self.osum = np.split(g[f"{name}/obs_sum"], cut)
        self.init = torch.tensor(g[f"{name}/init_hidden"])
        init = self.init[None]
        self.policy_dicts = [SimpleNamespace(init_hidden=lambda: init.clone())]
        self.args = SimpleNamespace(max_steps=case["max_steps"], action_scale=case["env_args"]["action_scale"],
                                    action_bias=case["env_args"]["action_bias"])
        self.obs_tol, self.k, self.checked = obs_tol, 0, 0

    def get_actions(self, state, status, exploration, actions_avail, target, last_hid):
        assert status == "test" and exploration is False and target is False
        B, n = state.shape[0], state.shape[1]
        r, t = divmod(self.k, self.args.max_steps)
        self.k += 1
        acts = torch.zeros(B, n, 1)
        hid = torch.zeros(B, n, self.init.shape[-1])
        lh = last_hid.detach().cpu().float()
        for b in range(B):
            e = r * B + b
            if e >= len(self.acts) or t >= len(self.acts[e]):
                continue
            assert abs(float(state[b].double().sum()) - self.osum[e][t]) < self.obs_tol * max(1.0, abs(self.osum[e][t])), (e, t)
            want = self.init if t == 0 else torch.tensor(self.hids[e][t - 1])
            assert torch.equal(lh[b], want), (e, t)                     # hidden state carried (tester.py:60)
            acts[b, :, 0] = torch.tensor(self.acts[e][t])
            hid[b] = torch.tensor(self.hids[e][t])
            self.checked += 1
        return acts.to(state.device), None, None, None, hid.to(state.device)


class OracleRecordEnv:
    """B oracle envs (oracle.voltage_control_ref) with the surface of BatchedVoltageControl the tester uses."""

    def __init__(self, net, prof, env_args, batch):
        from oracle.voltage_control_ref import INFO_KEYS, VoltageControlOracle
        self.keys = INFO_KEYS
        self.envs = [VoltageControlOracle(net, prof, env_args, env_id=i) for i in range(batch)]
        self.batch, self.n_agents, self.n_actions = batch, net.n_sgen, 1
        self.device = torch.device("cpu")
        w = [net.n_sgen, net.n_sgen, net.n_bus, net.n_bus, net.n_bus, net.n_line]
        self.record_slices = {k: (int(o), int(n)) for k, o, n in zip(RECORD_KEYS, np.cumsum([0] + w[:-1]), w)}
        self.record_len = int(sum(w))

    def _snap(self):
        self.obs = torch.tensor(np.array([np.array(e.get_obs()) for e in self.envs]))

    def reset(self, start=None, mask=None, add_noise=True, check=False, **kw):
        for i, e in enumerate(self.envs):
            e.reset(None if start is None else tuple(int(x) for x in start[i]), add_noise=add_noise)
        self._snap()
        return self.obs, None

    def record(self, out):
        for i, e in enumerate(self.envs):
            r = e.g.res
            out[i] = torch.tensor(np.concatenate([e.g.sgen_p, e.g.sgen_q, r.p_mw, r.q_mvar, r.vm_pu, r.pl_mw]))
        return out

    def step(self, a, add_noise=True, record=None):
        res = [e.step(a[i].numpy(), add_noise=add_noise) for i, e in enumerate(self.envs)]
        self._snap()
        if record is not None:
            self.record(record)
        return (torch.tensor([o[0] for o in res]), torch.tensor([int(o[1]) for o in res], dtype=torch.uint8),
                torch.tensor([[o[2][k] for k in self.keys] for o in res]))
