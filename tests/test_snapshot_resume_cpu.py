"""Host logic of env state snapshots, without a GPU: the fingerprint, placement of snapshot rows by global env id, the
checkpoint format, and BatchedRollout resuming on a CPU stand-in env that implements snapshot / restore."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from mapdn_b200 import cases
from mapdn_b200.env import BatchedVoltageControl, EnvSnapshot, snapshot_fingerprint
from mapdn_b200.network import ProfileDesc
from mapdn_b200.rollout import BatchedRollout, DeviceReplayBuffer
from test_autoreset_rollout_cpu import _AutoResetEnv

ARGS = dict(voltage_barrier_type="bowl", voltage_weight=1.0, q_weight=0.1, line_weight=None, v_upper=1.05, v_lower=0.95,
            episode_limit=240, action_scale=0.8, action_bias=0.0, reset_action=True, seed=3,
            state_space=["pv", "demand", "reactive", "vm_pu", "va_degree"])


def _fp(net=None, prof=None, args=None, history=1, tol=0.0, max_iter=0):
    net = net or cases.make_case("case33")
    prof = prof or cases.make_profiles("case33", n_days=3)
    return snapshot_fingerprint(net, prof, dict(ARGS, **(args or {})), history, tol, max_iter)


def test_fingerprint_is_stable_across_processes():
    code = ("from mapdn_b200 import cases; from mapdn_b200.env import snapshot_fingerprint; import test_snapshot_resume_cpu as t;"
            "print(t._fp())")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=ROOT, check=True)
    assert out.stdout.strip() == _fp() and len(_fp()) == 64


@pytest.mark.parametrize("change", [
    dict(args=dict(voltage_barrier_type="l2")), dict(args=dict(voltage_weight=2.0)), dict(args=dict(q_weight=0.2)),
    dict(args=dict(line_weight=0.5)), dict(args=dict(v_upper=1.06)), dict(args=dict(v_lower=0.94)),
    dict(args=dict(episode_limit=120)), dict(args=dict(action_scale=0.6)), dict(args=dict(action_bias=0.1)),
    dict(args=dict(reset_action=False)), dict(args=dict(state_space=["pv", "demand"])), dict(args=dict(seed=4)),
    dict(tol=1e-9), dict(max_iter=12), dict(history=3), "net", "profiles"])
def test_fingerprint_sees_every_input_of_the_dynamics(change):
    if change == "net":
        net = cases.make_case("case33")
        net.br_r = net.br_r.copy(); net.br_r[3] *= 1.01
        assert _fp(net=net) != _fp()
    elif change == "profiles":
        p = cases.make_profiles("case33", n_days=3)
        lp = p.load_p.copy(); lp[100, 2] += 1e-9
        assert _fp(prof=ProfileDesc(pv=p.pv, load_p=lp, load_q=p.load_q, steps_per_hour=p.steps_per_hour)) != _fp()
    else:
        assert _fp(**change) != _fp()


def test_fingerprint_fills_in_the_solver_defaults():
    assert _fp(tol=1e-8, max_iter=10) == _fp()


# ---- placement by global id, on a handle whose library calls are recorded ------------------------------------------------
class _RecordingLib:
    """mapdn_restore / the gathers of a handle, recorded instead of launched (pointers are CPU tensors' addresses)."""

    def __init__(self, bpe):
        self.bpe, self.calls = bpe, []

    def mapdn_restore(self, h, idx, n, buf, stream):
        ids = None if idx is None else list((C.c_int32 * n).from_address(idx.value))
        rows = np.frombuffer(C.string_at(buf.value, n * self.bpe), np.uint8).reshape(n, self.bpe).copy()
        self.calls.append(("restore", ids, rows))
        return 0

    def mapdn_get_obs(self, *a):
        self.calls.append(("get_obs",)); return 0

    def mapdn_get_state(self, *a):
        self.calls.append(("get_state",)); return 0

    def mapdn_get_obs_stacked(self, *a):
        self.calls.append(("get_obs_stacked",)); return 0


def _handle(batch, offset, history=1, bpe=32):
    env = BatchedVoltageControl.__new__(BatchedVoltageControl)
    env.batch, env.env_id_offset, env.history = batch, offset, history
    env.device = torch.device("cpu")
    env._h, env._L = C.c_void_p(1), _RecordingLib(bpe)
    env._snapshot_layout, env._fingerprint = [0] * 15 + [bpe], "fp"
    env.obs = env.state = env.obs_stacked = torch.zeros(1)
    env._stream = lambda: None
    return env


def _snap(ids, bpe=32, history=1):
    ids = torch.as_tensor(ids, dtype=torch.int64)
    data = (ids[:, None] * 3 + torch.arange(bpe)[None, :]).to(torch.uint8)
    return EnvSnapshot(data, ids, [0] * 15 + [bpe], history, "fp")


def test_restore_places_rows_by_global_id():
    snap = _snap(range(8))
    for offset in (0, 4):
        env = _handle(4, offset)
        slots = env.restore(snap)
        assert slots.tolist() == [0, 1, 2, 3]
        kind, ids, rows = env._L.calls[0]
        assert ids is None                                             # all envs in order: no index list
        assert np.array_equal(rows, snap.data[offset:offset + 4].numpy())
        assert [c[0] for c in env._L.calls[1:]] == ["get_obs", "get_state"]
    env = _handle(6, 5, history=3)                                     # ids 5..10: rows 5..7 of the snapshot
    slots = env.restore(_snap(range(8), history=3))
    kind, ids, rows = env._L.calls[0]
    assert slots.tolist() == [0, 1, 2] and ids == [0, 1, 2] and np.array_equal(rows, _snap(range(5, 8)).data.numpy())
    assert env._L.calls[-1] == ("get_obs_stacked",)
    assert _handle(4, 100).restore(snap).numel() == 0                  # no id of this handle: nothing launched
    env = _handle(4, 0)
    env.restore(_snap([3, 1]), idx=[0, 2])                             # explicit slots
    assert env._L.calls[0][1] == [0, 2]


def test_restore_refusals():
    env = _handle(4, 0)
    with pytest.raises(ValueError, match="duplicate"):
        env.restore(_snap([1, 2]), idx=[3, 3])
    with pytest.raises(ValueError, match="slots must be in"):
        env.restore(_snap([1, 2]), idx=[0, 4])
    with pytest.raises(ValueError, match="2 slots for 1"):
        env.restore(_snap([1]), idx=[0, 1])
    with pytest.raises(ValueError, match="duplicate"):
        env.restore(_snap([1, 1]))                                     # two rows for one global id
    with pytest.raises(ValueError, match="layout"):
        env.restore(_snap([1], bpe=48))
    with pytest.raises(ValueError, match="layout"):
        env.restore(_snap([1], history=2))
    bad = _snap([1]); bad.fingerprint = "other"
    with pytest.raises(ValueError, match="another net"):
        env.restore(bad)
    assert env._L.calls == []


def test_state_dict_loads_with_weights_only(tmp_path):
    snap = _snap([7, 2, 2])
    path = os.path.join(tmp_path, "snap.pt")
    torch.save(dict(env=snap.state_dict(), step=11), path)
    back = EnvSnapshot.from_state_dict(torch.load(path, weights_only=True)["env"])
    assert torch.equal(back.data, snap.data) and torch.equal(back.env_ids, snap.env_ids)
    assert (back.layout, back.history, back.fingerprint) == (snap.layout, snap.history, snap.fingerprint)
    row = np.zeros(32, np.uint8)
    row[0:8] = np.frombuffer(np.float64(1.5).tobytes(), np.uint8)         # cur_pl, one load
    row[16:24] = np.frombuffer(np.int64(2).tobytes(), np.uint8)           # start_row
    seg = EnvSnapshot(torch.from_numpy(row[None]), torch.tensor([0]), [0] + [16] * 10 + [32] * 5, 1, "fp")
    assert seg.segment("cur_pl", 1).tolist() == [[1.5]] and seg.segment("start_row", 1).tolist() == [[2]]


# ---- BatchedRollout resume on a CPU stand-in ----------------------------------------------------------------------------
class _SnapEnv(_AutoResetEnv):
    """The stand-in of test_autoreset_rollout_cpu with snapshot / restore / get_obs: a row holds an env's state x, its step
    counter and info row, and the stand-in's generator state (in every row; restore takes it from the first)."""

    def snapshot(self, idx=None):
        g = self.g.get_state()
        rows = [torch.cat([self.x[b].reshape(-1).view(torch.uint8), self.t[b:b + 1].view(torch.uint8),
                           self.info[b].view(torch.uint8), g]) for b in range(self.batch)]
        return EnvSnapshot(torch.stack(rows), torch.arange(self.batch), [0] * 15 + [rows[0].numel()], 1, "standin")

    def restore(self, snap, idx=None):
        nx = self.n_agents * self.obs_size * 8
        d = snap.data
        self.x = d[:, :nx].contiguous().view(torch.float64).reshape(self.x.shape).clone()
        self.t = d[:, nx:nx + 8].contiguous().view(torch.int64).reshape(-1).clone()
        self.info = d[:, nx + 8:nx + 8 + 88].contiguous().view(torch.float64).clone()
        self.g.set_state(d[0, nx + 96:].clone())
        return torch.arange(self.batch)

    def get_obs(self):
        return self.x.clone()


def _make(seed):
    env = _SnapEnv(seed=seed)
    w = torch.tensor([[0.7], [-0.4], [0.2]], dtype=torch.float32)
    buf = DeviceReplayBuffer(40, env.n_agents, env.obs_size, env.device)
    return env, buf, BatchedRollout(env, lambda o: torch.tanh(o @ w).squeeze(-1), buf, keep_returns=8)


@pytest.mark.parametrize("n1,n2", [(3, 5), (2, 7), (0, 4)])
def test_rollout_resumes_bit_for_bit(tmp_path, n1, n2):
    env, buf, ro = _make(0)
    ref_obs = ro.run(n1 + n2)
    env, buf, ro = _make(0)
    ro.run(n1)
    path = os.path.join(tmp_path, "ro.pt")
    torch.save(ro.state_dict(), path)
    env2, buf2, ro2 = _make(99)                                        # another generator: everything must come from the file
    ro2.load_state_dict(torch.load(path, weights_only=True))
    assert torch.equal(ro2._obs, ro._obs)                          # re-gathered from the restored env
    obs = ro2.run(n2)
    envr, bufr, ror = _make(0)
    assert torch.equal(ror.run(n1 + n2), ref_obs)
    assert torch.equal(obs, ref_obs)
    assert torch.equal(ro2.completed_episode_returns(), ror.completed_episode_returns()) and int(ror._ret_n) >= 6
    assert torch.equal(ro2.episode_return, ror.episode_return) and torch.equal(ro2.info_sum, ror.info_sum)
    assert ro2.mean_episode_return() == ror.mean_episode_return()
    for k in ("obs", "action", "reward", "next_obs", "done"):
        assert torch.equal(getattr(buf2, k), getattr(bufr, k)), k
    assert (buf2.head, buf2.count) == (bufr.head, bufr.count)
