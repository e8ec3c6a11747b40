"""Host logic of env state snapshots, without a GPU: the fingerprint, placement of snapshot rows by global env id (on the
CPU emulation of the library, tests/emu), the checkpoint format, and BatchedRollout resuming on a CPU stand-in env that
implements snapshot / restore."""
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

sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
from emu_env import make_env                                        # noqa: E402

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


# ---- placement by global id, on the emulated library ----------------------------------------------------------------------
def _emu(batch, offset=0, history=1):
    """A case33 handle of the CPU emulation of the kernel source (tests/emu), its envs reset and stepped once."""
    env = make_env(cases.make_case("case33"), cases.make_profiles("case33", n_days=3), dict(ARGS, history=history),
                   batch=batch, env_id_offset=offset, lanes_per_env=8)
    env.reset()
    env.step(torch.from_numpy(np.random.default_rng(batch + offset).uniform(-0.8, 0.8, (batch, env.n_agents))))
    return env


def _rows_of(env, gather=True):
    """The snapshot rows, and obs / state / obs_stacked: gathered now, or (gather=False) as the env's buffers hold them
    (restore gathers them again for all envs)."""
    if gather:
        out = dict(obs=env.get_obs().clone(), state=env.get_state().clone(), obs_stacked=env.get_obs_stacked().clone())
    else:
        out = dict(obs=env.obs.clone(), state=env.state.clone(), obs_stacked=env.obs_stacked.clone())
    out["rows"] = env.snapshot().data.clone()
    return out


def test_restore_places_rows_by_global_id():
    for H in (1, 3):
        src = _emu(12, history=H)
        snap, want = src.snapshot(range(8)), _rows_of(src)            # global ids 0..7
        for offset in (0, 4):
            env = _emu(4, offset, history=H)
            assert env.restore(snap).tolist() == [0, 1, 2, 3]
            got = _rows_of(env, gather=False)
            for k in want:
                assert torch.equal(got[k], want[k][offset:offset + 4]), (H, offset, k)
        env = _emu(6, 5, history=H)                                    # ids 5..10: rows 5..7 of the snapshot
        before = _rows_of(env)
        assert env.restore(snap).tolist() == [0, 1, 2]
        got = _rows_of(env, gather=False)
        for k in want:
            assert torch.equal(got[k][:3], want[k][5:8]) and torch.equal(got[k][3:], before[k][3:]), (H, k)
    env = _emu(4, 100)
    rows, n = env.snapshot().data, env.launch_count
    assert env.restore(_emu(4).snapshot()).numel() == 0               # no id of this handle: nothing launched
    assert env.launch_count == n and torch.equal(env.snapshot().data, rows)
    env = _emu(4, 0)
    src = _emu(4, 0)
    before, want = _rows_of(env), _rows_of(src)
    env.restore(src.snapshot([3, 1]), idx=[0, 2])                      # explicit slots
    got = _rows_of(env, gather=False)
    for k in want:
        assert torch.equal(got[k][[0, 2]], want[k][[3, 1]]) and torch.equal(got[k][[1, 3]], before[k][[1, 3]]), k


class _RecordingLib:
    """mapdn_restore / the gathers of a handle, recorded instead of launched (pointers are CPU tensors' addresses)."""

    def __init__(self, bpe):
        self.bpe, self.calls = bpe, []

    def mapdn_restore(self, h, idx, n, buf, stream):
        ids = None if idx is None else list((C.c_int32 * n).from_address(idx.value))
        self.calls.append(("restore", ids))
        return 0

    def mapdn_get_obs(self, *a):
        return 0

    def mapdn_get_state(self, *a):
        return 0


def test_no_index_list_when_all_envs_are_in_order():
    """Every slot in order goes to mapdn_restore without an index list; anything else with one."""
    env = BatchedVoltageControl.__new__(BatchedVoltageControl)
    env.batch, env.env_id_offset, env.history, env._cpu = 4, 4, 1, True
    env.device = torch.device("cpu")
    env._h, env._L = C.c_void_p(1), _RecordingLib(32)
    env._snapshot_layout, env._fingerprint = [0] * 15 + [32], "fp"
    env.obs = env.state = env.obs_stacked = torch.zeros(1)
    env.restore(_snap(range(8)))
    env.restore(_snap([0, 1]), idx=[3, 1])
    assert env._L.calls == [("restore", None), ("restore", [3, 1])]


def test_restore_refusals():
    env = _emu(4, 0)
    one, two = env.snapshot([1]), env.snapshot([1, 2])
    n = env.launch_count
    with pytest.raises(ValueError, match="duplicate"):
        env.restore(two, idx=[3, 3])
    with pytest.raises(ValueError, match="slots must be in"):
        env.restore(two, idx=[0, 4])
    with pytest.raises(ValueError, match="2 slots for 1"):
        env.restore(one, idx=[0, 1])
    with pytest.raises(ValueError, match="duplicate"):
        env.restore(env.snapshot([1, 1]))                              # two rows for one global id
    n = env.launch_count
    wider = EnvSnapshot(torch.zeros(1, one.layout[-1] + 16, dtype=torch.uint8), one.env_ids, one.layout[:-1] + [one.layout[-1] + 16],
                        1, one.fingerprint)
    with pytest.raises(ValueError, match="layout"):
        env.restore(wider)
    with pytest.raises(ValueError, match="layout"):
        env.restore(EnvSnapshot(one.data, one.env_ids, one.layout, 2, one.fingerprint))
    with pytest.raises(ValueError, match="another net"):
        env.restore(EnvSnapshot(one.data, one.env_ids, one.layout, 1, "other"))
    assert env.launch_count == n


def _snap(ids, bpe=32, history=1):
    ids = torch.as_tensor(ids, dtype=torch.int64)
    data = (ids[:, None] * 3 + torch.arange(bpe)[None, :]).to(torch.uint8)
    return EnvSnapshot(data, ids, [0] * 15 + [bpe], history, "fp")


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
