"""CPU tier for env state snapshots (mapdn_snapshot_layout / mapdn_snapshot / mapdn_restore), on the kernel source
compiled for the CPU SIMT emulation (tests/emu).

A snapshot row holds all the state an env's future depends on besides the seed and its global id, so restoring it puts
the env back bit for bit: every getter, and the outputs of every later step under the same actions (noise included, the
episode end, the auto-reset, a diverged power flow and the wrap of the frame ring). Index lists select rows, entries
outside the batch are skipped, and the C-level refusals hold."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from conftest import ROOT
from mapdn_b200 import _capi, cases
from test_autoreset_emu import step_autoreset
from test_history_emu import FIELDS, _mesh, _overload, _set_geometry, get_stacked, set_history

sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
import emu_env                                                       # noqa: E402
from emu_env import EmuEnv, _ptr                                     # noqa: E402

N_SEG = len(_capi.SNAPSHOT_SEGMENTS)
FILL = 0xAB


def _L():
    return emu_env.lib()


def layout(env):
    off = (C.c_int64 * (N_SEG + 1))()
    assert _L().mapdn_snapshot_layout(env._h, off) == 0
    return [int(x) for x in off]


def aligned(n, bpe, fill=FILL):
    """A [n, bpe] uint8 array whose data starts 16-byte aligned."""
    raw = np.full(n * bpe + 16, fill, np.uint8)
    s = (-raw.ctypes.data) % 16
    return raw[s:s + n * bpe].reshape(n, bpe)


def snapshot(env, idx=None, n=None):
    bpe = layout(env)[-1]
    ix = None if idx is None else np.ascontiguousarray(idx, np.int32)
    n = env.batch if ix is None else len(ix)
    buf = aligned(n, bpe)
    assert _L().mapdn_snapshot(env._h, _ptr(ix), n, _ptr(buf), None) == 0, _L().mapdn_last_error()
    return buf


def restore(env, buf, idx=None):
    ix = None if idx is None else np.ascontiguousarray(idx, np.int32)
    n = buf.shape[0] if ix is None else len(ix)
    assert _L().mapdn_restore(env._h, _ptr(ix), n, _ptr(buf), None) == 0, _L().mapdn_last_error()


def get_obs(env):
    out = np.full((env.batch, env.dims["n_agents"], env.dims["obs_dim"]), np.nan)
    env._chk(_L().mapdn_get_obs(env._h, _ptr(out), None))
    return out


def record(env):
    _, R = env.record_layout()
    return env.record(np.full((env.batch, R), np.nan))


def everything(env, H):
    """Every getter of the env state, copied."""
    d = {k: env.get_field(k).copy() for k in FIELDS}
    d.update(obs=get_obs(env), state=env.get_state().copy(), record=record(env))
    if H > 1:
        d["obs_stacked"] = get_stacked(env, H)
    return d


def assert_same(a, b, what=""):
    assert a.keys() == b.keys()
    for k in a:
        assert np.array_equal(a[k], b[k], equal_nan=True), (what, k)


def _case(name):
    return _overload(cases.make_case(name), cases.make_profiles(name, n_days=4), 3000.0 if name == "case322" else 60.0)


def _args(name, **kw):
    return dict(dict(voltage_barrier_type="bowl", seed=5, action_scale=cases.SCENARIOS[name]["action_scale"], episode_limit=4),
                **kw)


def _start(env, diverge_env):
    """Sampled reset of all envs, then env `diverge_env` restarted at row 58: its second step runs into the overload."""
    env.reset()
    B = env.batch
    start = np.tile(np.array([[1, 5, 3]], np.int32), (B, 1))
    start[diverge_env] = (0, 2, 18)
    mask = np.zeros(B, np.uint8); mask[diverge_env] = 1
    env.reset(start, mask=mask)


def autoreset_outputs(env, a, H):
    B, ng, od = env.batch, env.dims["n_agents"], env.dims["obs_dim"]
    out = dict(obs=np.full((B, ng, od), np.nan), reset_obs=np.full((B, ng, od), np.nan), reset_ok=np.full(B, 7, np.uint8))
    if H > 1:
        out.update(obs_stacked=np.full((B, ng, H * od), np.nan), reset_obs_stacked=np.full((B, ng, H * od), np.nan))
    st = step_autoreset(env, a, out["obs"], out.get("obs_stacked"), out["reset_obs"], out.get("reset_obs_stacked"),
                        out["reset_ok"])
    assert st == 0, _L().mapdn_last_error()
    out["grid"] = np.array([env.last_grid()])                         # CTAs of the step launch
    out.update(reward=env.reward.copy(), term=env.term.copy(), info=env.info.copy(), record=record(env))
    return out


# ---- round trip ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [1, 3])
def test_round_trip_restores_every_getter(monkeypatch, H):
    _set_geometry(monkeypatch, dict(MAPDN_EMU_SMS=1, MAPDN_EPB=4))
    net, prof = _case("case33")
    env = EmuEnv(net, prof, _args("case33"), batch=9, lanes_per_env=8)
    if H > 1:
        assert set_history(env, H) == 0
    _start(env, 3)
    rng = np.random.default_rng(1)
    for _ in range(2):
        env.step(rng.uniform(-0.8, 0.8, (9, net.n_sgen)))
    before = everything(env, H)
    buf = snapshot(env)
    for _ in range(3):
        autoreset_outputs(env, rng.uniform(-0.8, 0.8, (9, net.n_sgen)), H)
    assert not np.array_equal(everything(env, H)["vm"], before["vm"])
    restore(env, buf)
    assert_same(everything(env, H), before, "after restore")
    assert np.array_equal(snapshot(env), buf)                          # the rows themselves, padding included
    env.close()


# ---- replay ------------------------------------------------------------------------------------------------------------
def run_replay(monkeypatch, net, prof, args, batch, lanes, H, geom, diverge_env, K=1, M=7):
    _set_geometry(monkeypatch, geom)
    env = EmuEnv(net, prof, args, batch=batch, lanes_per_env=lanes)
    if H > 1:
        assert set_history(env, H) == 0
    _start(env, diverge_env)
    rng = np.random.default_rng(lanes + 10 * H)
    scale = float(args.get("action_scale", 0.8))
    for _ in range(K):
        autoreset_outputs(env, rng.uniform(-scale, scale, (batch, env.dims["n_agents"])), H)
    buf = snapshot(env)
    before = everything(env, H)
    acts = [rng.uniform(-scale, scale, (batch, env.dims["n_agents"])) for _ in range(M)]
    first = [autoreset_outputs(env, a, H) for a in acts]
    after = everything(env, H)
    restore(env, buf)
    assert_same(everything(env, H), before, "restored")
    for t, a in enumerate(acts):
        assert_same(autoreset_outputs(env, a, H), first[t], ("replayed step", t))
    assert_same(everything(env, H), after, "end of the replay")
    seen = dict(terminated=int(sum(o["term"].sum() for o in first)),
                diverged=int(sum((o["info"][:, 10] == 1.0).sum() for o in first)),
                G=env.dims["lanes_per_env"],
                rounds=min(-(-(-(-batch // env.dims["envs_per_block"])) // int(o["grid"][0])) for o in first))
    env.close()
    return seen


@pytest.mark.parametrize("H", [1, 3])
@pytest.mark.parametrize("lanes,batch,epb", [(4, 37, 32), (8, 23, 20)])   # one CTA per SM: two rounds
def test_replay_case33(monkeypatch, H, lanes, batch, epb):
    net, prof = _case("case33")
    seen = run_replay(monkeypatch, net, prof, _args("case33"), batch, lanes, H, dict(MAPDN_EMU_SMS=1, MAPDN_EPB=epb), 2)
    assert seen["G"] == lanes and seen["terminated"] >= batch and seen["diverged"] > 0 and seen["rounds"] >= 2, seen


@pytest.mark.parametrize("H", [1, 3])
@pytest.mark.parametrize("name,lanes,batch,epb", [("case141", 32, 7, 3), ("case322", 64, 5, 2), ("case322", 128, 3, 1)])
def test_replay_large_feeders(monkeypatch, H, name, lanes, batch, epb):
    net, prof = _case(name)
    seen = run_replay(monkeypatch, net, prof, _args(name), batch, lanes, H, dict(MAPDN_EMU_SMS=1, MAPDN_EPB=epb), 1, M=6)
    assert seen["G"] == lanes and seen["terminated"] >= batch and seen["diverged"] > 0 and seen["rounds"] >= 2, seen


@pytest.mark.parametrize("H", [1, 3])
def test_replay_dense_fallback(monkeypatch, H):
    net, prof = _overload(*_mesh())
    seen = run_replay(monkeypatch, net, prof, dict(voltage_barrier_type="l2", seed=2, episode_limit=4), 5, 0, H,
                      dict(MAPDN_EMU_SMS=1, MAPDN_EPB=2), 1)
    assert seen["terminated"] >= 5 and seen["diverged"] > 0 and seen["rounds"] >= 2, seen


# ---- index lists -------------------------------------------------------------------------------------------------------
def test_partial_and_out_of_range_indices(monkeypatch):
    _set_geometry(monkeypatch, dict(MAPDN_EMU_SMS=1, MAPDN_EPB=4))
    net, prof = _case("case33")
    B, H = 7, 3
    env = EmuEnv(net, prof, _args("case33"), batch=B, lanes_per_env=8)
    assert set_history(env, H) == 0
    _start(env, 2)
    rng = np.random.default_rng(3)
    env.step(rng.uniform(-0.8, 0.8, (B, net.n_sgen)))
    full = snapshot(env)
    # snapshot: out-of-range entries leave their rows untouched, repeats are allowed
    part = snapshot(env, [5, -1, 2, 99, 5])
    assert np.array_equal(part[[0, 2, 4]], full[[5, 2, 5]])
    assert np.all(part[[1, 3]] == FILL)
    # restore: envs 1 and 4 get other envs' rows, entries outside the batch are skipped, the rest stays as it was
    for _ in range(2):
        env.step(rng.uniform(-0.8, 0.8, (B, net.n_sgen)))
    now = snapshot(env)
    rows = aligned(4, full.shape[1])
    rows[:] = full[[6, 0, 0, 0]]
    restore(env, rows, [1, -3, 4, B])
    got = snapshot(env)
    assert np.array_equal(got[1], full[6]) and np.array_equal(got[4], full[0])
    keep = [b for b in range(B) if b not in (1, 4)]
    assert np.array_equal(got[keep], now[keep])
    env.close()


def test_snapshot_refusals():
    """Null handle or buffer, n <= 0, n > batch, no list with n != batch, a misaligned buffer and a handle without a profile
    store: MAPDN_ERR_INVALID and no launch."""
    L = _L()
    net, prof = cases.make_case("case33"), cases.make_profiles("case33", n_days=4)
    env = EmuEnv(net, prof, dict(seed=1), batch=3)
    bpe = layout(env)[-1]
    buf = aligned(4, bpe)
    ix = np.array([0, 1], np.int32)
    n0 = L.mapdn_launch_count(env._h)

    def refused(st, text, h=env._h):
        n = L.mapdn_launch_count(h)
        assert st == 1 and text in L.mapdn_last_error().decode(), L.mapdn_last_error()
        assert L.mapdn_launch_count(h) == n

    for fn in (L.mapdn_snapshot, L.mapdn_restore):
        refused(fn(None, None, 3, _ptr(buf), None), "null argument")
        refused(fn(env._h, None, 3, None, None), "null argument")
        refused(fn(env._h, _ptr(ix), 0, _ptr(buf), None), "n must be in [1, batch]")
        refused(fn(env._h, _ptr(ix), -2, _ptr(buf), None), "n must be in [1, batch]")
        refused(fn(env._h, _ptr(ix), 4, _ptr(buf), None), "n must be in [1, batch]")
        refused(fn(env._h, None, 2, _ptr(buf), None), "without an index list")
        refused(fn(env._h, None, 3, C.c_void_p(buf.ctypes.data + 8), None), "16-byte aligned")
    refused(L.mapdn_snapshot_layout(None, None), "null argument")
    refused(L.mapdn_snapshot_layout(env._h, None), "null argument")
    assert L.mapdn_launch_count(env._h) == n0
    assert L.mapdn_snapshot(env._h, None, 3, _ptr(buf), None) == 0
    assert L.mapdn_restore(env._h, _ptr(ix), 2, _ptr(buf), None) == 0
    assert L.mapdn_launch_count(env._h) == n0 + 2
    env.close()
    bare = EmuEnv(net, None, dict(seed=1), batch=3)
    for fn in (L.mapdn_snapshot, L.mapdn_restore):
        refused(fn(bare._h, None, 3, _ptr(buf), None), "without a profile store", bare._h)
    bare.close()


# ---- layout ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [1, 3])
def test_layout_segments_are_the_state_arrays(monkeypatch, H):
    _set_geometry(monkeypatch, {})
    net, prof = _case("case141")
    B = 4
    env = EmuEnv(net, prof, _args("case141"), batch=B)
    if H > 1:
        assert set_history(env, H) == 0
    d = env.dims
    env.reset()
    env.reset(mask=np.array([0, 1, 1, 0], np.uint8))
    env.step(np.random.default_rng(0).uniform(-0.6, 0.6, (B, net.n_sgen)))
    off = layout(env)
    counts = dict(cur_pl=d["n_load"], cur_ql=d["n_load"], cur_pv=d["n_sgen"], cur_q=d["n_sgen"], res_vm=d["n_bus"],
                  res_va=d["n_bus"], res_p=d["n_bus"], res_q=d["n_bus"], res_pl=d["n_line"], sum_rewards=1, start_row=1,
                  steps=1, episode=1, nr_iters=1, hist=H * d["n_agents"] * d["obs_dim"] if H > 1 else 0)
    dtypes = {k: np.dtype(_capi.SNAPSHOT_DTYPES.get(k, np.float64)) for k in counts}
    assert off[0] == 0 and off[-1] % 16 == 0
    buf = snapshot(env)
    seg = {}
    for s, k in enumerate(_capi.SNAPSHOT_SEGMENTS):
        nbytes = counts[k] * dtypes[k].itemsize
        assert off[s] % 16 == 0 and off[s + 1] - off[s] == -(-nbytes // 16) * 16, k
        assert np.all(buf[:, off[s] + nbytes:off[s + 1]] == 0), k                     # padding is zero
        seg[k] = np.ascontiguousarray(buf[:, off[s]:off[s] + nbytes]).view(dtypes[k]).reshape(B, counts[k])
    for k, f in (("cur_pl", "p_load"), ("cur_ql", "q_load"), ("cur_pv", "p_sgen"), ("cur_q", "q_sgen"), ("res_vm", "vm"),
                 ("res_p", "p_bus"), ("res_q", "q_bus"), ("res_pl", "line_loss"), ("sum_rewards", "sum_rewards")):
        assert np.array_equal(seg[k], env.get_field(f)), k
    assert np.array_equal(seg["res_va"] * 57.295779513082320876798, env.get_field("va_deg"))
    for k in ("start_row", "steps", "nr_iters"):
        assert np.array_equal(seg[k].astype(np.float64), env.get_field(k)), k
    assert seg["episode"][:, 0].tolist() == [1, 2, 2, 1]                             # resets per env
    if H > 1:                                                                          # the newest frame is get_obs
        ring = seg["hist"].reshape(B, H, -1)
        steps = seg["steps"][:, 0]
        for b in range(B):
            assert np.array_equal(ring[b, (steps[b] - 1) % H], get_obs(env)[b].reshape(-1))
    env.close()


# ---- fork ------------------------------------------------------------------------------------------------------------
def test_fork_one_env_into_every_slot(monkeypatch):
    _set_geometry(monkeypatch, dict(MAPDN_EMU_SMS=1, MAPDN_EPB=4))
    net, prof = _case("case33")
    B, src = 6, 4
    env = EmuEnv(net, prof, _args("case33", episode_limit=48), batch=B, lanes_per_env=8)
    env.reset()
    rng = np.random.default_rng(2)
    env.step(rng.uniform(-0.8, 0.8, (B, net.n_sgen)))
    row = snapshot(env, [src])
    # noise on: the first step after the fork gives the source's reward, info and power flow in every slot
    a = np.tile(rng.uniform(-0.8, 0.8, (1, net.n_sgen)), (B, 1))
    restore(env, snapshot(env, [src] * B))                            # rows through a temporary: every slot <- src
    r, _, info = [x.copy() for x in env.step(a)]
    vm = env.get_field("vm")
    restore(env, row, [src])                                          # the source back as it was
    r_src, _, i_src = [x.copy() for x in env.step(a)]
    assert np.array_equal(r, np.full(B, r_src[src])) and np.array_equal(info, np.tile(i_src[src], (B, 1)))
    assert np.array_equal(vm, np.tile(env.get_field("vm")[src], (B, 1)))
    # noise off: the copies stay identical step after step
    restore(env, snapshot(env, [src] * B))
    for _ in range(3):
        a = np.tile(rng.uniform(-0.8, 0.8, (1, net.n_sgen)), (B, 1))
        r, term, info = env.step(a, add_noise=False)
        obs = env.obs.copy()
        for x in (r, term, info, obs, env.get_field("vm"), env.get_field("p_sgen")):
            assert np.all(x == x[:1]), x
    env.close()


# ---- resharding and lane counts ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [1, 3])
def test_one_handle_restored_as_two_shards(monkeypatch, H):
    _set_geometry(monkeypatch, dict(MAPDN_EMU_SMS=1, MAPDN_EPB=2))
    net, prof = _case("case33")
    args = _args("case33")
    full = EmuEnv(net, prof, args, batch=8, lanes_per_env=8)
    halves = [EmuEnv(net, prof, args, batch=4, lanes_per_env=8, env_id_offset=o) for o in (0, 4)]
    for e in [full] + halves:
        if H > 1:
            assert set_history(e, H) == 0
    _start(full, 5)
    rng = np.random.default_rng(4)
    autoreset_outputs(full, rng.uniform(-0.8, 0.8, (8, net.n_sgen)), H)
    buf = snapshot(full)
    for i, e in enumerate(halves):
        e.reset()                                                      # some other state first
        restore(e, buf[4 * i:4 * i + 4])
    terminated = diverged = 0
    for t in range(7):
        a = rng.uniform(-0.8, 0.8, (8, net.n_sgen))
        want = autoreset_outputs(full, a, H)
        got = [autoreset_outputs(e, a[4 * i:4 * i + 4], H) for i, e in enumerate(halves)]
        for k in set(want) - {"grid"}:                                 # the launch geometry differs, nothing else
            assert np.array_equal(want[k], np.concatenate([g[k] for g in got]), equal_nan=True), (t, k)
        terminated += int(want["term"].sum()); diverged += int((want["info"][:, 10] == 1).sum())
    assert terminated >= 8 and diverged > 0
    for e in [full] + halves:
        e.close()


def test_restore_into_another_lane_count(monkeypatch):
    """A snapshot of an 8-lane handle continues on a 32-lane one within 1e-10, with identical iteration counts and
    terminated flags (the lane count changes the order of the Newton sums, nothing else)."""
    _set_geometry(monkeypatch, dict(MAPDN_EMU_SMS=1, MAPDN_EPB=4))
    net, prof = _case("case33")
    args = _args("case33")
    a8, a32 = EmuEnv(net, prof, args, batch=5, lanes_per_env=8), EmuEnv(net, prof, args, batch=5, lanes_per_env=32)
    assert layout(a8) == layout(a32)
    _start(a8, 1)
    rng = np.random.default_rng(6)
    a8.step(rng.uniform(-0.8, 0.8, (5, net.n_sgen)))
    a32.reset()
    restore(a32, snapshot(a8))
    for t in range(6):
        a = rng.uniform(-0.8, 0.8, (5, net.n_sgen))
        x, y = autoreset_outputs(a8, a, 1), autoreset_outputs(a32, a, 1)
        assert np.array_equal(x["term"], y["term"]) and np.array_equal(x["reset_ok"], y["reset_ok"]), t
        for k in ("reward", "info", "obs", "record"):
            d = np.abs(np.nan_to_num(x[k]) - np.nan_to_num(y[k]))
            assert d.max() <= 1e-10, (t, k, d.max())
        assert np.array_equal(a8.get_field("nr_iters"), a32.get_field("nr_iters")), t
        assert np.array_equal(a8.get_field("steps"), a32.get_field("steps")), t
    a8.close(); a32.close()
