"""CPU tier for env state snapshots (mapdn_snapshot_layout / mapdn_snapshot / mapdn_restore), on the kernel source
compiled for the CPU SIMT emulation (tests/emu).

A snapshot row holds all the state an env's future depends on besides the seed and its global id, so restoring it puts
the env back bit for bit: every getter, and the outputs of every later step under the same actions (noise included, the
episode end, the auto-reset, a diverged power flow and the wrap of the frame ring). Index lists select rows, entries
outside the batch are skipped, and the C-level refusals hold."""
import os
import sys

import numpy as np
import pytest
import torch

import geometry_cases as GC
from conftest import ROOT
from mapdn_b200 import _capi, cases
from test_autoreset_emu import prefill

sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
from emu_env import last_grid, make_env, nan_filled_outputs          # noqa: E402,F401  (autouse fixture)

N_SEG = len(_capi.SNAPSHOT_SEGMENTS)
FILL = 0xAB
NAN = float("nan")


def everything(env, H):
    """Every getter of the env state, copied."""
    d = {k: env.get_field(k).numpy() for k in GC.FIELDS}
    env.obs[:] = NAN
    d.update(obs=env.get_obs().numpy().copy(), state=env.get_state().numpy().copy(),
             record=env.record(torch.full((env.batch, env.record_len), NAN, dtype=torch.float64)).numpy())
    if H > 1:
        d["obs_stacked"] = env.get_obs_stacked().numpy()
    return d


def assert_same(a, b, what=""):
    assert a.keys() == b.keys()
    for k in a:
        assert np.array_equal(a[k], b[k], equal_nan=True), (what, k)


def _args(name, **kw):
    return dict(dict(voltage_barrier_type="bowl", seed=5, action_scale=cases.SCENARIOS[name]["action_scale"], episode_limit=4),
                **kw)


def _start(env, diverge_env):
    """Sampled reset of all envs, then env `diverge_env` restarted at row 58: its second step runs into the overload."""
    env.reset()
    B = env.batch
    start = torch.tensor([[1, 5, 3]] * B, dtype=torch.int32)
    start[diverge_env] = torch.tensor((0, 2, 18))
    mask = torch.zeros(B, dtype=torch.uint8); mask[diverge_env] = 1
    env.reset(start, mask=mask)


def _actions(rng, env, scale=0.8):
    return torch.from_numpy(rng.uniform(-scale, scale, (env.batch, env.n_agents)))


def autoreset_outputs(env, a):
    prefill(env)
    env.step_autoreset(a)
    out = {k: getattr(env, k).numpy().copy() for k in ("obs", "obs_stacked", "reset_obs", "reset_obs_stacked", "reset_ok",
                                                       "reward", "terminated", "info")}
    out["grid"] = np.array([last_grid()])                             # CTAs of the step launch
    out["record"] = env.record(torch.full((env.batch, env.record_len), NAN, dtype=torch.float64)).numpy()
    return out


# ---- round trip ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [1, 3])
def test_round_trip_restores_every_getter(monkeypatch, H):
    GC.set_geometry(monkeypatch, dict(MAPDN_EMU_SMS=1, MAPDN_EPB=4))
    net, prof = GC.overloaded_case("case33")
    env = make_env(net, prof, _args("case33", history=H), batch=9, lanes_per_env=8)
    _start(env, 3)
    rng = np.random.default_rng(1)
    for _ in range(2):
        env.step(_actions(rng, env))
    before = everything(env, H)
    snap = env.snapshot()
    for _ in range(3):
        autoreset_outputs(env, _actions(rng, env))
    assert not np.array_equal(everything(env, H)["vm"], before["vm"])
    env.restore(snap)
    assert_same(everything(env, H), before, "after restore")
    assert torch.equal(env.snapshot().data, snap.data)                # the rows themselves, padding included
    env.close()


# ---- replay ------------------------------------------------------------------------------------------------------------
def run_replay(monkeypatch, net, prof, args, batch, lanes, H, geom, diverge_env, K=1, M=7):
    GC.set_geometry(monkeypatch, geom)
    env = make_env(net, prof, dict(args, history=H), batch=batch, lanes_per_env=lanes)
    _start(env, diverge_env)
    rng = np.random.default_rng(lanes + 10 * H)
    scale = float(args.get("action_scale", 0.8))
    for _ in range(K):
        autoreset_outputs(env, _actions(rng, env, scale))
    snap = env.snapshot()
    before = everything(env, H)
    acts = [_actions(rng, env, scale) for _ in range(M)]
    first = [autoreset_outputs(env, a) for a in acts]
    after = everything(env, H)
    env.restore(snap)
    assert_same(everything(env, H), before, "restored")
    for t, a in enumerate(acts):
        assert_same(autoreset_outputs(env, a), first[t], ("replayed step", t))
    assert_same(everything(env, H), after, "end of the replay")
    seen = dict(terminated=int(sum(o["terminated"].sum() for o in first)),
                diverged=int(sum((o["info"][:, 10] == 1.0).sum() for o in first)),
                G=env.dims["lanes_per_env"],
                rounds=min(-(-(-(-batch // env.dims["envs_per_block"])) // int(o["grid"][0])) for o in first))
    env.close()
    return seen


@pytest.mark.parametrize("H", [1, 3])
@pytest.mark.parametrize("lanes,batch,epb", [(4, 37, 32), (8, 23, 20)])   # one CTA per SM: two rounds
def test_replay_case33(monkeypatch, H, lanes, batch, epb):
    net, prof = GC.overloaded_case("case33")
    seen = run_replay(monkeypatch, net, prof, _args("case33"), batch, lanes, H, dict(MAPDN_EMU_SMS=1, MAPDN_EPB=epb), 2)
    assert seen["G"] == lanes and seen["terminated"] >= batch and seen["diverged"] > 0 and seen["rounds"] >= 2, seen


@pytest.mark.parametrize("H", [1, 3])
@pytest.mark.parametrize("name,lanes,batch,epb", [("case141", 32, 7, 3), ("case322", 64, 5, 2), ("case322", 128, 3, 1)])
def test_replay_large_feeders(monkeypatch, H, name, lanes, batch, epb):
    net, prof = GC.overloaded_case(name)
    seen = run_replay(monkeypatch, net, prof, _args(name), batch, lanes, H, dict(MAPDN_EMU_SMS=1, MAPDN_EPB=epb), 1, M=6)
    assert seen["G"] == lanes and seen["terminated"] >= batch and seen["diverged"] > 0 and seen["rounds"] >= 2, seen


@pytest.mark.parametrize("H", [1, 3])
def test_replay_dense_fallback(monkeypatch, H):
    net, prof = GC.overload(*GC.mesh4())
    seen = run_replay(monkeypatch, net, prof, dict(voltage_barrier_type="l2", seed=2, episode_limit=4), 5, 0, H,
                      dict(MAPDN_EMU_SMS=1, MAPDN_EPB=2), 1)
    assert seen["terminated"] >= 5 and seen["diverged"] > 0 and seen["rounds"] >= 2, seen


# ---- index lists ------------------------------------------------------------------------------------------------------
def test_partial_and_out_of_range_indices(monkeypatch):
    """The C-ABI's index lists: entries outside the batch are skipped (the binding refuses them before the call)."""
    GC.set_geometry(monkeypatch, dict(MAPDN_EMU_SMS=1, MAPDN_EPB=4))
    net, prof = GC.overloaded_case("case33")
    B, H = 7, 3
    env = make_env(net, prof, _args("case33", history=H), batch=B, lanes_per_env=8)
    L, bpe = env._L, env.snapshot_layout[-1]

    def rows(n):
        return torch.full((n, bpe), FILL, dtype=torch.uint8)

    def idx(ix):
        return torch.tensor(ix, dtype=torch.int32)

    _start(env, 2)
    rng = np.random.default_rng(3)
    env.step(_actions(rng, env))
    full = env.snapshot().data
    # snapshot: out-of-range entries leave their rows untouched, repeats are allowed
    part, ix = rows(5), idx([5, -1, 2, 99, 5])
    assert L.mapdn_snapshot(env._h, ix.data_ptr(), 5, part.data_ptr(), None) == 0, L.mapdn_last_error()
    assert torch.equal(part[[0, 2, 4]], full[[5, 2, 5]])
    assert torch.all(part[[1, 3]] == FILL)
    # restore: envs 1 and 4 get other envs' rows, entries outside the batch are skipped, the rest stays as it was
    for _ in range(2):
        env.step(_actions(rng, env))
    now = env.snapshot().data
    back, ix = full[[6, 0, 0, 0]].contiguous(), idx([1, -3, 4, B])
    assert L.mapdn_restore(env._h, ix.data_ptr(), 4, back.data_ptr(), None) == 0, L.mapdn_last_error()
    got = env.snapshot().data
    assert torch.equal(got[1], full[6]) and torch.equal(got[4], full[0])
    keep = [b for b in range(B) if b not in (1, 4)]
    assert torch.equal(got[keep], now[keep])
    env.close()


def test_snapshot_refusals():
    """Null handle or buffer, n <= 0, n > batch, no list with n != batch, a misaligned buffer and a handle without a profile
    store: MAPDN_ERR_INVALID and no launch."""
    net, prof = cases.make_case("case33"), cases.make_profiles("case33", n_days=4)
    env = make_env(net, prof, dict(seed=1), batch=3)
    L = env._L
    bpe = env.snapshot_layout[-1]
    buf = torch.full((4, bpe), FILL, dtype=torch.uint8)
    B, ix = buf.data_ptr(), torch.tensor([0, 1], dtype=torch.int32).data_ptr()
    n0 = L.mapdn_launch_count(env._h)

    def refused(st, text, h=env._h):
        n = L.mapdn_launch_count(h)
        assert st == 1 and text in L.mapdn_last_error().decode(), L.mapdn_last_error()
        assert L.mapdn_launch_count(h) == n

    for fn in (L.mapdn_snapshot, L.mapdn_restore):
        refused(fn(None, None, 3, B, None), "null argument")
        refused(fn(env._h, None, 3, None, None), "null argument")
        refused(fn(env._h, ix, 0, B, None), "n must be in [1, batch]")
        refused(fn(env._h, ix, -2, B, None), "n must be in [1, batch]")
        refused(fn(env._h, ix, 4, B, None), "n must be in [1, batch]")
        refused(fn(env._h, None, 2, B, None), "without an index list")
        refused(fn(env._h, None, 3, B + 8, None), "16-byte aligned")
    refused(L.mapdn_snapshot_layout(None, None), "null argument")
    refused(L.mapdn_snapshot_layout(env._h, None), "null argument")
    assert L.mapdn_launch_count(env._h) == n0
    assert L.mapdn_snapshot(env._h, None, 3, B, None) == 0
    assert L.mapdn_restore(env._h, ix, 2, B, None) == 0
    assert L.mapdn_launch_count(env._h) == n0 + 2
    env.close()
    bare = make_env(net, None, dict(seed=1), batch=3)
    for fn in (L.mapdn_snapshot, L.mapdn_restore):
        refused(fn(bare._h, None, 3, B, None), "without a profile store", bare._h)
    bare.close()


# ---- layout ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [1, 3])
def test_layout_segments_are_the_state_arrays(monkeypatch, H):
    GC.set_geometry(monkeypatch, {})
    net, prof = GC.overloaded_case("case141")
    B = 4
    env = make_env(net, prof, _args("case141", history=H), batch=B)
    d = env.dims
    env.reset()
    env.reset(mask=torch.tensor([0, 1, 1, 0], dtype=torch.uint8))
    env.step(torch.from_numpy(np.random.default_rng(0).uniform(-0.6, 0.6, (B, net.n_sgen))))
    off = env.snapshot_layout
    counts = dict(cur_pl=d["n_load"], cur_ql=d["n_load"], cur_pv=d["n_sgen"], cur_q=d["n_sgen"], res_vm=d["n_bus"],
                  res_va=d["n_bus"], res_p=d["n_bus"], res_q=d["n_bus"], res_pl=d["n_line"], sum_rewards=1, start_row=1,
                  steps=1, episode=1, nr_iters=1, hist=H * d["n_agents"] * d["obs_dim"] if H > 1 else 0)
    dtypes = {k: np.dtype(_capi.SNAPSHOT_DTYPES.get(k, np.float64)) for k in counts}
    assert off[0] == 0 and off[-1] % 16 == 0
    buf = env.snapshot().data.numpy()
    seg = {}
    for s, k in enumerate(_capi.SNAPSHOT_SEGMENTS):
        nbytes = counts[k] * dtypes[k].itemsize
        assert off[s] % 16 == 0 and off[s + 1] - off[s] == -(-nbytes // 16) * 16, k
        assert np.all(buf[:, off[s] + nbytes:off[s + 1]] == 0), k                     # padding is zero
        seg[k] = np.ascontiguousarray(buf[:, off[s]:off[s] + nbytes]).view(dtypes[k]).reshape(B, counts[k])
    for k, f in (("cur_pl", "p_load"), ("cur_ql", "q_load"), ("cur_pv", "p_sgen"), ("cur_q", "q_sgen"), ("res_vm", "vm"),
                 ("res_p", "p_bus"), ("res_q", "q_bus"), ("res_pl", "line_loss"), ("sum_rewards", "sum_rewards")):
        assert np.array_equal(seg[k], env.get_field(f).numpy()), k
    assert np.array_equal(seg["res_va"] * 57.295779513082320876798, env.get_field("va_deg").numpy())
    for k in ("start_row", "steps", "nr_iters"):
        assert np.array_equal(seg[k].astype(np.float64), env.get_field(k).numpy()), k
    assert seg["episode"][:, 0].tolist() == [1, 2, 2, 1]                             # resets per env
    if H > 1:                                                                          # the newest frame is get_obs
        ring = seg["hist"].reshape(B, H, -1)
        steps = seg["steps"][:, 0]
        env.obs[:] = NAN
        obs = env.get_obs().numpy()
        for b in range(B):
            assert np.array_equal(ring[b, (steps[b] - 1) % H], obs[b].reshape(-1))
    env.close()


# ---- fork ------------------------------------------------------------------------------------------------------------
def test_fork_one_env_into_every_slot(monkeypatch):
    GC.set_geometry(monkeypatch, dict(MAPDN_EMU_SMS=1, MAPDN_EPB=4))
    net, prof = GC.overloaded_case("case33")
    B, src = 6, 4
    env = make_env(net, prof, _args("case33", episode_limit=48), batch=B, lanes_per_env=8)
    env.reset()
    rng = np.random.default_rng(2)
    env.step(_actions(rng, env))
    row = env.snapshot([src])
    # noise on: the first step after the fork gives the source's reward, info and power flow in every slot
    a = torch.from_numpy(np.tile(rng.uniform(-0.8, 0.8, (1, net.n_sgen)), (B, 1)))
    env.fork([src] * B, range(B))                                     # rows through a temporary: every slot <- src
    r, _, info = [x.numpy().copy() for x in env.step(a)]
    vm = env.get_field("vm").numpy()
    env.restore(row, [src])                                           # the source back as it was
    r_src, _, i_src = [x.numpy().copy() for x in env.step(a)]
    assert np.array_equal(r, np.full(B, r_src[src])) and np.array_equal(info, np.tile(i_src[src], (B, 1)))
    assert np.array_equal(vm, np.tile(env.get_field("vm").numpy()[src], (B, 1)))
    # noise off: the copies stay identical step after step
    env.fork([src] * B, range(B))
    for _ in range(3):
        a = torch.from_numpy(np.tile(rng.uniform(-0.8, 0.8, (1, net.n_sgen)), (B, 1)))
        r, term, info = [x.numpy() for x in env.step(a, add_noise=False)]
        obs = env.obs.numpy().copy()
        for x in (r, term, info, obs, env.get_field("vm").numpy(), env.get_field("p_sgen").numpy()):
            assert np.all(x == x[:1]), x
    env.close()


# ---- resharding and lane counts ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [1, 3])
def test_one_handle_restored_as_two_shards(monkeypatch, H):
    """Rows placed by global id: each shard takes the rows of its own envs from one snapshot of the whole batch."""
    GC.set_geometry(monkeypatch, dict(MAPDN_EMU_SMS=1, MAPDN_EPB=2))
    net, prof = GC.overloaded_case("case33")
    args = _args("case33", history=H)
    full = make_env(net, prof, args, batch=8, lanes_per_env=8)
    halves = [make_env(net, prof, args, batch=4, lanes_per_env=8, env_id_offset=o) for o in (0, 4)]
    _start(full, 5)
    rng = np.random.default_rng(4)
    autoreset_outputs(full, _actions(rng, full))
    snap = full.snapshot()
    for i, e in enumerate(halves):
        e.reset()                                                      # some other state first
        assert e.restore(snap).tolist() == [0, 1, 2, 3]
    terminated = diverged = 0
    for t in range(7):
        a = _actions(rng, full)
        want = autoreset_outputs(full, a)
        got = [autoreset_outputs(e, a[4 * i:4 * i + 4].contiguous()) for i, e in enumerate(halves)]
        for k in set(want) - {"grid"}:                                 # the launch geometry differs, nothing else
            assert np.array_equal(want[k], np.concatenate([g[k] for g in got]), equal_nan=True), (t, k)
        terminated += int(want["terminated"].sum()); diverged += int((want["info"][:, 10] == 1).sum())
    assert terminated >= 8 and diverged > 0
    for e in [full] + halves:
        e.close()


def test_restore_into_another_lane_count(monkeypatch):
    """A snapshot of an 8-lane handle continues on a 32-lane one within 1e-10, with identical iteration counts and
    terminated flags (the lane count changes the order of the Newton sums, nothing else)."""
    GC.set_geometry(monkeypatch, dict(MAPDN_EMU_SMS=1, MAPDN_EPB=4))
    net, prof = GC.overloaded_case("case33")
    args = _args("case33")
    a8, a32 = make_env(net, prof, args, batch=5, lanes_per_env=8), make_env(net, prof, args, batch=5, lanes_per_env=32)
    assert a8.snapshot_layout == a32.snapshot_layout
    _start(a8, 1)
    rng = np.random.default_rng(6)
    a8.step(_actions(rng, a8))
    a32.reset()
    a32.restore(a8.snapshot())
    for t in range(6):
        a = _actions(rng, a8)
        x, y = autoreset_outputs(a8, a), autoreset_outputs(a32, a)
        assert np.array_equal(x["terminated"], y["terminated"]) and np.array_equal(x["reset_ok"], y["reset_ok"]), t
        for k in ("reward", "info", "obs", "record"):
            d = np.abs(np.nan_to_num(x[k]) - np.nan_to_num(y[k]))
            assert d.max() <= 1e-10, (t, k, d.max())
        assert np.array_equal(a8.get_field("nr_iters").numpy(), a32.get_field("nr_iters").numpy()), t
        assert np.array_equal(a8.get_field("steps").numpy(), a32.get_field("steps").numpy()), t
    a8.close(); a32.close()
