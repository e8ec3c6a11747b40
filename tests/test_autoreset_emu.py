"""CPU tier for the auto-reset step (mapdn_step_autoreset), on the kernel source compiled for the CPU SIMT emulation
(tests/emu).

Two handles with the same seed take the same actions: A calls mapdn_step_autoreset, B calls the step, then
mapdn_reset(mask = terminated, add_noise = 1) and, with history, mapdn_get_obs_stacked. Every output of the step, the
reset outputs of the terminated envs and all env state must be equal after every call: bit for bit up to 32 lanes per env,
within 1e-10 at 64 / 128 lanes with identical iteration counts, terminated flags and reset outcomes. Episodes run out of
phase (half the batch is reset early), so terminated and running envs share a warp, and an env diverges mid-episode."""
import os
import sys

import numpy as np
import pytest

from conftest import ROOT
from mapdn_b200 import cases
from mapdn_b200.network import ProfileDesc
from test_geometry_emu import _net
from test_history_emu import FIELDS, _mesh, _overload, _set_geometry, get_stacked, set_history

sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
import emu_env                                                       # noqa: E402
from emu_env import EmuEnv, _ptr                                     # noqa: E402

NOT_WRITTEN = 7                                                      # prefill of the reset_ok rows


def step_autoreset(env, a, obs, stacked, reset_obs, reset_stacked, reset_ok, add_noise=True):
    a = np.ascontiguousarray(a, np.float64)
    return emu_env.lib().mapdn_step_autoreset(env._h, _ptr(a), int(add_noise), _ptr(env.reward), _ptr(env.term),
                                              _ptr(env.info), _ptr(obs), _ptr(stacked), _ptr(reset_obs),
                                              _ptr(reset_stacked), _ptr(reset_ok), None)


def _same(a, b, exact, what):
    if exact:
        assert np.array_equal(a, b, equal_nan=True), what
    else:
        assert a.shape == b.shape and np.array_equal(np.isnan(a), np.isnan(b)), what
        d = np.abs(np.nan_to_num(a) - np.nan_to_num(b))
        assert d.size == 0 or d.max() <= 1e-10, (what, float(d.max()))


def run_pair(monkeypatch, net, prof, args, batch, lanes, H, geom, n_steps, diverge_env=None, min_rounds=1):
    """A: mapdn_step_autoreset; B: step + masked reset (+ gather). Returns counters of what the run went through."""
    _set_geometry(monkeypatch, geom)
    L = emu_env.lib()
    A = EmuEnv(net, prof, args, batch=batch, lanes_per_env=lanes)
    Bh = EmuEnv(net, prof, args, batch=batch, lanes_per_env=lanes)
    if H > 1:
        assert set_history(A, H) == 0 and set_history(Bh, H) == 0
    d = A.dims
    G, epb, B = d["lanes_per_env"], d["envs_per_block"], batch
    exact = G <= 32
    ng, od = d["n_agents"], d["obs_dim"]
    seen = dict(terminated=0, mixed_warp=0, diverged=0, reset_failed=0, rounds=[])
    A.reset(); Bh.reset()
    rng = np.random.default_rng(G + 7 * H)
    scale = float(args.get("action_scale", 0.8))
    for t in range(n_steps):
        if t == 1:                              # half the batch starts over: episodes out of phase from here on
            mask = (np.arange(B) % 2).astype(np.uint8)
            start = None
            if diverge_env is not None:         # row 58: the reset solves row 59, the next steps run into the overload
                assert mask[diverge_env]
                start = np.tile(np.array([[1, 5, 3]], np.int32), (B, 1))
                start[diverge_env] = (0, 2, 18)
            A.reset(start, mask=mask); Bh.reset(start, mask=mask)
            _same(A.obs[mask == 1], Bh.obs[mask == 1], exact, "early reset")
        a = rng.uniform(-scale, scale, (B, ng))
        obs_a = np.full((B, ng, od), np.nan)
        stk_a = np.full((B, ng, H * od), np.nan) if H > 1 else None
        robs_a = np.full((B, ng, od), np.nan)
        rstk_a = np.full((B, ng, H * od), np.nan) if H > 1 else None
        rok_a = np.full(B, NOT_WRITTEN, np.uint8)
        n0 = L.mapdn_launch_count(A._h)
        assert step_autoreset(A, a, obs_a, stk_a, robs_a, rstk_a, rok_a) == 0, L.mapdn_last_error()
        assert L.mapdn_launch_count(A._h) == n0 + 1
        seen["rounds"].append(-(-(-(-B // epb)) // A.last_grid()))

        stk_b = None
        if H > 1:
            stk_b = np.full((B, ng, H * od), np.nan)
            assert L.mapdn_step_stacked(Bh._h, _ptr(a), 1, _ptr(Bh.reward), _ptr(Bh.term), _ptr(Bh.info), _ptr(Bh.obs),
                                        _ptr(stk_b), None, 0, None) == 0
        else:
            Bh.step(a)
        term = Bh.term.copy()
        robs_b = np.full((B, ng, od), np.nan)
        rok_b = np.full(B, NOT_WRITTEN, np.uint8)
        assert L.mapdn_reset(Bh._h, None, _ptr(term), 1, _ptr(robs_b), None, _ptr(rok_b), None) == 0

        assert np.array_equal(A.term, term), t
        _same(A.reward, Bh.reward, exact, (t, "reward"))
        _same(A.info, Bh.info, exact, (t, "info"))
        _same(obs_a, Bh.obs, exact, (t, "obs"))
        tm = term == 1
        _same(robs_a[tm], robs_b[tm], exact, (t, "reset_obs"))
        assert np.all(np.isnan(robs_a[~tm])), t
        assert np.array_equal(rok_a, rok_b), t                        # terminated: the outcome; the others: not written
        if H > 1:
            _same(stk_a, stk_b, exact, (t, "obs_stacked"))
            rstk_b = get_stacked(Bh, H)
            _same(rstk_a[tm], rstk_b[tm], exact, (t, "reset_obs_stacked"))
            assert np.all(np.isnan(rstk_a[~tm])), t
            _same(get_stacked(A, H), rstk_b, exact, (t, "get_obs_stacked"))
        for k in FIELDS:
            fa, fb = A.get_field(k), Bh.get_field(k)
            if k in ("steps", "nr_iters", "start_row"):
                assert np.array_equal(fa, fb), (t, k)
            else:
                _same(fa, fb, exact, (t, k))
        _same(A.get_state(), Bh.get_state(), exact, (t, "state"))

        seen["terminated"] += int(tm.sum())
        seen["diverged"] += int((Bh.info[:, 10] == 1.0).sum())
        seen["reset_failed"] += int((rok_b[tm] == 0).sum())
        if G < 32:                              # a warp holds 32 / G consecutive groups of one CTA
            per = 32 // G
            for b0 in range(0, B, epb):
                blk = term[b0:b0 + epb]
                for w0 in range(0, len(blk), per):
                    w = blk[w0:w0 + per]
                    seen["mixed_warp"] += int(w.any() and not w.all())
    assert min(seen["rounds"]) >= min_rounds, seen["rounds"]
    A.close(); Bh.close()
    seen["G"], seen["epb"] = G, epb
    return seen


def _case(name):
    return _overload(cases.make_case(name), cases.make_profiles(name, n_days=4), 3000.0 if name == "case322" else 60.0)


def _args(name, **kw):
    return dict(voltage_barrier_type="bowl", seed=5, action_scale=cases.SCENARIOS[name]["action_scale"], episode_limit=4, **kw)


@pytest.mark.parametrize("H", [1, 3])
@pytest.mark.parametrize("lanes,batch,geom,min_rounds", [
    (4, 37, dict(MAPDN_EMU_SMS=1, MAPDN_EPB=32), 2),               # one CTA per SM: 2 rounds, the last CTA ragged
    (8, 23, dict(MAPDN_EMU_SMS=1, MAPDN_EPB=20), 2),
    (16, 35, dict(MAPDN_EMU_SMS=1, MAPDN_EPB=16), 2),              # two CTAs per SM, three CTAs of work
    (8, 13, dict(), 1),                                            # one round
])
def test_case33_autoreset_equals_step_then_reset(monkeypatch, H, lanes, batch, geom, min_rounds):
    net, prof = _case("case33")
    seen = run_pair(monkeypatch, net, prof, _args("case33"), batch, lanes, H, geom, n_steps=11, diverge_env=5,
                    min_rounds=min_rounds)
    assert seen["G"] == lanes
    if geom:
        assert batch % seen["epb"] != 0
    assert seen["terminated"] >= batch and seen["mixed_warp"] > 0 and seen["diverged"] > 0, seen


@pytest.mark.parametrize("H", [1, 3])
@pytest.mark.parametrize("name,lanes,batch,epb", [("case141", 32, 7, 3), ("case322", 64, 5, 2), ("case322", 128, 3, 1)])
def test_large_feeders_autoreset(monkeypatch, H, name, lanes, batch, epb):
    net, prof = _case(name)
    seen = run_pair(monkeypatch, net, prof, _args(name), batch, lanes, H, dict(MAPDN_EMU_SMS=1, MAPDN_EPB=epb), n_steps=9,
                    diverge_env=1, min_rounds=2)           # case141: two CTAs per SM, three CTAs of work
    assert seen["G"] == lanes and seen["terminated"] >= batch and seen["diverged"] > 0, seen


@pytest.mark.parametrize("H", [1, 3])
def test_dense_meshed_and_hub_autoreset(monkeypatch, H):
    net, prof = _overload(*_mesh())
    seen = run_pair(monkeypatch, net, prof, dict(voltage_barrier_type="l2", seed=2, episode_limit=4), 5, 0, H,
                    dict(MAPDN_EMU_SMS=1, MAPDN_EPB=2), n_steps=9, diverge_env=1, min_rounds=2)
    assert seen["terminated"] >= 5 and seen["diverged"] > 0, seen
    net, prof, scale = _net("hub")
    seen = run_pair(monkeypatch, net, prof, dict(voltage_barrier_type="l1", seed=4, action_scale=scale, episode_limit=3),
                    12, 0, H, dict(MAPDN_EMU_SMS=1, MAPDN_EPB=4), n_steps=8)
    assert seen["G"] == 8 and seen["mixed_warp"] > 0, seen


@pytest.mark.parametrize("H", [1, 3])
def test_reset_that_never_converges_keeps_the_state(monkeypatch, H):
    """Every row overloaded: every step diverges and every draw of every reset does too (reset_ok = 0)."""
    net, prof = cases.make_case("case33"), cases.make_profiles("case33", n_days=4)
    prof = ProfileDesc(pv=prof.pv, load_p=prof.load_p * 60.0, load_q=prof.load_q, steps_per_hour=prof.steps_per_hour,
                       n_days=prof.n_days)
    seen = run_pair(monkeypatch, net, prof, _args("case33"), 6, 8, H, dict(MAPDN_EMU_SMS=1, MAPDN_EPB=4), n_steps=3)
    assert seen["reset_failed"] == seen["terminated"] > 0, seen


def test_autoreset_refusals():
    """Null handle / actions / reward / terminated, a handle without a profile store, stacked pointers without history:
    refused with MAPDN_ERR_INVALID and no launch."""
    L = emu_env.lib()
    net, prof = cases.make_case("case33"), cases.make_profiles("case33", n_days=4)
    env = EmuEnv(net, prof, dict(seed=1), batch=3)
    ng, od = net.n_sgen, env.dims["obs_dim"]
    a, buf = np.zeros((3, ng)), np.zeros((3, ng, 3 * od))
    P = (_ptr(env.reward), _ptr(env.term))

    def refused(h, st, text):
        n = L.mapdn_launch_count(h)
        assert st == 1 and text in L.mapdn_last_error().decode(), L.mapdn_last_error()
        assert L.mapdn_launch_count(h) == n

    refused(env._h, L.mapdn_step_autoreset(None, _ptr(a), 1, *P, None, None, None, None, None, None, None), "null argument")
    refused(env._h, L.mapdn_step_autoreset(env._h, None, 1, *P, None, None, None, None, None, None, None), "null argument")
    refused(env._h, L.mapdn_step_autoreset(env._h, _ptr(a), 1, None, P[1], None, None, None, None, None, None, None),
            "null argument")
    refused(env._h, L.mapdn_step_autoreset(env._h, _ptr(a), 1, P[0], None, None, None, None, None, None, None, None),
            "null argument")
    refused(env._h, L.mapdn_step_autoreset(env._h, _ptr(a), 1, *P, None, None, _ptr(buf), None, None, None, None),
            "no observation history")
    refused(env._h, L.mapdn_step_autoreset(env._h, _ptr(a), 1, *P, None, None, None, None, _ptr(buf), None, None),
            "no observation history")
    n = L.mapdn_launch_count(env._h)
    assert L.mapdn_step_autoreset(env._h, _ptr(a), 1, *P, None, None, None, None, None, None, None) == 0
    assert L.mapdn_launch_count(env._h) == n + 1
    env.close()
    bare = EmuEnv(net, None, dict(seed=1), batch=3)
    refused(bare._h, L.mapdn_step_autoreset(bare._h, _ptr(a), 1, *P, None, None, None, None, None, None, None),
            "without a profile store")
    bare.close()
