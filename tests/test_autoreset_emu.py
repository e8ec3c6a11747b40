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
import torch

import geometry_cases as GC
from conftest import ROOT
from mapdn_b200 import cases
from mapdn_b200.network import ProfileDesc
from test_geometry_emu import _net

sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
from emu_env import last_grid, make_env, nan_filled_outputs          # noqa: E402,F401  (autouse fixture)

NOT_WRITTEN = 7                                                      # prefill of the reset_ok rows
NAN = float("nan")


def prefill(env):
    """Sentinels in the buffers step_autoreset writes, so rows it must not write stay recognisable."""
    if getattr(env, "reset_obs", None) is None:
        env.reset_obs = torch.empty_like(env.obs)
        env.reset_obs_stacked = torch.empty_like(env.obs_stacked) if env.history > 1 else env.reset_obs
    for t in (env.obs, env.obs_stacked, env.reset_obs, env.reset_obs_stacked):
        t[:] = NAN
    env.reset_ok[:] = NOT_WRITTEN


def _same(a, b, exact, what):
    GC.same(a, b, exact, what, equal_nan=True)


def run_pair(monkeypatch, net, prof, args, batch, lanes, H, geom, n_steps, diverge_env=None, min_rounds=1):
    """A: step_autoreset; B: step + masked reset (+ gather). Returns counters of what the run went through."""
    GC.set_geometry(monkeypatch, geom)
    A = make_env(net, prof, dict(args, history=H), batch=batch, lanes_per_env=lanes)
    Bh = make_env(net, prof, dict(args, history=H), batch=batch, lanes_per_env=lanes)
    L = A._L
    d = A.dims
    G, epb, B = d["lanes_per_env"], d["envs_per_block"], batch
    exact = G <= 32
    seen = dict(terminated=0, mixed_warp=0, diverged=0, reset_failed=0, rounds=[])
    A.reset(); Bh.reset()
    rng = np.random.default_rng(G + 7 * H)
    scale = float(args.get("action_scale", 0.8))
    for t in range(n_steps):
        if t == 1:                              # half the batch starts over: episodes out of phase from here on
            mask = torch.from_numpy((np.arange(B) % 2).astype(np.uint8))
            start = None
            if diverge_env is not None:         # row 58: the reset solves row 59, the next steps run into the overload
                assert mask[diverge_env]
                start = torch.tensor([[1, 5, 3]] * B, dtype=torch.int32)
                start[diverge_env] = torch.tensor((0, 2, 18))
            A.reset(start, mask=mask); Bh.reset(start, mask=mask)
            _same(A.obs.numpy()[mask == 1], Bh.obs.numpy()[mask == 1], exact, "early reset")
        a = torch.from_numpy(rng.uniform(-scale, scale, (B, d["n_agents"])))
        prefill(A)
        n0 = L.mapdn_launch_count(A._h)
        A.step_autoreset(a)
        assert L.mapdn_launch_count(A._h) == n0 + 1
        seen["rounds"].append(-(-(-(-B // epb)) // last_grid()))

        Bh.obs_stacked[:] = NAN
        r_b, term, i_b = [x.numpy().copy() for x in Bh.step(a)]
        obs_b, stk_b = Bh.obs.numpy().copy(), Bh.obs_stacked.numpy().copy()
        Bh.obs[:] = NAN; Bh.obs_stacked[:] = NAN; Bh.reset_ok[:] = NOT_WRITTEN
        Bh.reset(mask=torch.from_numpy(term), want_state=False)     # the reset outputs and, with history, the gather
        robs_b, rstk_b, rok_b = Bh.obs.numpy(), Bh.obs_stacked.numpy(), Bh.reset_ok.numpy()

        assert np.array_equal(A.terminated.numpy(), term), t
        _same(A.reward.numpy(), r_b, exact, (t, "reward"))
        _same(A.info.numpy(), i_b, exact, (t, "info"))
        _same(A.obs.numpy(), obs_b, exact, (t, "obs"))
        tm = term == 1
        robs_a = A.reset_obs.numpy()
        _same(robs_a[tm], robs_b[tm], exact, (t, "reset_obs"))
        assert np.all(np.isnan(robs_a[~tm])), t
        assert np.array_equal(A.reset_ok.numpy(), rok_b), t            # terminated: the outcome; the others: not written
        if H > 1:
            _same(A.obs_stacked.numpy(), stk_b, exact, (t, "obs_stacked"))
            rstk_a = A.reset_obs_stacked.numpy()
            _same(rstk_a[tm], rstk_b[tm], exact, (t, "reset_obs_stacked"))
            assert np.all(np.isnan(rstk_a[~tm])), t
            _same(A.get_obs_stacked().numpy(), rstk_b, exact, (t, "get_obs_stacked"))
        for k in GC.FIELDS:
            fa, fb = A.get_field(k).numpy(), Bh.get_field(k).numpy()
            if k in ("steps", "nr_iters", "start_row"):
                assert np.array_equal(fa, fb), (t, k)
            else:
                _same(fa, fb, exact, (t, k))
        _same(A.get_state().numpy().copy(), Bh.get_state().numpy(), exact, (t, "state"))

        seen["terminated"] += int(tm.sum())
        seen["diverged"] += int((i_b[:, 10] == 1.0).sum())
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
    net, prof = GC.overloaded_case("case33")
    seen = run_pair(monkeypatch, net, prof, _args("case33"), batch, lanes, H, geom, n_steps=11, diverge_env=5,
                    min_rounds=min_rounds)
    assert seen["G"] == lanes
    if geom:
        assert batch % seen["epb"] != 0
    assert seen["terminated"] >= batch and seen["mixed_warp"] > 0 and seen["diverged"] > 0, seen


@pytest.mark.parametrize("H", [1, 3])
@pytest.mark.parametrize("name,lanes,batch,epb", [("case141", 32, 7, 3), ("case322", 64, 5, 2), ("case322", 128, 3, 1)])
def test_large_feeders_autoreset(monkeypatch, H, name, lanes, batch, epb):
    net, prof = GC.overloaded_case(name)
    seen = run_pair(monkeypatch, net, prof, _args(name), batch, lanes, H, dict(MAPDN_EMU_SMS=1, MAPDN_EPB=epb), n_steps=9,
                    diverge_env=1, min_rounds=2)           # case141: two CTAs per SM, three CTAs of work
    assert seen["G"] == lanes and seen["terminated"] >= batch and seen["diverged"] > 0, seen


@pytest.mark.parametrize("H", [1, 3])
def test_dense_meshed_and_hub_autoreset(monkeypatch, H):
    net, prof = GC.overload(*GC.mesh4())
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
    net, prof = cases.make_case("case33"), cases.make_profiles("case33", n_days=4)
    env = make_env(net, prof, dict(seed=1), batch=3)
    L = env._L
    ng, od = net.n_sgen, env.dims["obs_dim"]
    a, buf = torch.zeros(3, ng, dtype=torch.float64), torch.zeros(3, ng, 3 * od, dtype=torch.float64)
    A = a.data_ptr()
    P = (env.reward.data_ptr(), env.terminated.data_ptr())

    def refused(h, st, text):
        n = L.mapdn_launch_count(h)
        assert st == 1 and text in L.mapdn_last_error().decode(), L.mapdn_last_error()
        assert L.mapdn_launch_count(h) == n

    refused(env._h, L.mapdn_step_autoreset(None, A, 1, *P, None, None, None, None, None, None, None), "null argument")
    refused(env._h, L.mapdn_step_autoreset(env._h, None, 1, *P, None, None, None, None, None, None, None), "null argument")
    refused(env._h, L.mapdn_step_autoreset(env._h, A, 1, None, P[1], None, None, None, None, None, None, None),
            "null argument")
    refused(env._h, L.mapdn_step_autoreset(env._h, A, 1, P[0], None, None, None, None, None, None, None, None),
            "null argument")
    refused(env._h, L.mapdn_step_autoreset(env._h, A, 1, *P, None, None, buf.data_ptr(), None, None, None, None),
            "no observation history")
    refused(env._h, L.mapdn_step_autoreset(env._h, A, 1, *P, None, None, None, None, buf.data_ptr(), None, None),
            "no observation history")
    n = L.mapdn_launch_count(env._h)
    assert L.mapdn_step_autoreset(env._h, A, 1, *P, None, None, None, None, None, None, None) == 0
    assert L.mapdn_launch_count(env._h) == n + 1
    env.close()
    bare = make_env(net, None, dict(seed=1), batch=3)
    refused(bare._h, L.mapdn_step_autoreset(bare._h, A, 1, *P, None, None, None, None, None, None, None),
            "without a profile store")
    bare.close()
