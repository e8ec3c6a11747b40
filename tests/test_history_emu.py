"""CPU tier for the observation history (mapdn_set_history / mapdn_step_stacked / mapdn_get_obs_stacked), on the kernel
source compiled for the CPU SIMT emulation (tests/emu).

A handle with history H keeps a frame ring on the device; every reset and every step records the env's newest frame,
whichever entry point ran it. The stacked rows (reference get_obs :303-315: the last H frames side by side, oldest first,
zero frames before the episode start) written by the step kernel and by the standalone gather must equal the rule applied
in NumPy to the single frames of the same launches, bit for bit, and history must be a pure side output: every other
output equals that of a history = 1 handle with the same seed."""
import json
import os
import sys

import numpy as np
import pytest

from conftest import ROOT
from mapdn_b200 import cases
from mapdn_b200.network import ProfileDesc
from oracle import ref_scenarios as S

sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
import emu_env                                                       # noqa: E402
from emu_env import EmuEnv, _ptr                                     # noqa: E402

FIELDS = ("vm", "va_deg", "p_bus", "q_bus", "p_sgen", "q_sgen", "line_loss", "p_load", "q_load", "sum_rewards", "steps",
          "start_row", "nr_iters")


def _lib():
    return emu_env.lib()


def _overload(net, prof, factor=60.0):
    """The profile with rows 60..459 carrying a demand the feeder cannot serve (the divergence branch of step)."""
    lp = prof.load_p.copy(); lp[60:460] *= factor
    return net, ProfileDesc(pv=prof.pv, load_p=lp, load_q=prof.load_q, steps_per_hour=prof.steps_per_hour, n_days=prof.n_days)


def _mesh():
    from mapdn_b200.network import NetDesc
    z = np.array([0.02 + 0.04j, 0.01 + 0.03j, 0.0125 + 0.025j, 0.015 + 0.03j])
    net = NetDesc(base_mva=100.0, n_bus=4, slack_bus=0, slack_vm=1.03, br_from=np.array([0, 0, 1, 2]), br_to=np.array([1, 2, 2, 3]),
                  br_r=z.real, br_x=z.imag, load_bus=np.array([1, 2, 3]), sgen_bus=np.array([2, 3]), sgen_zone=np.array([1, 1]),
                  bus_zone=np.array([0, 1, 1, 1]), name="mesh4")
    rng = np.random.default_rng(3)
    T = 4 * 24 * 20 + 1
    prof = ProfileDesc(pv=rng.uniform(0, 40, (T, 2)), load_p=rng.uniform(60, 180, (T, 3)), load_q=rng.uniform(10, 60, (T, 3)),
                       steps_per_hour=20)
    return net, prof


def set_history(env, H):
    return _lib().mapdn_set_history(env._h, H)


def step_stacked(env, a, stacked, obs=True, rec=None, add_noise=True):
    """mapdn_step_stacked on an EmuEnv; returns the status."""
    a = np.ascontiguousarray(a, np.float64)
    return _lib().mapdn_step_stacked(env._h, _ptr(a), int(add_noise), _ptr(env.reward), _ptr(env.term), _ptr(env.info),
                                     _ptr(env.obs) if obs else None, _ptr(stacked), _ptr(rec),
                                     0 if rec is None else rec.strides[0] // 8, None)


def get_stacked(env, H):
    out = np.full((env.batch, env.dims["n_agents"], H * env.dims["obs_dim"]), np.nan)
    env._chk(_lib().mapdn_get_obs_stacked(env._h, _ptr(out), None))
    return out


def stacking_rule(frames, H):
    """frames: per env, the frames since its last reset (oldest first) -> [B, n_agents, H * obs_dim]."""
    rows = []
    for fr in frames:
        z = np.zeros_like(fr[0])
        last = ([z] * H + fr)[-H:]
        rows.append(np.concatenate(last, axis=1))
    return np.stack(rows)


def _same(a, b, exact, what):
    if exact:
        assert np.array_equal(a, b), what
    else:
        assert a.shape == b.shape and np.abs(a - b).max() <= 1e-10, (what, float(np.abs(a - b).max()))


def _set_geometry(monkeypatch, geom):
    for k in ("MAPDN_PLAN", "MAPDN_EPB", "MAPDN_HELPERS", "MAPDN_EMU_SMS"):
        monkeypatch.delenv(k, raising=False)
    for k, v in geom.items():
        monkeypatch.setenv(k, str(v))


# step paths of the handle with history, cycled; the history = 1 handle always takes mapdn_step_record with obs
KINDS = ("stacked", "record", "pinned", "no_obs", "f32", "plain")


def run_history(monkeypatch, net, prof, args, batch, lanes, H, geom, diverge_env):
    _set_geometry(monkeypatch, geom)
    plain = EmuEnv(net, prof, args, batch=batch, lanes_per_env=lanes)
    hist = EmuEnv(net, prof, args, batch=batch, lanes_per_env=lanes)
    assert set_history(hist, H) == 0
    d = hist.dims
    exact = d["lanes_per_env"] <= 32
    grid_rounds = []
    ng, od = d["n_agents"], d["obs_dim"]
    _, R = hist.record_layout()
    B = batch

    plain.reset(None, add_noise=True); hist.reset(None, add_noise=True)
    _same(plain.obs, hist.obs, exact, "reset obs")
    frames = [[plain.obs[b].copy()] for b in range(B)]
    got = get_stacked(hist, H)
    assert np.array_equal(got, stacking_rule(frames, H))
    assert np.all(got[:, :, :(H - 1) * od] == 0.0)                   # before the episode start: exactly zero

    rng = np.random.default_rng(H + 10 * d["lanes_per_env"])
    scale = float(args.get("action_scale", 0.8))
    n_steps = 2 * H + 4
    mid = H + 2                                         # the ring has wrapped: masked reset of two envs before this step
    mask = np.zeros(B, np.uint8); mask[[diverge_env, B - 1]] = 1
    start = np.tile(np.array([[1, 5, 3]], np.int32), (B, 1))
    start[diverge_env] = (0, 2, 18)                     # row 58: the reset solves row 59, its second step diverges
    diverged = False
    for t in range(n_steps):
        if t == mid:
            plain.reset(start, add_noise=True, mask=mask); hist.reset(start, add_noise=True, mask=mask)
            assert np.array_equal(plain.reset_ok[mask == 1], hist.reset_ok[mask == 1]) and hist.reset_ok[mask == 1].all()
            _same(plain.obs[mask == 1], hist.obs[mask == 1], exact, "masked reset obs")
            for b in np.nonzero(mask)[0]:
                frames[b] = [plain.obs[b].copy()]
            got = get_stacked(hist, H)
            assert np.array_equal(got, stacking_rule(frames, H))
            assert np.all(got[mask == 1][:, :, :(H - 1) * od] == 0.0)
        kind = KINDS[t % len(KINDS)]
        a = rng.uniform(-scale, scale, (B, ng))
        rec0, rec1 = np.full((B, R + 2), np.nan), np.full((B, R + 2), np.nan)
        r0, t0, i0 = [x.copy() for x in plain.step_record(a, rec0[:, :R])]
        stacked = np.full((B, ng, H * od), np.nan)
        if kind in ("stacked", "record", "no_obs"):
            hist.obs[:] = np.nan
            st = step_stacked(hist, a, None if kind == "no_obs" else stacked, obs=kind != "no_obs",
                              rec=rec1[:, :R] if kind == "record" else None)
            assert st == 0, _lib().mapdn_last_error()
            r1, t1, i1, o1 = hist.reward.copy(), hist.term.copy(), hist.info.copy(), hist.obs.copy()
        elif kind == "plain":
            r1, t1, i1 = [x.copy() for x in hist.step(a)]
            o1 = hist.obs.copy()
        else:
            r1, t1, i1, o1 = hist.step_host(a, f32=kind == "f32", path="pinned" if kind == "pinned" else "staged")
        grid_rounds.append(-(-(-(-B // d["envs_per_block"])) // hist.last_grid()))     # rounds of this step's launch
        _same(r0, r1, exact, (kind, t, "reward")); assert np.array_equal(t0, t1), (kind, t)
        _same(i0, i1, exact, (kind, t, "info"))
        if kind == "f32":
            assert np.array_equal(plain.obs.astype(np.float32), o1) if exact else np.abs(plain.obs - o1).max() < 1e-5
        elif kind != "no_obs":
            _same(plain.obs, o1, exact, (kind, t, "obs"))
        else:
            assert np.all(np.isnan(o1))                                        # nothing written
        if kind == "record":
            _same(rec0[:, :R], rec1[:, :R], exact, (t, "record")); assert np.all(np.isnan(rec1[:, R:]))
        for k in FIELDS:
            _same(plain.get_field(k), hist.get_field(k), exact, (kind, t, k))
        _same(plain.get_state(), hist.get_state(), exact, (kind, t, "state"))
        for b in range(B):
            frames[b].append(plain.obs[b].copy())
        want = stacking_rule(frames, H)
        got = get_stacked(hist, H)
        # the ring holds the padded fp64 frames of the history handle's own launches: exact against them
        if exact:
            assert np.array_equal(got, want), (kind, t)
        else:
            assert np.abs(got - want).max() <= 1e-10, (kind, t)
        if kind in ("stacked", "record"):
            assert np.array_equal(stacked, got), (kind, t)                     # fused == gather, bit for bit
        diverged |= bool(i1[diverge_env, 10] == 1.0)
    assert diverged
    assert min(grid_rounds) >= 2 and B % d["envs_per_block"] != 0, (grid_rounds, d["envs_per_block"])   # ragged last CTA
    plain.close(); hist.close()
    return d


def _case(name):
    # case322's synthetic demand is light: 60 times of it can still be served
    return _overload(cases.make_case(name), cases.make_profiles(name, n_days=4), 3000.0 if name == "case322" else 60.0)


@pytest.mark.parametrize("H", [2, 3, 5])
def test_case33_stacked_rows(monkeypatch, H):
    net, prof = _case("case33")
    d = run_history(monkeypatch, net, prof, dict(voltage_barrier_type="l1", seed=3, action_scale=0.8), batch=24, lanes=0,
                    H=H, geom=dict(MAPDN_EMU_SMS=1, MAPDN_EPB=20), diverge_env=5)
    assert d["lanes_per_env"] == 8


@pytest.mark.parametrize("name,lanes,batch,epb", [("case141", 32, 9, 4), ("case322", 64, 4, 3), ("case322", 128, 3, 2)])
def test_large_feeders_stacked_rows(monkeypatch, name, lanes, batch, epb):
    net, prof = _case(name)
    d = run_history(monkeypatch, net, prof, dict(voltage_barrier_type="bowl", seed=4,
                                                 action_scale=cases.SCENARIOS[name]["action_scale"]),
                    batch=batch, lanes=lanes, H=3, geom=dict(MAPDN_EMU_SMS=1, MAPDN_EPB=epb), diverge_env=1)
    assert d["lanes_per_env"] == lanes


def test_dense_meshed_fallback_stacked_rows(monkeypatch):
    net, prof = _overload(*_mesh())
    run_history(monkeypatch, net, prof, dict(voltage_barrier_type="l2", seed=2, episode_limit=48), batch=5, lanes=0, H=3,
                geom=dict(MAPDN_EMU_SMS=1, MAPDN_EPB=2), diverge_env=1)


def reference_rows_one_frame_per_transition(g, ops, H, od):
    """The reference's stacked rows of the fixture, as one frame per reset / step gives them. The reference stacks one
    frame per get_obs() call (:303-315), and its constructor's reset (:85) calls get_obs() before the recording's own
    call at "init": the initial frame sits in its history twice. Until H - 1 steps later that duplicate shows in the
    oldest non-zero block; here it is checked to be the initial frame and replaced by the zero frame the engine holds."""
    rows = [g["obs"][k, 0].copy() for k in range(len(ops))]
    assert ops[0] == ("init",)
    for i in range(H - 1):                                   # op i: i steps after the construction
        if i >= len(ops) or (i > 0 and ops[i][0] != "step"):
            break
        k = H - 2 - i                                        # block of the duplicate
        assert np.array_equal(rows[i][:, k * od:(k + 1) * od], g["obs"][0, 0][:, (H - 1) * od:])
        rows[i][:, k * od:(k + 1) * od] = 0.0
    return rows


def test_reference_history_fixture_on_the_emulation():
    """tests/golden/ref_env_case33_history.npz holds the reference's own stacked rows (history = 3, a second episode):
    the fused rows and the gather reproduce all of them, not just the newest frame (frames per reset / step; the
    duplicate of the constructor's frame aside, see reference_rows_one_frame_per_transition)."""
    g = np.load(S.fixture_path(ROOT, "case33_history"))
    ops = [tuple(op) for op in json.loads(str(g["ops"]))]
    sc = S.SCENARIOS["case33_history"]
    net, prof = sc["build"]()
    H = sc["args"]["history"]
    env = EmuEnv(net, prof, sc["args"], batch=1)
    assert set_history(env, H) == 0
    assert g["obs"].shape[-1] == H * env.dims["obs_dim"]
    want = reference_rows_one_frame_per_transition(g, ops, H, env.dims["obs_dim"])
    t = 0
    for k_op, op in enumerate(ops):
        if op[0] == "step":
            stacked = np.full((1, net.n_sgen, H * env.dims["obs_dim"]), np.nan)
            assert step_stacked(env, g["actions"][t], stacked, add_noise=op[1]) == 0
            assert np.array_equal(stacked, get_stacked(env, H))
            t += 1
        else:
            assert op[0] in ("init", "reset")
            env.reset()
        assert np.abs(get_stacked(env, H)[0] - want[k_op]).max() < 1e-9, (k_op, op)
    env.close()


def test_refusals_and_the_history_lifecycle():
    """Refusals leave the launch count alone; H = 1 frees the ring, H > 1 (again) records from the next reset on; a reset
    of a handle with history is two launches (the reset, frame 0 into the ring), a step one."""
    L = _lib()
    net, prof = cases.make_case("case33"), cases.make_profiles("case33", n_days=4)
    env = EmuEnv(net, prof, dict(seed=1), batch=3)
    od, ng, B = env.dims["obs_dim"], net.n_sgen, 3
    a = np.zeros((B, ng))
    buf = np.zeros((B, 5 * ng * od))
    n = L.mapdn_launch_count(env._h)

    def refused(st, text):
        assert st == 1 and text in L.mapdn_last_error().decode(), L.mapdn_last_error()
        assert L.mapdn_launch_count(env._h) == n

    refused(L.mapdn_set_history(None, 3), "null handle")
    refused(set_history(env, 0), "history must be >= 1")
    refused(set_history(env, -2), "history must be >= 1")
    refused(step_stacked(env, a, buf), "no observation history")
    refused(L.mapdn_get_obs_stacked(env._h, _ptr(buf), None), "no observation history")
    refused(L.mapdn_get_obs_stacked(None, _ptr(buf), None), "null argument")
    refused(L.mapdn_step_stacked(None, _ptr(a), 1, _ptr(env.reward), _ptr(env.term), None, None, None, None, 0, None), "null argument")
    assert set_history(env, 3) == 0
    rec = np.zeros((B, 4))
    refused(step_stacked(env, a, buf, rec=rec), "record_stride")
    refused(L.mapdn_get_obs_stacked(env._h, None, None), "null argument")

    frames = None
    for H in (3, 1, 2):
        assert set_history(env, H) == 0
        env.reset()
        n = L.mapdn_launch_count(env._h)
        if H == 1:
            refused(step_stacked(env, a, buf), "no observation history")
            env.step(a)
            assert L.mapdn_launch_count(env._h) == n + 1
            continue
        frames = [[env.obs[b].copy()] for b in range(B)]
        assert np.array_equal(get_stacked(env, H), stacking_rule(frames, H))
        n = L.mapdn_launch_count(env._h)
        for _ in range(H + 1):
            st = np.zeros((B, ng, H * od))
            assert step_stacked(env, a, st) == 0
            for b in range(B):
                frames[b].append(env.obs[b].copy())
            assert np.array_equal(st, stacking_rule(frames, H))
        assert L.mapdn_launch_count(env._h) == n + H + 1
        env.reset(mask=np.array([0, 1, 0], np.uint8))
        assert L.mapdn_launch_count(env._h) == n + H + 3
        frames[1] = [env.obs[1].copy()]
        assert np.array_equal(get_stacked(env, H), stacking_rule(frames, H))
    env.close()
