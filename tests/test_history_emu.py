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
import torch

import geometry_cases as GC
from conftest import ROOT
from mapdn_b200 import cases
from oracle import ref_scenarios as S

sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
from emu_env import last_grid, make_env, nan_filled_outputs          # noqa: E402,F401  (autouse fixture)

NAN = float("nan")


def stacking_rule(frames, H):
    """frames: per env, the frames since its last reset (oldest first) -> [B, n_agents, H * obs_dim]."""
    rows = []
    for fr in frames:
        z = np.zeros_like(fr[0])
        last = ([z] * H + fr)[-H:]
        rows.append(np.concatenate(last, axis=1))
    return np.stack(rows)


# step paths of the handle with history, cycled; the history = 1 handle always takes mapdn_step_record with obs
KINDS = ("stacked", "record", "pinned", "no_obs", "f32", "plain")


def run_history(monkeypatch, net, prof, args, batch, lanes, H, geom, diverge_env):
    GC.set_geometry(monkeypatch, geom)
    plain = make_env(net, prof, args, batch=batch, lanes_per_env=lanes)
    hist = make_env(net, prof, dict(args, history=H), batch=batch, lanes_per_env=lanes)
    d = hist.dims
    exact = d["lanes_per_env"] <= 32
    grid_rounds = []
    ng, od = d["n_agents"], d["obs_dim"]
    R = hist.record_len
    B = batch
    p_obs, h_obs, stacked = plain.obs.numpy(), hist.obs.numpy(), hist.obs_stacked.numpy()

    plain.reset(None, add_noise=True)
    hist.obs_stacked[:] = NAN
    hist.reset(None, add_noise=True)
    GC.same(p_obs, h_obs, exact, "reset obs")
    frames = [[p_obs[b].copy()] for b in range(B)]
    assert np.array_equal(stacked, stacking_rule(frames, H))
    assert np.all(stacked[:, :, :(H - 1) * od] == 0.0)               # before the episode start: exactly zero

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
            plain.reset(torch.from_numpy(start), add_noise=True, mask=torch.from_numpy(mask))
            hist.obs_stacked[:] = NAN
            hist.reset(torch.from_numpy(start), add_noise=True, mask=torch.from_numpy(mask))
            p_ok, h_ok = plain.reset_ok.numpy(), hist.reset_ok.numpy()
            assert np.array_equal(p_ok[mask == 1], h_ok[mask == 1]) and h_ok[mask == 1].all()
            GC.same(p_obs[mask == 1], h_obs[mask == 1], exact, "masked reset obs")
            for b in np.nonzero(mask)[0]:
                frames[b] = [p_obs[b].copy()]
            assert np.array_equal(stacked, stacking_rule(frames, H))
            assert np.all(stacked[mask == 1][:, :, :(H - 1) * od] == 0.0)
        kind = KINDS[t % len(KINDS)]
        a = torch.from_numpy(rng.uniform(-scale, scale, (B, ng)))
        rec0, rec1 = torch.full((B, R + 2), NAN, dtype=torch.float64), torch.full((B, R + 2), NAN, dtype=torch.float64)
        r0, t0, i0 = [x.numpy().copy() for x in plain.step(a, record=rec0[:, :R])]
        hist.obs_stacked[:] = NAN
        if kind in ("stacked", "record", "no_obs"):
            hist.obs[:] = NAN
            r1, t1, i1 = [x.numpy().copy() for x in hist.step(a, want_obs=kind != "no_obs",
                                                             record=rec1[:, :R] if kind == "record" else None)]
            o1 = h_obs.copy()
        elif kind == "plain":                           # mapdn_step on a handle with history: the ring still records
            L = hist._L
            assert L.mapdn_step(hist._h, a.data_ptr(), 1, hist.reward.data_ptr(), hist.terminated.data_ptr(),
                                hist.info.data_ptr(), hist.obs.data_ptr(), None) == 0, L.mapdn_last_error()
            r1, t1, i1, o1 = hist.reward.numpy().copy(), hist.terminated.numpy().copy(), hist.info.numpy().copy(), h_obs.copy()
        else:
            host = hist._host_buffers()                 # padded host rows: the pinned path never writes the padding
            host["obs"].zero_(); host["obs32"][:] = NAN
            r1, t1, i1, o1 = hist.step_host(a.numpy(), obs_dtype=np.float32 if kind == "f32" else np.float64,
                                            staged=kind == "f32")
        grid_rounds.append(-(-(-(-B // d["envs_per_block"])) // last_grid()))     # rounds of this step's launch
        GC.same(r0, r1, exact, (kind, t, "reward")); assert np.array_equal(t0, t1), (kind, t)
        GC.same(i0, i1, exact, (kind, t, "info"))
        if kind == "f32":
            assert np.array_equal(p_obs.astype(np.float32), o1) if exact else np.abs(p_obs - o1).max() < 1e-5
        elif kind != "no_obs":
            GC.same(p_obs, o1, exact, (kind, t, "obs"))
        else:
            assert np.all(np.isnan(o1)) and np.all(np.isnan(stacked))              # nothing written
        if kind == "record":
            GC.same(rec0[:, :R].numpy(), rec1[:, :R].numpy(), exact, (t, "record")); assert torch.all(rec1[:, R:].isnan())
        for k in GC.FIELDS:
            GC.same(plain.get_field(k).numpy(), hist.get_field(k).numpy(), exact, (kind, t, k))
        GC.same(plain.get_state().numpy(), hist.get_state().numpy(), exact, (kind, t, "state"))
        for b in range(B):
            frames[b].append(p_obs[b].copy())
        want = stacking_rule(frames, H)
        got = hist.get_obs_stacked().numpy()
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


@pytest.mark.parametrize("H", [2, 3, 5])
def test_case33_stacked_rows(monkeypatch, H):
    net, prof = GC.overloaded_case("case33")
    d = run_history(monkeypatch, net, prof, dict(voltage_barrier_type="l1", seed=3, action_scale=0.8), batch=24, lanes=0,
                    H=H, geom=dict(MAPDN_EMU_SMS=1, MAPDN_EPB=20), diverge_env=5)
    assert d["lanes_per_env"] == 8


@pytest.mark.parametrize("name,lanes,batch,epb", [("case141", 32, 9, 4), ("case322", 64, 4, 3), ("case322", 128, 3, 2)])
def test_large_feeders_stacked_rows(monkeypatch, name, lanes, batch, epb):
    net, prof = GC.overloaded_case(name)
    d = run_history(monkeypatch, net, prof, dict(voltage_barrier_type="bowl", seed=4,
                                                 action_scale=cases.SCENARIOS[name]["action_scale"]),
                    batch=batch, lanes=lanes, H=3, geom=dict(MAPDN_EMU_SMS=1, MAPDN_EPB=epb), diverge_env=1)
    assert d["lanes_per_env"] == lanes


def test_dense_meshed_fallback_stacked_rows(monkeypatch):
    net, prof = GC.overload(*GC.mesh4())
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
    env = make_env(net, prof, sc["args"], batch=1)
    assert env.history == H and g["obs"].shape[-1] == H * env.dims["obs_dim"]
    want = reference_rows_one_frame_per_transition(g, ops, H, env.dims["obs_dim"])
    t = 0
    for k_op, op in enumerate(ops):
        env.obs_stacked[:] = NAN
        if op[0] == "step":
            env.step(torch.from_numpy(np.asarray(g["actions"][t], np.float64).reshape(1, net.n_sgen)), add_noise=bool(op[1]))
            assert np.array_equal(env.obs_stacked.numpy(), env.get_obs_stacked().numpy())
            t += 1
        else:
            assert op[0] in ("init", "reset")
            env.reset()
        assert np.abs(env.get_obs_stacked().numpy()[0] - want[k_op]).max() < 1e-9, (k_op, op)
        assert np.abs(env.obs_stacked.numpy()[0] - want[k_op]).max() < 1e-9, (k_op, op)
    env.close()


def test_refusals_and_the_history_lifecycle():
    """Refusals leave the launch count alone; H = 1 frees the ring, H > 1 (again) records from the next reset on; a reset
    of a handle with history is two launches (the reset, frame 0 into the ring), a step one. The history is set on the
    handle directly (mapdn_set_history), so the ring's entry points are called directly too."""
    net, prof = cases.make_case("case33"), cases.make_profiles("case33", n_days=4)
    env = make_env(net, prof, dict(seed=1), batch=3)
    L, h = env._L, env._h
    od, ng, B = env.dims["obs_dim"], net.n_sgen, 3
    a = torch.zeros(B, ng, dtype=torch.float64)
    buf = torch.zeros(B, 5 * ng * od, dtype=torch.float64)
    n = L.mapdn_launch_count(h)

    def step_stacked(out, rec=None):
        return L.mapdn_step_stacked(h, a.data_ptr(), 1, env.reward.data_ptr(), env.terminated.data_ptr(), env.info.data_ptr(),
                                    env.obs.data_ptr(), out.data_ptr(), None if rec is None else rec.data_ptr(),
                                    0 if rec is None else rec.stride(0), None)

    def gather(H):
        out = torch.full((B, ng, H * od), NAN, dtype=torch.float64)
        assert L.mapdn_get_obs_stacked(h, out.data_ptr(), None) == 0, L.mapdn_last_error()
        return out.numpy()

    def refused(st, text):
        assert st == 1 and text in L.mapdn_last_error().decode(), L.mapdn_last_error()
        assert L.mapdn_launch_count(h) == n

    refused(L.mapdn_set_history(None, 3), "null handle")
    refused(L.mapdn_set_history(h, 0), "history must be >= 1")
    refused(L.mapdn_set_history(h, -2), "history must be >= 1")
    refused(step_stacked(buf), "no observation history")
    refused(L.mapdn_get_obs_stacked(h, buf.data_ptr(), None), "no observation history")
    refused(L.mapdn_get_obs_stacked(None, buf.data_ptr(), None), "null argument")
    refused(L.mapdn_step_stacked(None, a.data_ptr(), 1, env.reward.data_ptr(), env.terminated.data_ptr(), None, None, None,
                                 None, 0, None), "null argument")
    assert L.mapdn_set_history(h, 3) == 0
    rec = torch.zeros(B, 4, dtype=torch.float64)
    refused(step_stacked(buf, rec=rec), "record_stride")
    refused(L.mapdn_get_obs_stacked(h, None, None), "null argument")

    frames = None
    obs = env.obs.numpy()
    for H in (3, 1, 2):
        assert L.mapdn_set_history(h, H) == 0
        env.reset()
        n = L.mapdn_launch_count(h)
        if H == 1:
            refused(step_stacked(buf), "no observation history")
            env.step(a)
            assert L.mapdn_launch_count(h) == n + 1
            continue
        frames = [[obs[b].copy()] for b in range(B)]
        assert np.array_equal(gather(H), stacking_rule(frames, H))
        n = L.mapdn_launch_count(h)
        for _ in range(H + 1):
            st = torch.zeros(B, ng, H * od, dtype=torch.float64)
            assert step_stacked(st) == 0
            for b in range(B):
                frames[b].append(obs[b].copy())
            assert np.array_equal(st.numpy(), stacking_rule(frames, H))
        assert L.mapdn_launch_count(h) == n + H + 1
        env.reset(mask=torch.tensor([0, 1, 0], dtype=torch.uint8), want_state=False)
        assert L.mapdn_launch_count(h) == n + H + 3
        frames[1] = [obs[1].copy()]
        assert np.array_equal(gather(H), stacking_rule(frames, H))
    env.close()
