"""Step time with observation history (history = 3) on the GPU, three variants per config:

  (a) plain    history = 1: one step launch (the single-frame observations only)
  (b) fused    history = 3: one step launch that also writes the frame ring and the stacked rows (mapdn_step_stacked)
  (c) former   history = 1 step, then the torch ring the batched env used to keep: torch.roll of the whole ring [B, H,
               n_agents, obs_dim], the copy of the newest frame into it, and get_obs_stacked (permute + reshape copy)

    python scripts/history_throughput.py [--steps 200] [--reps 3] [--out DIR]

Configs: case33 x 4096 and case322 x 1024 (the benchmark's batch sizes). Fixed random actions, noisy steps, no policy.
Per step: the L2 cache is flushed (256 MiB memset, outside the event pair), then a CUDA-event pair around the variant's
work; the time reported is the sum over the steps. The variants alternate within every repetition, after a warm-up of
each. The three variants' outputs are compared before timing (reward, terminated, info, obs and the stacked rows).
Prints the GPU name and power limit read in the same run, and the per-step HBM traffic that the ring work adds, computed
from the shapes (an estimate, not a measurement)."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mapdn_b200 import cases                         # noqa: E402
from mapdn_b200.env import BatchedVoltageControl     # noqa: E402

H = 3


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def traffic_mb(B, n_agents, obs_dim):
    """Extra bytes per step over the plain step, from the shapes: (c) the roll reads and writes the ring, the newest
    frame is read and written into it, get_obs_stacked reads the ring and writes the rows; (b) the ring write of the
    newest frame, the ring read of the H - 1 older frames, the stacked-row write."""
    f = 8 * B * n_agents * obs_dim / 1e6                  # one frame of every env, MB
    return dict(former_roll_and_copy=2 * H * f + 2 * f, former_with_get_obs_stacked=2 * H * f + 2 * f + 2 * H * f,
                fused=f + (H - 1) * f + H * f)


def run(name, B, steps, reps, flush):
    net, prof = cases.make_case(name), cases.make_profiles(name, n_days=4)
    args = dict(voltage_barrier_type=cases.SCENARIOS[name]["barrier"], action_scale=cases.SCENARIOS[name]["action_scale"],
                episode_limit=480, seed=3)
    envs = dict(plain=BatchedVoltageControl(net, prof, args, batch=B),
                fused=BatchedVoltageControl(net, prof, dict(args, history=H), batch=B),
                former=BatchedVoltageControl(net, prof, args, batch=B))
    dev = envs["plain"].device
    na, od = envs["plain"].n_agents, envs["plain"].obs_size
    g = torch.Generator(device=dev).manual_seed(5)
    acts = (torch.rand(16, B, na, generator=g, device=dev, dtype=torch.float64) * 2 - 1) * args["action_scale"]
    ring = torch.zeros(B, H, na, od, dtype=torch.float64, device=dev)
    sink = {}

    def one_step(kind, t):
        nonlocal ring
        env = envs[kind]
        env.step(acts[t % acts.shape[0]])
        if kind == "former":
            ring = torch.roll(ring, -1, dims=1)
            ring[:, -1] = env.obs
            sink["stacked"] = ring.permute(0, 2, 1, 3).reshape(B, na, H * od)

    # the same trajectory on all three: check that history changes nothing else, then warm up
    for env in envs.values():
        env.reset()
    # (bit for bit up to 32 lanes per env; 64 / 128 lanes: separately compiled instantiations may round differently)
    tol = 0.0 if envs["plain"].dims["lanes_per_env"] <= 32 else 1e-10
    p, f = envs["plain"], envs["fused"]
    for t in range(3):
        for kind in envs:
            one_step(kind, t)
        assert torch.equal(p.terminated, f.terminated)
        for x, y in ((p.reward, f.reward), (p.info, f.info), (p.obs, f.obs)):
            assert float((x - y).abs().max()) <= tol
    assert float((f.obs_stacked - sink["stacked"]).abs().max()) <= tol    # H steps after the reset: the same frames
    out = []
    for r in range(reps):
        for kind in envs:
            envs[kind].reset()
            torch.cuda.synchronize()
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
            for t in range(steps):
                if flush is not None:
                    flush.zero_()
                ev[t][0].record()
                one_step(kind, t)
                ev[t][1].record()
            torch.cuda.synchronize()
            ms = sum(a.elapsed_time(b) for a, b in ev)
            out.append(dict(config=f"{name} x {B}", history=H, variant=kind, rep=r, us_per_step=round(ms * 1e3 / steps, 2),
                            M_env_steps_per_s=round(B * steps / ms / 1e3, 2)))
            print(json.dumps(out[-1]), flush=True)
    est = {k: round(v, 1) for k, v in traffic_mb(B, na, od).items()}
    print(json.dumps(dict(config=f"{name} x {B}", extra_hbm_mb_per_step_estimate=est)), flush=True)
    for env in envs.values():
        env.close()
    return out, est


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-flush", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("history_throughput.py measures on the GPU; there is no CPU fallback")
    gpu = gpu_info()
    print("gpu:", gpu, flush=True)
    flush = None if a.no_flush else torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    res = {}
    for name, B in (("case33", 4096), ("case322", 1024)):
        res[f"{name} x {B}"] = run(name, B, a.steps, a.reps, flush)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "history_throughput.json"), "w") as f:
            json.dump(dict(gpu=gpu, l2="flushed before every step" if flush is not None else "not flushed", results=res),
                      f, indent=1)


if __name__ == "__main__":
    main()
