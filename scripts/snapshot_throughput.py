"""Time of env state snapshots on the GPU (BatchedVoltageControl.snapshot / restore / fork), with the step for scale:

  snapshot  mapdn_snapshot of all envs into a preallocated buffer (one launch)
  restore   mapdn_restore of all envs from it (one launch; without the obs / state re-gathers of env.restore)
  fork      env.fork(src, dst) of B / 2 envs: the index upload, snapshot into a temporary, restore, and the re-gathers
  step      one auto-reset step launch (env.step_autoreset)

    python scripts/snapshot_throughput.py [--iters 50] [--reps 3] [--out DIR]

Configs: the benchmark's four (case33 x 4096, case141 x 2048, case322 x 512 / x 1024), each with history 1 and 3. The
kinds alternate within every repetition after a warm-up of each; before every timed call the L2 cache is flushed (256 MiB
memset outside the event pair), then a CUDA-event pair around the call. Prints bytes per env, the HBM bytes a snapshot or
restore moves (read + write, computed from the layout: an estimate of the traffic, not a measurement) and the implied
bandwidth, and the GPU name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mapdn_b200 import cases                         # noqa: E402
from mapdn_b200.env import BatchedVoltageControl, _ptr   # noqa: E402

CONFIGS = (("case33", 4096), ("case141", 2048), ("case322", 512), ("case322", 1024))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def run(name, B, H, iters, reps, flush):
    net, prof = cases.make_case(name), cases.make_profiles(name, n_days=4)
    args = dict(voltage_barrier_type=cases.SCENARIOS[name]["barrier"], action_scale=cases.SCENARIOS[name]["action_scale"],
                episode_limit=480, seed=3, history=H)
    env = BatchedVoltageControl(net, prof, args, batch=B)
    env.reset()
    bpe = env.snapshot_layout[-1]
    buf = torch.empty(B, bpe, dtype=torch.uint8, device=env.device)
    acts = (torch.rand(8, B, env.n_agents, device=env.device, dtype=torch.float64) * 2 - 1) * args["action_scale"]
    src, dst = torch.arange(B // 2), torch.arange(B // 2, B)
    st = env._stream

    def call(kind, t):
        if kind == "snapshot":
            env._L.mapdn_snapshot(env._h, None, B, _ptr(buf), st())
        elif kind == "restore":
            env._L.mapdn_restore(env._h, None, B, _ptr(buf), st())
        elif kind == "fork":
            env.fork(src, dst)
        else:
            env.step_autoreset(acts[t % acts.shape[0]])

    kinds = ("step", "snapshot", "restore", "fork")
    env.fingerprint                                   # hashed once, outside the timed window
    for kind in kinds:
        for t in range(3):
            call(kind, t)
    torch.cuda.synchronize()
    res = {k: [] for k in kinds}
    for _ in range(reps):
        for kind in kinds:
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
            for t in range(iters):
                flush.zero_()
                ev[t][0].record()
                call(kind, t)
                ev[t][1].record()
            torch.cuda.synchronize()
            res[kind].append(sum(a.elapsed_time(b) for a, b in ev) * 1e3 / iters)
    moved = 2 * B * bpe                               # every byte of a row read once and written once
    med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
    out = dict(config=f"{name} x {B}", history=H, bytes_per_env=bpe, mb_moved_per_call=round(moved / 1e6, 2),
               us_median={k: round(v, 2) for k, v in med.items()},
               us_all={k: [round(x, 2) for x in v] for k, v in res.items()},
               gb_per_s={k: round(moved / (med[k] * 1e-6) / 1e9, 1) for k in ("snapshot", "restore")})
    print(json.dumps(out), flush=True)
    env.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("snapshot_throughput.py measures on the GPU; there is no CPU fallback")
    gpu = gpu_info()
    print("gpu:", gpu, flush=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    res = [run(name, B, H, a.iters, a.reps, flush) for name, B in CONFIGS for H in (1, 3)]
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "snapshot_throughput.json"), "w") as f:
            json.dump(dict(gpu=gpu, l2="flushed before every call", results=res), f, indent=1)


if __name__ == "__main__":
    main()
