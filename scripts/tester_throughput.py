"""Tester step time on the GPU: 480 noise-free steps of B test days (test.py's single-day protocol, episode_limit 480)
with the six tester records written by the step kernel (``step(..., record=)``: one launch per step) against the same
steps followed by six ``get_field`` gathers copied into the record rows (seven launches plus copies per step).

    python scripts/tester_throughput.py [--reps 2] [--out DIR]

Configs: case33 x 730 days and case322 x 512 days. The days cycle through the first 30 days of a 32-day synthetic profile
store (the step time does not depend on the calendar). Actions are fixed random values (no policy network in the timed
loop). CUDA events around the 480 steps, after a warm-up episode; the variants alternate. Prints the GPU name and power
limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mapdn_b200 import cases                         # noqa: E402
from mapdn_b200.env import BatchedVoltageControl     # noqa: E402

FIELDS = ("p_sgen", "q_sgen", "p_bus", "q_bus", "vm", "line_loss")
T = 480


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def episode(env, start, acts, buf, fused):
    env.reset(start, add_noise=False)
    env.record(buf[:, 0])
    sl = env.record_slices
    for t in range(T):
        if fused:
            env.step(acts[t % acts.shape[0]], add_noise=False, want_obs=True, record=buf[:, t + 1])
        else:
            env.step(acts[t % acts.shape[0]], add_noise=False, want_obs=True)
            for f, k in zip(FIELDS, sl):
                o, w = sl[k]
                buf[:, t + 1, o:o + w].copy_(env.get_field(f))


def run(name, n_days, reps):
    net, prof = cases.make_case(name), cases.make_profiles(name, n_days=32)
    env = BatchedVoltageControl(net, prof, dict(voltage_barrier_type=cases.SCENARIOS[name]["barrier"], episode_limit=T,
                                                action_scale=cases.SCENARIOS[name]["action_scale"]), batch=n_days)
    dev = env.device
    start = torch.tensor([[d % 30, 23, 2] for d in range(n_days)], dtype=torch.int32, device=dev)
    g = torch.Generator(device=dev).manual_seed(5)
    acts = (torch.rand(16, n_days, env.n_agents, generator=g, device=dev, dtype=torch.float64) * 2 - 1) * 0.5
    buf = torch.empty(n_days, T + 1, env.record_len, dtype=torch.float64, device=dev)
    out = []
    for fused in (True, False):                           # warm-up of both paths
        episode(env, start, acts, buf, fused)
    torch.cuda.synchronize()
    for r in range(reps):
        for fused in (True, False):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            episode(env, start, acts, buf, fused)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1)
            out.append(dict(config=f"{name} x {n_days} days", records="fused" if fused else "six get_field", rep=r,
                            us_per_step=round(ms * 1e3 / T, 2)))
            print(json.dumps(out[-1]), flush=True)
    env.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = gpu_info()
    print("gpu:", gpu, flush=True)
    res = run("case33", 730, a.reps) + run("case322", 512, a.reps)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "tester_throughput.json"), "w") as f:
            json.dump(dict(gpu=gpu, results=res), f, indent=1)


if __name__ == "__main__":
    main()
