"""Lock-step time of the batched training loops' env work on the GPU, three variants per config:

  (a) separate  step, then reset(mask = terminated, want_state = False): the reset launch (and, with history, the
                frame-0 kernel and the stacked-row gather) on every lock-step, as the loops did before auto-reset
  (b) fused     step_autoreset: one launch; the envs that terminate are reset inside it
  (c) step      the plain step launch alone, no reset: what a lock-step where no env ends costs without the auto-reset
                instantiation (its rows after the episode boundary are not comparable and are left out)

    python scripts/autoreset_throughput.py [--reps 3] [--out DIR]

Configs: case33 x 4096 and case322 x 1024 (the benchmark's batch sizes), each with history 1 and 3. Every repetition runs
one full episode (episode_limit = 240 lock-steps from a reset, so the last one is the boundary where every env ends) on
each variant in turn, with fixed random actions and noisy steps. Per lock-step: the L2 cache is flushed (256 MiB memset,
outside the event pair), then a CUDA-event pair around the variant's env work. Lock-steps are reported by how many envs
ended in them: none, all (the episode boundary), or some (divergence). The two variants' outputs are compared over one
episode before timing. Prints the GPU name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mapdn_b200 import cases                         # noqa: E402
from mapdn_b200.env import BatchedVoltageControl     # noqa: E402

LIMIT = 240


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def lock_step(kind, env, a):
    if kind == "fused":
        return env.step_autoreset(a)[1]
    done = env.step(a)[1]
    if kind == "step":
        return done
    env.reset(mask=done, want_state=False)
    return done


def run(name, B, H, reps, flush):
    net, prof = cases.make_case(name), cases.make_profiles(name, n_days=4)
    args = dict(voltage_barrier_type=cases.SCENARIOS[name]["barrier"], action_scale=cases.SCENARIOS[name]["action_scale"],
                episode_limit=LIMIT, seed=3, history=H)
    envs = {k: BatchedVoltageControl(net, prof, args, batch=B) for k in ("separate", "fused", "step")}
    dev = envs["fused"].device
    g = torch.Generator(device=dev).manual_seed(5)
    acts = (torch.rand(16, B, envs["fused"].n_agents, generator=g, device=dev, dtype=torch.float64) * 2 - 1) * args["action_scale"]
    # one episode on both: the same transitions and the same first observations of the new episodes
    s, f = envs["separate"], envs["fused"]
    s.reset(); f.reset()
    tol = 0.0 if f.dims["lanes_per_env"] <= 32 else 1e-10
    for t in range(LIMIT + 1):
        ds, df = lock_step("separate", s, acts[t % 16]), lock_step("fused", f, acts[t % 16])
        assert torch.equal(ds, df), t
        for x, y in ((s.reward, f.reward), (s.info, f.info)):
            assert float((x - y).abs().max()) <= tol, t
        m = df.bool()
        first_s = s.obs_stacked if H > 1 else s.obs
        first_f = f.reset_obs_stacked if H > 1 else f.reset_obs
        if bool(m.any()):
            assert float((first_s[m] - first_f[m]).abs().max()) <= tol, t
    out = []
    for r in range(reps):
        for kind, env in envs.items():
            env.reset()
            torch.cuda.synchronize()
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(LIMIT)]
            ended = torch.zeros(LIMIT, dtype=torch.int64, device=dev)
            for t in range(LIMIT):
                if flush is not None:
                    flush.zero_()
                ev[t][0].record()
                done = lock_step(kind, env, acts[t % 16])
                ev[t][1].record()
                ended[t] = done.sum()
            torch.cuda.synchronize()
            ms = [a.elapsed_time(b) for a, b in ev]
            n_end = ended.tolist()
            groups = dict(no_env_ends=[m for m, n in zip(ms, n_end) if n == 0],
                          all_envs_end=[m for m, n in zip(ms, n_end) if n == B],
                          some_envs_end=[m for m, n in zip(ms, n_end) if 0 < n < B])
            row = dict(config=f"{name} x {B}", history=H, variant=kind, rep=r)
            if kind == "step":          # no reset: after the boundary every env stays terminated
                groups = dict(no_env_ends=groups["no_env_ends"])
            for k, v in groups.items():
                row[k] = dict(lock_steps=len(v), us_mean=round(1e3 * sum(v) / len(v), 2) if v else None)
            if kind != "step":
                row["episode_ms"] = round(sum(ms), 3)
            out.append(row)
            print(json.dumps(row), flush=True)
    for env in envs.values():
        env.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-flush", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("autoreset_throughput.py measures on the GPU; there is no CPU fallback")
    gpu = gpu_info()
    print("gpu:", gpu, flush=True)
    flush = None if a.no_flush else torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    res = []
    for name, B in (("case33", 4096), ("case322", 1024)):
        for H in (1, 3):
            res += run(name, B, H, a.reps, flush)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "autoreset_throughput.json"), "w") as f:
            json.dump(dict(gpu=gpu, l2="flushed before every lock-step" if flush is not None else "not flushed", results=res),
                      f, indent=1)


if __name__ == "__main__":
    main()
