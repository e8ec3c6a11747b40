"""Race check of the kernel source on the CPU: the emulated library (tests/emu) built with -fsanitize=thread. Every CUDA
thread is an OS thread and every barrier (__syncwarp, __syncthreads, bar.sync / arrive / red) a mutex-protected counting
barrier, so ThreadSanitizer's happens-before analysis covers shared AND global memory (compute-sanitizer's racecheck only
sees shared memory) and is stricter than the hardware (no implicit warp-synchronous ordering).
    python scripts/emu_tsan.py            # builds /tmp/mapdn_emu_tsan/libemu_tsan.so, runs reset / step / solve / droop,
                                          # then the auto-reset step at 4, 8, 32 and 64 lanes per env
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = "/tmp/mapdn_emu_tsan"
LIB = os.path.join(OUT, "libemu_tsan.so")
CHILD = r'''
import sys, numpy as np, torch
sys.path.insert(0, %(root)r); sys.path.insert(0, %(root)r + "/tests/emu")
import emu_env
emu_env.LIB = %(lib)r; emu_env.build = lambda force=False: emu_env.LIB
from mapdn_b200 import baselines, cases
name, lanes, B = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
net, prof = cases.make_case(name), cases.make_profiles(name, n_days=3)
scale = cases.SCENARIOS[name]["action_scale"]
env = emu_env.make_env(net, prof, dict(seed=3, voltage_barrier_type="bowl", action_scale=scale), batch=B, lanes_per_env=lanes)
env.reset()
rng = np.random.default_rng(0)
for t in range(2):
    env.step(torch.from_numpy(rng.uniform(-scale, scale, (B, net.n_sgen))))
env.step_host(rng.uniform(-scale, scale, (B, net.n_sgen)), layout="compact")
inp = cases.synthetic_inputs(name, 3, seed=1)
env.solve(inp["p_load"], inp["q_load"], inp["p_pv"], np.zeros_like(inp["p_pv"]))
baselines.droop_control(env, inp["p_load"], inp["q_load"], inp["p_pv"], inp["s_max"], max_ite=6)
print("ran", name, lanes, B)
'''
# auto-reset leg: episodes of 3 steps, half the batch reset early (terminated and running envs in one warp), one env per
# step diverging, >= 2 persistent rounds (MAPDN_EMU_SMS / MAPDN_EPB from the caller)
CHILD_AR = r'''
import sys, numpy as np, torch
sys.path.insert(0, %(root)r); sys.path.insert(0, %(root)r + "/tests/emu")
import emu_env
emu_env.LIB = %(lib)r; emu_env.build = lambda force=False: emu_env.LIB
from mapdn_b200 import cases
from mapdn_b200.network import ProfileDesc
name, lanes, B, H = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4])
net, prof = cases.make_case(name), cases.make_profiles(name, n_days=3)
lp = prof.load_p.copy(); lp[60:460] *= 3000.0 if name == "case322" else 60.0
prof = ProfileDesc(pv=prof.pv, load_p=lp, load_q=prof.load_q, steps_per_hour=prof.steps_per_hour, n_days=prof.n_days)
scale = cases.SCENARIOS[name]["action_scale"]
env = emu_env.make_env(net, prof, dict(seed=3, voltage_barrier_type="bowl", action_scale=scale, episode_limit=3, history=H),
                       batch=B, lanes_per_env=lanes)
env.reset()
start = torch.tensor([[1, 5, 3]] * B, dtype=torch.int32); start[1] = torch.tensor((0, 2, 18))
env.reset(start, mask=torch.from_numpy((np.arange(B) %% 2).astype(np.uint8)))
d = env.dims
rng = np.random.default_rng(0)
for t in range(5):
    env.step_autoreset(torch.from_numpy(rng.uniform(-scale, scale, (B, net.n_sgen))))
rounds = -(-(-(-B // d["envs_per_block"])) // emu_env.last_grid())
print("ran", name, lanes, B, "rounds", rounds)
'''


def main():
    os.makedirs(OUT, exist_ok=True)
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-pthread", "-fsanitize=thread", "-DMAPDN_HOST_EMU",
                    "-DMAPDN_EMU_DEFINE_GLOBALS", "-I", os.path.join(ROOT, "tests", "emu"), "-x", "c++",
                    os.path.join(ROOT, "mapdn_b200", "csrc", "mapdn_b200.cu"), "-o", LIB], check=True, stderr=subprocess.DEVNULL)
    tsan = subprocess.run(["g++", "-print-file-name=libtsan.so"], capture_output=True, text=True).stdout.strip()
    child = os.path.join(OUT, "child.py")
    open(child, "w").write(CHILD % dict(root=ROOT, lib=LIB))
    child_ar = os.path.join(OUT, "child_autoreset.py")
    open(child_ar, "w").write(CHILD_AR % dict(root=ROOT, lib=LIB))
    env = dict(os.environ, LD_PRELOAD=os.path.realpath(tsan), TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0 exitcode=0")
    total = 0
    for cfg in (("case33", "8", "9"), ("case33", "4", "5"), ("case33", "64", "2"), ("case141", "32", "3"), ("case322", "64", "2")):
        res = subprocess.run([sys.executable, child, *cfg], env=env, capture_output=True, text=True)
        n = res.stderr.count("WARNING: ThreadSanitizer")
        total += n
        ok = "ran" in res.stdout
        print(f"{cfg[0]} lanes/env={cfg[1]} B={cfg[2]} (reset, 2 steps, compact host step, solve, droop): "
              f"{'completed' if ok else 'FAILED'}, ThreadSanitizer reports: {n}")
        if n:
            sys.stderr.write(res.stderr[:6000])
    # (net, lanes per env, batch, history, envs per CTA): one CTA per SM of the emulated one-SM device, >= 2 rounds
    for name, lanes, B, H, epb in (("case33", 4, 37, 3, 32), ("case33", 8, 23, 1, 20), ("case141", 32, 7, 3, 3),
                                   ("case322", 64, 5, 1, 2)):
        ar_env = dict(env, MAPDN_EMU_SMS="1", MAPDN_EPB=str(epb))
        res = subprocess.run([sys.executable, child_ar, name, str(lanes), str(B), str(H)], env=ar_env, capture_output=True,
                             text=True)
        n = res.stderr.count("WARNING: ThreadSanitizer")
        total += n
        ok = "ran" in res.stdout
        print(f"{name} lanes/env={lanes} B={B} history={H} (auto-reset, 5 steps, mixed termination, "
              f"{res.stdout.split()[-1] if ok else '?'} rounds): {'completed' if ok else 'FAILED'}, ThreadSanitizer reports: {n}")
        if n or not ok:
            sys.stderr.write(res.stderr[:6000])
    return 1 if total else 0


if __name__ == "__main__":
    sys.exit(main())
