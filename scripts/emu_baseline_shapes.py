"""The BASELINE.json launch shapes (envs per CTA, helper warps, shared-memory plan as chosen by mapdn_create for the full
batch) executed on the CPU SIMT emulation (tests/emu) and checked against the oracle on six envs spread over the batch:
    python scripts/emu_baseline_shapes.py case33 4096 bowl | case141 2048 l1 | case322 1024 l2     (1 - 3 minutes each)"""
import sys, numpy as np, time, torch
import os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests', 'emu'))
from emu_env import make_env
from mapdn_b200 import cases
from oracle.voltage_control_ref import INFO_KEYS, VoltageControlOracle
name, B, barrier = sys.argv[1], int(sys.argv[2]), sys.argv[3]
net, prof = cases.make_case(name), cases.make_profiles(name, n_days=4)
scale = cases.SCENARIOS[name]["action_scale"]
t0=time.time()
env = make_env(net, prof, dict(voltage_barrier_type=barrier, seed=0, action_scale=scale), batch=B)
print("dims", {k: env.dims[k] for k in ("lanes_per_env","envs_per_block","smem_bytes")}, flush=True)
obs, state = [x.numpy() for x in env.reset()]
print("reset done %.0fs"%(time.time()-t0), flush=True)
ids=[0, 27, 28, B//2+3, B-29, B-1]; ors=[VoltageControlOracle(net, prof, env.args, env_id=i) for i in ids]
d=0
for o,i in zip(ors,ids):
    oo,_=o.reset(); d=max(d, np.abs(np.array(oo)-obs[i]).max())
rng=np.random.default_rng(0)
a=rng.uniform(-scale,scale,(B,net.n_sgen)); r,term,info=[x.numpy() for x in env.step(torch.from_numpy(a))]
for o,i in zip(ors,ids):
    ro,to,io=o.step(a[i]); d=max(d, abs(ro-r[i]), max(abs(io[k]-info[i,j]) for j,k in enumerate(INFO_KEYS)), np.abs(np.array(o.get_obs())-obs[i]).max())
    assert to==bool(term[i])
print(name, "B", B, "max diff", d, "time %.0fs"%(time.time()-t0))
assert d < 1e-9
