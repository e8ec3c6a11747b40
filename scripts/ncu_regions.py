"""Sum ncu_lines.py output by kernel region (line ranges found from marker comments in env_kernel.cuh)."""
import re, sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
src = open(os.path.join(ROOT, "mapdn_b200/csrc/env_kernel.cuh")).read().splitlines()
marks = [("helpers(reduce,rcp,barrier,stage)", 1), ("nr:init", None, "flat start (pandapower"), ("nr:edges", None, "per-edge terms of"),
         ("nr:F/diag", None, "mismatch F ="), ("nr:elim", None, "forward elimination"), ("nr:backsub", None, "back substitution by"),
         ("nr:update", None, "update (theta"), ("kernel setup", None, "sgen.q_mvar from an action"),
         ("helper warps", None, "void helper_draw_rows("), ("reset start", None, "long long reset_start("),
         ("prologue", None, "void prologue("), ("droop", None, "relaxed fixed-point loop of pf_droop"),
         ("epi:fallback+slack", None, "void fallback_and_slack("), ("epi:q+nextrow", None, "void effective_q_and_next_row("),
         ("epi:bus results", None, "void bus_results("), ("epi:lines", None, "line losses: res_line"),
         ("epi:explicit", None, "void explicit_outputs("), ("epi:reward/info", None, "reward (reference _calc_reward :612-618"),
         ("epi:reset", None, "void reset_bookkeeping("), ("epi:obs, then history / state calls, ballot", None, "Observations of the new state"),
         ("epi:history", None, "void step_history("), ("epi:state", None, "void write_state("),
         ("kernel: setup, prefetch, round loop, nr call", None, "env_kernel(const __grid_constant__")]
starts = []
for m in marks:
    if m[1] is not None: starts.append((m[1], m[0])); continue
    key = m[2].split("\n")[0]
    ln = next((i + 1 for i, l in enumerate(src) if key in l and (len(m[2].split("\n")) == 1 or "cnt_lo" in src[i + 1])), None)
    if ln: starts.append((ln, m[0]))
starts.sort()
agg = {n: [0, 0] for _, n in starts}
for ln in sys.stdin:
    m = re.match(r"\s*(\d+)\s+(\d+)\s+[\d.]+%\s+inst\s+(\d+)", ln)
    if not m: continue
    L, s, i = int(m.group(1)), int(m.group(2)), int(m.group(3))
    name = [n for st, n in starts if st <= L][-1]
    agg[name][0] += s; agg[name][1] += i
ts = sum(v[0] for v in agg.values()); ti = sum(v[1] for v in agg.values())
for _, n in starts:
    s, i = agg[n]
    print(f"{n:36s} samples {s:5d} {100*s/ts:5.1f}%   inst {100*i/ti:5.1f}%")
