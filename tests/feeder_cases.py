"""Generated feeders for the power-flow sweep tests (tests/test_feeder_sweep_emu.py on the CPU emulation,
tests/test_feeder_sweep_gpu.py on the H100): seeded, deterministic ``NetDesc`` builders whose shapes and numerics are
where the tree solve's schedules and its fp64 arithmetic can go wrong.

A topology is a parent list over abstract nodes, node 0 the slack (``parent[0] = -1``). ``feeder`` shuffles the bus ids
(the slack is never bus 0), flips branch directions at random and gives the branches electrical data:

* R/X from 0.1 to 10, series impedances spread over ``decades`` decades within the net;
* off-nominal taps within +-5 % on about a sixth of the branches, at most eight (transformers: not in ``res_line``), and with ``shift`` phase
  shifters within +-10 degrees on those and up to four more branches, which makes Ybus asymmetric;
* line charging, bus shunts, a parallel twin and two out-of-service branches, one of them closing a loop.

``loadings`` places a batch of load patterns on a net: every env a different multiple of one injection pattern, from
zero injection through reverse flow and light load to the nose of the PV curve (where Newton needs 6 to 10 iterations)
and beyond it (no solution: not converged after max_it)."""
import dataclasses
import re

import numpy as np

from mapdn_b200.network import NetDesc
from oracle.mp_newton import MpNewton
from oracle.pandapower_nr import PandapowerEquivalent

LANES = (0, 4, 8, 16, 32, 64, 128)
TOL_NR = 1e-8              # the Newton tolerance of both sides (runpp default)
V_ABS = 1e-9               # |V - V_mp|inf, p.u.
C_ORACLE = 10.0            # kernel error <= C_ORACLE x fp64 oracle error + V_FLOOR; on the CPU tier's 1141 converged
V_FLOOR = 1e-12            # cases the kernel's largest error was 9.8e-13 and the oracle's 5.0e-13
P_TOL = 1e-8               # p_bus / q_bus, MW / MVAr (as tests/test_emu_kernel.py)
PL_TOL = 1e-9              # line losses, MW
P_REL = 1e-12              # plus this much of the largest bus power / line loss of the env

# ---- topologies: parent lists, node 0 = slack ----


def random_tree(n, rng):
    """Uniform random recursive tree of n nodes: node k hangs off a uniformly chosen earlier node."""
    return [-1] + [int(rng.integers(0, k)) for k in range(1, n)]


def chain(n):
    return [-1] + list(range(n - 1))


def caterpillar(spine, rng, max_legs=3):
    """A chain of ``spine`` buses behind the slack, each with 0..max_legs leaves."""
    par = chain(spine + 1)
    for s in range(1, spine + 1):
        par += [s] * int(rng.integers(0, max_legs + 1))
    return par


def broom(handle, bristles):
    """A chain of ``handle`` buses behind the slack, ending in a star of ``bristles`` leaves."""
    return chain(handle + 1) + [handle] * bristles


def complete_tree(arity, depth):
    """A complete ``arity``-ary tree of the given depth whose root hangs off the slack."""
    par, level = [-1, 0], [1]
    for _ in range(depth):
        nxt = []
        for p in level:
            for _ in range(arity):
                nxt.append(len(par))
                par.append(p)
        level = nxt
    return par


def levels(widths, rng):
    """A tree with ``widths[l]`` buses at depth l + 1 below one root bus next to the slack. Where a level is not narrower
    than the one above it, every bus of the level above gets a child, so the height levels of the forward sweep are the
    depth levels reversed: the prescribed widths reach both sweeps."""
    par, above = [-1, 0], [1]
    for w in widths:
        here = list(range(len(par), len(par) + w))
        for k, _ in enumerate(here):
            par.append(above[k] if k < len(above) else above[int(rng.integers(0, len(above)))])
        above = here
    return par


def star(k):
    """k buses next to the slack: a forest of single-bus trees."""
    return [-1] + [0] * k


def hub(k, tail=2):
    """The slack, one hub bus with k children, and chains of ``tail`` buses below two of them: the hub stays the centre
    its tree is re-rooted at, so it keeps all k children."""
    par = [-1, 0] + [1] * k
    for first in (2, 3)[:min(k, 2)]:
        prev = first
        for _ in range(tail):
            par.append(prev)
            prev = len(par) - 1
    return par


def forest(n_roots, n, rng):
    """``n_roots`` random trees next to the slack, n buses in all."""
    par = [-1] + [0] * n_roots
    for k in range(n_roots + 1, n):
        par.append(int(rng.integers(1, k)))
    return par


# ---- electrical data ----

def feeder(par, seed, shift=False, decades=1.0, name="feeder", extra_lines=0):
    """A NetDesc on the topology ``par``. ``extra_lines`` loop-closing lines make it meshed (the dense fallback)."""
    rng = np.random.default_rng(seed)
    n = len(par)
    perm = rng.permutation(n)
    if perm[0] == 0:                                         # the slack is never bus 0
        perm[[0, 1]] = perm[[1, 0]]
    f = np.array([perm[par[k]] for k in range(1, n)])
    t = perm[1:].copy()
    while f.size < n - 1 + extra_lines:
        a, b = rng.choice(np.arange(1, n), 2, replace=False)
        if par[a] != b and par[b] != a:                      # closes a loop, not a parallel pair
            f, t = np.r_[f, perm[a]], np.r_[t, perm[b]]
    nbr = f.size
    flip = rng.random(nbr) < 0.5
    f, t = np.where(flip, t, f), np.where(flip, f, t)
    # impedances, charging, shunts and taps add up along a feeder: a few hundred buses at the per-bus values of a small
    # net have no power-flow solution even without load, so large nets get proportionally less of each
    small = min(1.0, 40.0 / n)
    zmag = small * 10.0 ** rng.uniform(-2.5, -2.5 + decades, nbr)
    ratio = 10.0 ** rng.uniform(-1.0, 1.0, nbr)              # R/X
    x = zmag / np.sqrt(1.0 + ratio ** 2)
    r = ratio * x
    b = rng.uniform(0.0, 2e-3 * small, nbr)
    g = rng.uniform(0.0, 1e-4 * small, nbr)
    tap = np.ones(nbr)
    sh = np.zeros(nbr)
    is_line = np.ones(nbr, np.uint8)
    k = rng.choice(nbr, max(1, min(nbr // 6, 8)), replace=False)
    tap[k] = 1.0 + small * rng.uniform(-0.05, 0.05, k.size)
    is_line[k] = 0
    if shift:
        ks = np.union1d(k, rng.choice(nbr, min(4, nbr), replace=False))
        sh[ks] = rng.uniform(-10.0, 10.0, ks.size)
    # a parallel twin of branch 0, an out-of-service copy of branch 1 and, when the net has room, an out-of-service
    # line closing a loop: neither of the last two may change the topology
    f, t = np.r_[f, f[0], f[1]], np.r_[t, t[0], t[1]]
    r, x = np.r_[r, 1.3 * r[0], r[1]], np.r_[x, 0.9 * x[0], x[1]]
    b, g = np.r_[b, 0.0, 0.0], np.r_[g, 0.0, 0.0]
    tap, sh = np.r_[tap, tap[0], 1.0], np.r_[sh, sh[0], 0.0]
    is_line = np.r_[is_line, is_line[0], 1]
    status = np.ones(f.size, np.uint8)
    status[-1] = 0
    if n > 3:
        a, c = rng.choice(np.arange(1, n), 2, replace=False)
        f, t = np.r_[f, perm[a]], np.r_[t, perm[c]]
        r, x, b, g = np.r_[r, r[0]], np.r_[x, x[0]], np.r_[b, 0.0], np.r_[g, 0.0]
        tap, sh, is_line, status = np.r_[tap, 1.0], np.r_[sh, 0.0], np.r_[is_line, 1], np.r_[status, 0]
    n_sgen = int(min(n - 1, 2 + rng.integers(0, 3)))
    zone = rng.integers(0, 4, n).astype(np.int32)
    sgen_bus = rng.choice(perm[1:], n_sgen, replace=False).astype(np.int32)
    zone[sgen_bus] = np.maximum(zone[sgen_bus], 1)
    load_bus = np.r_[perm[1:], rng.choice(perm[1:], 3)].astype(np.int32)
    return NetDesc(base_mva=10.0, n_bus=n, slack_bus=int(perm[0]), slack_vm=1.02, slack_va_deg=float(rng.uniform(-5, 5)),
                   vm_init=float(rng.choice([1.0, 1.02])), br_from=f, br_to=t, br_r=r, br_x=x, br_b=b, br_g=g, br_tap=tap,
                   br_shift=sh, br_status=status, br_is_line=is_line.astype(np.uint8),
                   bus_gs=rng.uniform(0.0, 0.05 * small, n), bus_bs=rng.uniform(-0.05 * small, 0.05 * small, n), load_bus=load_bus,
                   load_scaling=rng.uniform(0.8, 1.2, load_bus.size), sgen_bus=sgen_bus, sgen_zone=zone[sgen_bus],
                   sgen_scaling=rng.uniform(0.9, 1.1, n_sgen), bus_zone=zone, name=name)


def without_shift(net):
    return dataclasses.replace(net, br_shift=np.zeros_like(net.br_shift), name=net.name + "_noshift")


# ---- loadings ----

# multiples of the nose loading, one per env: zero injection, reverse flow, light to heavy load, the nose, beyond it
LOADINGS = (0.0, -0.4, 0.6, 0.97, 0.995, 1.05)


def _pattern(net, seed):
    """One injection pattern (MW / MVAr): loads with mixed power factors, sgens at a tenth of the mean load."""
    rng = np.random.default_rng(seed + 7919)
    pl = rng.uniform(0.0, 1.0, net.n_load)
    ql = pl * rng.uniform(-0.2, 0.6, net.n_load)
    ps = np.full(net.n_sgen, 0.1 * pl.mean())
    qs = ps * rng.uniform(-0.3, 0.3, net.n_sgen)
    return pl, ql, ps, qs


def nose(net, seed, pf=None):
    """The largest multiple of the pattern the fp64 oracle still solves within max_it (to 1e-3 relative)."""
    pf = pf or PandapowerEquivalent(net)
    pat = _pattern(net, seed)

    def ok(lam):
        return pf.runpp(*(lam * a for a in pat)).converged
    lo, hi = 0.0, 1.0
    while ok(hi):
        lo, hi = hi, 2.0 * hi
    while hi - lo > 1e-3 * hi:
        mid = 0.5 * (lo + hi)
        lo, hi = (mid, hi) if ok(mid) else (lo, mid)
    return lo


def loadings(net, seed, fractions=LOADINGS, pf=None):
    """(p_load, q_load, p_sgen, q_sgen) [B, ...] with env k at fractions[k] x the nose loading."""
    pat = _pattern(net, seed)
    lam = nose(net, seed, pf) * np.asarray(fractions)
    return tuple(lam[:, None] * a[None] for a in pat)


# ---- the catalogue ----

def catalogue(tier="emu"):
    """{name: NetDesc}: every family, with and without phase shifters. The GPU tier adds seeds and larger nets."""
    rng = np.random.default_rng(2024)
    tops = {
        "random40": random_tree(40, rng),
        "caterpillar": caterpillar(14, rng),
        "broom": broom(12, 10),
        "binary4": complete_tree(2, 4),
        "ternary3": complete_tree(3, 3),
        "chain48": chain(48),
        "levels_g4_g8": levels([2, 3, 4, 5, 7, 8, 9], rng),
        "levels_g16": levels([2, 15, 16, 17], rng),
        "levels_g32": levels([2, 31, 32, 33], rng),
        "levels_mixed": levels([2, 9, 8, 12, 3, 17, 1], rng),
        "star4": star(4),
        "hub3": hub(3),
        "hub4": hub(4),
        "hub255": hub(255),
        "hub257": hub(257),
        "forest1": forest(1, 30, rng),
        "forest2": forest(2, 30, rng),
        "forest12": forest(12, 40, rng),
    }
    if tier == "gpu":
        tops.update({
            "random200": random_tree(200, rng),
            "caterpillar60": caterpillar(60, rng),
            "levels_g64": levels([2, 31, 32, 33, 63, 64, 65], rng),
            "levels_g128": levels([2, 32, 33, 127, 128, 129], rng),
            "levels_probe": levels([2, 65, 64, 70, 3, 129, 1], rng),
            "star250": star(250),
            "forest40": forest(40, 200, rng),
            "chain300": chain(300),
        })
    nets = {}
    for k, (name, par) in enumerate(sorted(tops.items())):
        net = feeder(par, seed=100 + k, shift=True, name=name)
        if name not in ("chain300", "caterpillar60"):    # a dozen shifters in series: beyond a flat start's reach
            nets[name] = net
        if len(par) < 200 or tier == "gpu":
            nets[name + "_noshift"] = without_shift(net)
    nets["decades4"] = feeder(random_tree(36, rng), seed=7, shift=True, decades=4.0, name="decades4")
    nets["decades4_noshift"] = without_shift(nets["decades4"])
    return nets


def meshed_catalogue():
    """Small meshed variants for the dense fallback."""
    rng = np.random.default_rng(77)
    return {"mesh_random12": feeder(random_tree(12, rng), seed=3, shift=True, extra_lines=1, name="mesh_random12"),
            "mesh_caterpillar": feeder(caterpillar(6, rng), seed=4, shift=True, extra_lines=2, name="mesh_caterpillar")}


# ---- the comparisons both tiers make ----

def check_env(out, k, r_mp, r_or, where):
    """Env k of a solve (``out``: NumPy arrays) against the mp reference ``r_mp``: same converged flag and iteration
    count; when converged |V - V_mp| <= V_ABS and at most C_ORACLE x the fp64 oracle's own error (``r_or``) + V_FLOOR,
    bus powers and line losses at the usual tolerances plus P_REL of their magnitude. The caller has dropped ambiguous envs. Returns the kernel's and
    the oracle's |V - V_mp| (0 when not converged)."""
    assert bool(out["converged"][k]) == r_mp.converged and int(out["iterations"][k]) == r_mp.iterations, \
        (where, int(out["iterations"][k]), r_mp.iterations, r_mp.norms)
    if not r_mp.converged:
        return 0.0, 0.0
    Vm = MpNewton.complex_V(r_mp)
    e_k = float(np.abs(out["vm"][k] * np.exp(1j * np.deg2rad(out["va_deg"][k])) - Vm).max())
    e_o = float(np.abs(r_or.V - Vm).max())
    assert e_k <= V_ABS and e_k <= C_ORACLE * e_o + V_FLOOR, (where, e_k, e_o)
    for key, want, tol in (("p_bus", r_mp.p_mw, P_TOL), ("q_bus", r_mp.q_mvar, P_TOL), ("pl", r_mp.pl_mw, PL_TOL)):
        # near the nose of a stiff net the powers reach 1e4 MW: fp64 sums carry 1e-12 of that
        assert np.abs(out[key][k] - want).max() < tol + P_REL * np.abs(want).max(initial=0.0), (where, key)
    return e_k, e_o


def refusal_bytes(msg):
    """(bytes needed, at lanes per env, bytes available) of a shared-memory refusal of mapdn_create."""
    got = re.search(r"\((\d+) B needed at (\d+) lanes per env, (\d+) B available\)", msg)
    assert got, msg
    return [int(x) for x in got.groups()]
