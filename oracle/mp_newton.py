"""ORACLE - TEST INFRASTRUCTURE ONLY. pandapower's ``newtonpf`` (the restatement in ``oracle/pandapower_nr.py``) in
extended precision with ``mpmath``: the yardstick two fp64 implementations of the same Newton iteration are measured
against when they drift apart (loading near the nose of the PV curve, impedances over several decades, phase shifters).

Every step is the fp64 oracle's, computed at ``dps`` decimal digits from the exact values of the fp64 inputs:

* Ybus with the formulas of ``make_ybus`` (taps, phase shift, charging, bus shunts; out-of-service branches dropped);
* the same flat start (``vm_init``, slack magnitude and angle), the same mismatch test ``||F||inf < tol`` before every
  solve, the same ``max_it``;
* an exact linear solve of the polar Jacobian: on a radial net the PQ buses form a forest and the 2x2-block
  elimination along it (leaves first) has no fill, so it is linear in the number of buses; a meshed net is solved densely
  with ``mp.lu_solve`` (small nets only).

``run`` returns every iterate, the mismatch norm at each iterate, the iteration count, the converged flag, and from the
final iterate the bus powers and line losses as ``PandapowerEquivalent.runpp`` reports them.
"""
from __future__ import annotations

import mpmath
import numpy as np

from oracle.pandapower_nr import MAX_IT_DEFAULT, TOL_DEFAULT

mp = mpmath.mp


class MpResult:
    __slots__ = ("converged", "iterations", "iterates", "norms", "V", "vm_pu", "va_degree", "p_mw", "q_mvar", "pl_mw")

    def ambiguous(self, tol, rel=1e-6):
        """True when a convergence test this run decided lies within ``rel`` (relative) of ``tol``: there two correct
        fp64 implementations may stop at different iterations."""
        return any(abs(nm / tol - 1) <= rel for nm in self.norms)


class MpNewton:
    """Extended-precision ``PandapowerEquivalent``: ``MpNewton(net).run(p_load, q_load, p_sgen, q_sgen)``."""

    def __init__(self, net, tol=TOL_DEFAULT, max_it=MAX_IT_DEFAULT, dps=40):
        self.net, self.tol, self.max_it, self.dps = net, tol, max_it, dps
        self.ref = int(net.slack_bus)
        self.pq = [b for b in range(net.n_bus) if b != self.ref]
        with mp.workdps(dps):
            self._make_ybus()
            self._plan_solve()

    # ---- makeYbus ----
    def _make_ybus(self):
        net = self.net
        nb = net.n_bus
        Y = [dict() for _ in range(nb)]
        self.branch_y = []                      # per branch: (Yff, Yft, Ytf, Ytt), zeros when out of service
        j = mpmath.mpc(0, 1)
        for k in range(len(net.br_from)):
            f, t = int(net.br_from[k]), int(net.br_to[k])
            if not net.br_status[k]:
                self.branch_y.append((0, 0, 0, 0))
                continue
            Ys = 1 / mpmath.mpc(float(net.br_r[k]), float(net.br_x[k]))
            Bc = mpmath.mpc(float(net.br_b[k]), -float(net.br_g[k]))
            tap = float(net.br_tap[k]) or 1.0
            tap = mpmath.mpf(tap) * mpmath.expjpi(mpmath.mpf(float(net.br_shift[k])) / 180) if net.br_shift[k] else mpmath.mpc(tap)
            Ytt = Ys + j * Bc / 2
            Yff = Ytt / (tap * mpmath.conj(tap))
            Yft = -Ys / mpmath.conj(tap)
            Ytf = -Ys / tap
            self.branch_y.append((Yff, Yft, Ytf, Ytt))
            for a, b, v in ((f, f, Yff), (f, t, Yft), (t, f, Ytf), (t, t, Ytt)):
                Y[a][b] = Y[a].get(b, 0) + v
        base = mpmath.mpf(float(net.base_mva))
        for b in range(nb):
            if net.bus_gs[b] or net.bus_bs[b]:
                Y[b][b] = Y[b].get(b, 0) + mpmath.mpc(float(net.bus_gs[b]), float(net.bus_bs[b])) / base
        self.Y = Y

    def ybus_dense(self):
        """Ybus rounded to complex128 (for comparisons with fp64 assemblies)."""
        nb = self.net.n_bus
        out = np.zeros((nb, nb), np.complex128)
        for a in range(nb):
            for b, v in self.Y[a].items():
                out[a, b] = complex(v)
        return out

    # ---- the linear solve: elimination forest of the PQ buses, or dense ----
    def _plan_solve(self):
        nb, ref = self.net.n_bus, self.ref
        adj = [[b for b in self.Y[a] if b != a] for a in range(nb)]
        n_edges = sum(len(a) for a in adj) // 2
        self.radial = n_edges == nb - 1
        if not self.radial:
            return
        parent, order, seen = {}, [], [False] * nb
        seen[ref] = True
        for r in adj[ref]:                      # one tree of PQ buses per slack neighbour
            if seen[r]:
                continue
            seen[r] = True
            parent[r] = -1
            q = [r]
            for u in q:
                for v in adj[u]:
                    if not seen[v]:
                        seen[v] = True
                        parent[v] = u
                        q.append(v)
            order += q
        self.parent, self.order = parent, order     # parents before children

    # ---- newtonpf ----
    def _mismatch(self, V, S):
        I = [sum((y * V[b] for b, y in row.items()), mpmath.mpc(0)) for row in self.Y]
        mis = {i: V[i] * mpmath.conj(I[i]) - S[i] for i in self.pq}
        norm = max((max(abs(m.real), abs(m.imag)) for m in mis.values()), default=mpmath.mpf(0))
        return I, mis, norm

    def _blocks(self, V, I):
        """J[i,k] as 2x2 real blocks ((dP/dVa, dP/dVm), (dQ/dVa, dQ/dVm)) of dSbus_dV, PQ rows and columns."""
        j = mpmath.mpc(0, 1)
        J = {}
        for i in self.pq:
            for k, y in self.Y[i].items():
                if k == self.ref:
                    continue
                if k == i:
                    dvm = V[i] * mpmath.conj(y * V[i] / abs(V[i])) + mpmath.conj(I[i]) * V[i] / abs(V[i])
                    dva = j * V[i] * mpmath.conj(I[i] - y * V[i])
                else:
                    dvm = V[i] * mpmath.conj(y * V[k] / abs(V[k]))
                    dva = -j * V[i] * mpmath.conj(y * V[k])
                J[i, k] = ((dva.real, dvm.real), (dva.imag, dvm.imag))
        return J

    def _solve(self, J, F):
        """x with J x = F; F, x: {bus: (p, q)}."""
        if not self.radial:
            idx = {b: k for k, b in enumerate(self.pq)}
            m = len(self.pq)
            A = mpmath.matrix(2 * m, 2 * m)
            rhs = mpmath.matrix(2 * m, 1)
            for (i, k), blk in J.items():
                for r in range(2):
                    for c in range(2):
                        A[2 * idx[i] + r, 2 * idx[k] + c] = blk[r][c]
            for b in self.pq:
                rhs[2 * idx[b]], rhs[2 * idx[b] + 1] = F[b]
            x = mpmath.lu_solve(A, rhs)
            return {b: (x[2 * idx[b]], x[2 * idx[b] + 1]) for b in self.pq}

        def mul(a, b):
            return ((a[0][0] * b[0][0] + a[0][1] * b[1][0], a[0][0] * b[0][1] + a[0][1] * b[1][1]),
                    (a[1][0] * b[0][0] + a[1][1] * b[1][0], a[1][0] * b[0][1] + a[1][1] * b[1][1]))

        def mulv(a, v):
            return (a[0][0] * v[0] + a[0][1] * v[1], a[1][0] * v[0] + a[1][1] * v[1])

        def inv(a):
            d = a[0][0] * a[1][1] - a[0][1] * a[1][0]
            return ((a[1][1] / d, -a[0][1] / d), (-a[1][0] / d, a[0][0] / d))

        D = {b: J[b, b] for b in self.pq}
        r = dict(F)
        Dinv = {}
        for i in reversed(self.order):          # leaves first: fold each bus into its parent
            Dinv[i] = inv(D[i])
            p = self.parent[i]
            if p < 0:
                continue
            L = mul(J[p, i], Dinv[i])
            U = mul(L, J[i, p])
            D[p] = tuple(tuple(D[p][a][c] - U[a][c] for c in range(2)) for a in range(2))
            Lr = mulv(L, r[i])
            r[p] = (r[p][0] - Lr[0], r[p][1] - Lr[1])
        x = {}
        for i in self.order:                    # roots first
            p = self.parent[i]
            v = r[i]
            if p >= 0:
                u = mulv(J[i, p], x[p])
                v = (v[0] - u[0], v[1] - u[1])
            x[i] = mulv(Dinv[i], v)
        return x

    def run(self, p_load, q_load, p_sgen, q_sgen) -> MpResult:
        with mp.workdps(self.dps):
            return self._run(p_load, q_load, p_sgen, q_sgen)

    def _run(self, p_load, q_load, p_sgen, q_sgen):
        net = self.net
        nb = net.n_bus
        mpf = mpmath.mpf
        PD, QD = [mpf(0)] * nb, [mpf(0)] * nb
        for k, b in enumerate(net.load_bus):
            PD[b] += mpf(float(p_load[k])) * mpf(float(net.load_scaling[k]))
            QD[b] += mpf(float(q_load[k])) * mpf(float(net.load_scaling[k]))
        for k, b in enumerate(net.sgen_bus):
            PD[b] -= mpf(float(p_sgen[k])) * mpf(float(net.sgen_scaling[k]))
            QD[b] -= mpf(float(q_sgen[k])) * mpf(float(net.sgen_scaling[k]))
        base = mpf(float(net.base_mva))
        S = [-mpmath.mpc(PD[b], QD[b]) / base for b in range(nb)]
        V = [mpmath.mpc(float(net.vm_init))] * nb
        V[self.ref] = mpf(float(net.slack_vm)) * mpmath.expjpi(mpf(float(net.slack_va_deg)) / 180)
        tol = mpf(self.tol)
        res = MpResult()
        res.iterates, res.norms = [list(V)], []
        I, mis, norm = self._mismatch(V, S)
        res.norms.append(float(norm))
        converged, i = norm < tol, 0
        while not converged and i < self.max_it:
            i += 1
            J = self._blocks(V, I)
            x = self._solve(J, {b: (mis[b].real, mis[b].imag) for b in self.pq})
            V = list(V)
            for b in self.pq:                   # Va += dx, Vm += dx with dx = -x
                vm, va = abs(V[b]) - x[b][1], mpmath.arg(V[b]) - x[b][0]
                V[b] = vm * mpmath.expj(va)
            res.iterates.append(V)
            I, mis, norm = self._mismatch(V, S)
            res.norms.append(float(norm))
            converged = norm < tol
        res.converged, res.iterations, res.V = bool(converged), i, V
        res.vm_pu = np.array([float(abs(v)) for v in V])
        res.va_degree = np.array([float(mpmath.arg(v) * 180 / mp.pi) for v in V])
        # pfsoln + results_bus, as PandapowerEquivalent.runpp
        p, q = list(PD), list(QD)
        Sref = V[self.ref] * mpmath.conj(I[self.ref]) * base
        p[self.ref], q[self.ref] = -Sref.real, -Sref.imag
        for b in range(nb):
            vm2 = abs(V[b]) ** 2
            p[b] += mpf(float(net.bus_gs[b])) * vm2
            q[b] -= mpf(float(net.bus_bs[b])) * vm2
        res.p_mw, res.q_mvar = np.array([float(v) for v in p]), np.array([float(v) for v in q])
        pl = []
        for k in range(len(net.br_from)):
            if not net.br_is_line[k]:
                continue
            Yff, Yft, Ytf, Ytt = self.branch_y[k]
            vf, vt = V[int(net.br_from[k])], V[int(net.br_to[k])]
            sft = vf * mpmath.conj(Yff * vf + Yft * vt) + vt * mpmath.conj(Ytf * vf + Ytt * vt)
            pl.append(float(mpmath.re(sft) * base))
        res.pl_mw = np.array(pl)
        return res

    @staticmethod
    def complex_V(res):
        return np.array([complex(v) for v in res.V])
