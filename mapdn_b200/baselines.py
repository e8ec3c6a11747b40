"""Traditional-control baselines on the batched GPU power flow (SURVEY §8 f4).

Restates reference ``traditional_control/pf_droop_matpower_all.m`` without MATLAB/MATPOWER:

* ``no_control``    - power flow with q = 0 (script lines :107-119);
* ``droop_control`` - the relaxed fixed-point loop of lines :121-152 with the piece-wise linear
  ``q(v)`` characteristic of lines :196-231 (saturation below 0.95 / above 1.05 p.u., dead band
  collapsed at 1.0, ``q_max = min(sqrt(S_rated^2 - p^2), q_max_manual)``), relaxation ``gain`` 0.1,
  at most 100 power flows per control instant, stop when ||dv_pv||_2 < 1e-4.

``droop_control`` is ONE kernel launch per control instant (``mapdn_droop``: the whole relaxed loop, the
characteristic and the per-env early exit run inside the fused env kernel, no host synchronisation).
``droop_control_host_loop`` is the round-1 formulation - one ``mapdn_solve`` launch plus a handful of PyTorch
kernels and a host sync per iteration - kept as the cross-check / timing baseline (``scripts/droop_timing.py``).
OPF (``opf_matpower_all.m``) needs an interior-point solver and stays out of scope.
"""
from __future__ import annotations

import torch

import ctypes as C

__all__ = ["droop_characteristic", "no_control", "droop_control", "droop_control_host_loop"]


def droop_characteristic(p, s_rated, v, q_max_manual, va=0.95, vb=1.0, vc=1.0, vd=1.05):
    """Vectorised ``droop_control`` of the reference script (:196-231). All tensors broadcastable."""
    q_max = torch.minimum(torch.sqrt(s_rated ** 2 - p ** 2), q_max_manual)
    k_low = q_max / (va - vb)                  # (q_max - 0) / (va - vb)
    k_high = -q_max / (vc - vd)                # (0 - q_max) / (vc - vd)
    q = torch.zeros_like(v)
    q = torch.where(v < vb, k_low * (v - vb), q)
    q = torch.where(v > vc, k_high * (vc - v), q)
    q = torch.where(v <= va, q_max, q)
    q = torch.where(v > vd, -q_max, q)
    return q


def _loss(out, p_load, p_pv):
    # reference: loss = sum(gen P) - sum(bus Pd) = slack infeed + PV - load
    return out["pl"].sum(dim=1)


def no_control(env, p_load, q_load, p_pv):
    """Power flow without reactive support. Returns dict(vm, q, loss, converged)."""
    q0 = torch.zeros_like(p_pv)
    out = env.solve(p_load, q_load, p_pv, q0)
    return dict(vm=out["vm"], q=q0, loss=_loss(out, p_load, p_pv), converged=out["converged"])


def droop_control(env, p_load, q_load, p_pv, s_rated, q_max_manual=None, max_ite=100, gain=0.1, tol=1e-4):
    """Batched droop control, one launch. ``p_load/q_load [B, n_load]``, ``p_pv [B, n_sgen]`` fp64 on ``env.device``;
    ``s_rated [n_sgen]`` (= 1.2 * max PV in the reference). Returns dict(vm, q, loss, iterations) where ``q`` is the
    reactive power of the last power flow (``result.gen(:,3)`` in the script) and ``iterations`` the number of power
    flows run per env."""
    from . import _capi
    dev = env.device
    t = lambda x: torch.as_tensor(x, dtype=torch.float64, device=dev).contiguous()
    p_load, q_load, p_pv, s_rated = t(p_load), t(q_load), t(p_pv), t(s_rated)
    q_max_manual = s_rated if q_max_manual is None else t(q_max_manual)
    B, d = int(p_pv.shape[0]), env.dims
    if tuple(p_load.shape) != (B, d["n_load"]) or tuple(p_pv.shape) != (B, d["n_sgen"]) or s_rated.numel() != d["n_sgen"]:
        raise ValueError("droop_control: shape mismatch")
    vm = torch.empty(B, d["n_bus"], dtype=torch.float64, device=dev)
    q = torch.empty(B, d["n_sgen"], dtype=torch.float64, device=dev)
    loss = torch.empty(B, dtype=torch.float64, device=dev)
    iters = torch.empty(B, dtype=torch.int32, device=dev)
    ptr = lambda x: C.c_void_p(x.data_ptr())
    _capi.check(env._L.mapdn_droop(env._h, B, ptr(p_load), ptr(q_load), ptr(p_pv), ptr(s_rated), ptr(q_max_manual),
                                   float(gain), float(tol), int(max_ite), ptr(vm), ptr(q), ptr(loss), ptr(iters),
                                   env._stream()), env._L)
    return dict(vm=vm, q=q, loss=loss, iterations=iters)


def droop_control_host_loop(env, p_load, q_load, p_pv, s_rated, q_max_manual=None, max_ite=100, gain=0.1, tol=1e-4):
    """The same loop driven from the host: one ``mapdn_solve`` launch + elementwise PyTorch kernels + one host sync per
    iteration (cross-check of ``droop_control``; envs that met the stopping rule keep their q)."""
    dev = env.device
    p_load = torch.as_tensor(p_load, dtype=torch.float64, device=dev)
    q_load = torch.as_tensor(q_load, dtype=torch.float64, device=dev)
    p_pv = torch.as_tensor(p_pv, dtype=torch.float64, device=dev)
    s_rated = torch.as_tensor(s_rated, dtype=torch.float64, device=dev)
    q_max_manual = s_rated if q_max_manual is None else torch.as_tensor(q_max_manual, dtype=torch.float64, device=dev)
    pv_bus = torch.as_tensor(env.net.sgen_bus, dtype=torch.long, device=dev)
    B = p_pv.shape[0]
    q_last = torch.zeros_like(p_pv)
    v_last = torch.full_like(p_pv, 100.0)
    active = torch.ones(B, dtype=torch.bool, device=dev)
    iters = torch.zeros(B, dtype=torch.int32, device=dev)
    vm = loss = None
    for i in range(max_ite):
        out = env.solve(p_load, q_load, p_pv, q_last)
        v_pv = out["vm"][:, pv_bus]
        new_vm, new_loss = out["vm"], _loss(out, p_load, p_pv)
        vm = new_vm if vm is None else torch.where(active[:, None], new_vm, vm)
        loss = new_loss if loss is None else torch.where(active, new_loss, loss)
        iters = torch.where(active, torch.full_like(iters, i + 1), iters)
        done = torch.linalg.vector_norm(v_last - v_pv, dim=1) < tol
        active = active & ~done
        if not bool(active.any()):
            break
        v_last = torch.where(active[:, None], v_pv, v_last)
        q_new = droop_characteristic(p_pv, s_rated, v_pv, q_max_manual)
        q_last = torch.where(active[:, None], (1 - gain) * q_last + gain * q_new, q_last)
    return dict(vm=vm, q=q_last, loss=loss, iterations=iters)
