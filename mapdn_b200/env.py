"""Host-side mirror of the reference env API over the C-ABI.

* :class:`BatchedVoltageControl` - B independent env instances resident in HBM, tensor in/out,
  one fused CUDA launch per ``step``.
* :class:`VoltageControl` - drop-in for the reference class of the same name
  (reference ``environments/var_voltage_control/voltage_control_env.py:24``): B = 1, NumPy in/out,
  same method names, argument meaning and return shapes (PyMARL ``MultiAgentEnv`` API,
  reference ``environments/multiagentenv.py``).

There is no CPU fallback: both classes need the CUDA library and a GPU.
"""
from __future__ import annotations

import ctypes as C
from collections import namedtuple
from typing import Optional

import numpy as np
import torch

from . import _capi
from ._capi import INFO_KEYS, MapdnError
from .network import NetDesc, ProfileDesc

__all__ = ["BatchedVoltageControl", "VoltageControl", "ActionSpace", "DEFAULT_ENV_ARGS", "INFO_KEYS"]

# reference args/env_args/var_voltage_control.yaml:3-20
DEFAULT_ENV_ARGS = dict(voltage_barrier_type="l1", voltage_weight=1.0, q_weight=0.1, line_weight=None,
                        dq_dv_weight=None, history=1, pv_scale=1.0, demand_scale=1.0,
                        state_space=["pv", "demand", "reactive", "vm_pu", "va_degree"],
                        v_upper=1.05, v_lower=0.95, episode_limit=240, action_scale=0.8, action_bias=0.0,
                        mode="distributed", reset_action=True, seed=0)


def convert(dictionary):
    return namedtuple('GenericDict', dictionary.keys())(**dictionary)


class ActionSpace(object):
    """reference voltage_control_env.py:18-21"""

    def __init__(self, low, high):
        self.low = low
        self.high = high


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


class BatchedVoltageControl:
    """``batch`` env instances on one GPU. All tensors are fp64 CUDA tensors, row-major ``[B, ...]``.

    ``env_args``: dict with the keys of the reference's ``env_args`` (DEFAULT_ENV_ARGS).
    ``env_id_offset``: global id of env 0 (multi-GPU sharding keeps the RNG streams per env id).
    """

    def __init__(self, net: NetDesc, profiles: Optional[ProfileDesc], env_args: Optional[dict] = None,
                 batch: int = 1, device: Optional[int] = None, env_id_offset: int = 0,
                 lanes_per_env: int = 0, tol: float = 0.0, max_iter: int = 0):
        if not torch.cuda.is_available():
            raise MapdnError("mapdn_b200 needs a CUDA device (there is no CPU fallback)")
        args = dict(DEFAULT_ENV_ARGS)
        args.update(env_args or {})
        if args.get("mode", "distributed") != "distributed":
            # the reference's decentralised mode raises KeyError in get_obs at this commit
            # (voltage_control_env.py:239 indexes clusters["sgen{i}"], absent in that mode)
            raise NotImplementedError("only mode='distributed' is supported (decentralised is broken upstream)")
        self.history = int(args.get("history", 1) or 1)
        unknown = set(args["state_space"]) - set(_capi.STATE_SPACE_BITS)
        if unknown or not args["state_space"]:
            raise ValueError(f"state_space must be a non-empty subset of {sorted(_capi.STATE_SPACE_BITS)}, got {unknown}")
        self.args = args
        self.net, self.profiles = net, profiles
        self.batch = int(batch)
        self.device_index = torch.cuda.current_device() if device is None else int(device)
        self.device = torch.device("cuda", self.device_index)
        L = _capi.lib()
        cfg = _capi.CfgC(
            batch=self.batch, barrier=_capi.BARRIERS[args["voltage_barrier_type"]],
            voltage_weight=float(args["voltage_weight"]),
            q_weight=float(args["q_weight"] if args["q_weight"] is not None else 0.0),
            line_weight=float(args["line_weight"] or 0.0),
            use_line_weight=int(args["line_weight"] is not None),
            v_upper=float(args["v_upper"]), v_lower=float(args["v_lower"]),
            episode_limit=int(args["episode_limit"]),
            action_low=float(-args["action_scale"] + args["action_bias"]),
            action_high=float(args["action_scale"] + args["action_bias"]),
            reset_action=int(bool(args["reset_action"])), seed=int(args["seed"]) & 0xFFFFFFFFFFFFFFFF,
            env_id_offset=int(env_id_offset), tol=float(tol), max_iter=int(max_iter),
            lanes_per_env=int(lanes_per_env),
            state_space_mask=sum(_capi.STATE_SPACE_BITS[k] for k in set(args["state_space"])))
        if args["line_weight"] is None and args["q_weight"] is None:
            raise NotImplementedError("Please at least give one weight, either q_weight or line_weight.")
        nd, keep1 = _capi.make_net_desc(net)
        pd_, keep2 = (None, None) if profiles is None else _capi.make_profile_desc(profiles)
        h = C.c_void_p()
        _capi.check(L.mapdn_create(C.byref(nd), None if pd_ is None else C.byref(pd_), C.byref(cfg),
                                   self.device_index, C.byref(h)))
        del keep1, keep2
        self._h, self._L = h, L
        d = _capi.DimsC()
        _capi.check(L.mapdn_get_dims(h, C.byref(d)))
        self.dims = {k: getattr(d, k) for k, _ in d._fields_}
        self.n_agents, self.n_actions = d.n_agents, d.n_actions
        self.obs_size, self.state_size = d.obs_dim, d.state_dim
        self.episode_limit = int(args["episode_limit"])
        self.action_space = ActionSpace(low=-args["action_scale"] + args["action_bias"],
                                        high=args["action_scale"] + args["action_bias"])
        self.s_max = None if profiles is None else profiles.s_max
        B, f64 = self.batch, torch.float64
        with torch.cuda.device(self.device):
            self.obs = torch.zeros(B, d.n_agents, d.obs_dim, dtype=f64, device=self.device)
            self.state = torch.zeros(B, d.state_dim, dtype=f64, device=self.device)
            self.reward = torch.zeros(B, dtype=f64, device=self.device)
            self.terminated = torch.zeros(B, dtype=torch.uint8, device=self.device)
            self.info = torch.zeros(B, len(INFO_KEYS), dtype=f64, device=self.device)
            self.reset_ok = torch.ones(B, dtype=torch.uint8, device=self.device)
        self._hist = None       # [B, history, n_agents, obs_dim] ring of the last observations (history > 1)
        self._host = None
        # raw pointers of the internal buffers (ctypes converts plain ints for c_void_p parameters): keeps the
        # per-step Python overhead of the hot call small
        self._p_obs, self._p_state = self.obs.data_ptr(), self.state.data_ptr()
        self._p_reward, self._p_term, self._p_info = self.reward.data_ptr(), self.terminated.data_ptr(), self.info.data_ptr()
        self._act_shape = (self.batch, self.n_agents)

    # ------------------------------------------------------------------------------------------
    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            self._L.mapdn_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _chk(self, t: torch.Tensor, shape, dtype=torch.float64, name="tensor"):
        if t.device != self.device or t.dtype != dtype or tuple(t.shape) != tuple(shape) or not t.is_contiguous():
            raise ValueError(f"{name}: expected contiguous {dtype} {tuple(shape)} on {self.device}, got "
                             f"{t.dtype} {tuple(t.shape)} on {t.device}")
        return t

    @property
    def launch_count(self) -> int:
        return int(self._L.mapdn_launch_count(self._h))

    # ---- reset / step -----------------------------------------------------------------------
    def reset(self, start: Optional[torch.Tensor] = None, mask: Optional[torch.Tensor] = None,
              add_noise: bool = True, check: bool = False, max_retries: int = 8, want_state: bool = True):
        """``start``: int32 ``[B,3]`` (day, hour, interval) = ``manual_reset`` per env, or None to
        sample (reference :111-113). ``mask``: uint8 ``[B]`` selecting the envs to reset.
        Returns (obs ``[B,n_agents,obs_dim]``, state ``[B,state_dim]``) - views of internal buffers.

        The reference re-draws an env until its initial power flow converges (:108-133). The device does up to 16
        draws per call and records the outcome in ``self.reset_ok`` (uint8 ``[B]``, stream-ordered, no host sync).
        ``check=True`` reads it back (one host sync), repeats the reset for the envs that are still unsolved (sampled
        starts only) and raises ``MapdnError`` after ``max_retries`` rounds - the B = 1 shim does this."""
        if start is not None:
            self._chk(start, (self.batch, 3), torch.int32, "start")
        if mask is not None:
            self._chk(mask, (self.batch,), torch.uint8, "mask")
        p_state = _ptr(self.state) if want_state else None          # rollouts that never read get_state skip it
        _capi.check(self._L.mapdn_reset(self._h, _ptr(start), _ptr(mask), int(add_noise), _ptr(self.obs),
                                        p_state, _ptr(self.reset_ok), self._stream()))
        if check:
            sel = torch.ones_like(self.reset_ok) if mask is None else mask
            for _ in range(max_retries + 1):
                bad = ((self.reset_ok == 0) & (sel != 0)).to(torch.uint8)
                if not bool(bad.any()):
                    break
                if start is not None:
                    raise MapdnError("manual_reset: the power flow of the requested start does not converge")
                _capi.check(self._L.mapdn_reset(self._h, None, _ptr(bad), int(add_noise), _ptr(self.obs),
                                                p_state, _ptr(self.reset_ok), self._stream()))
                sel = bad
            else:
                raise MapdnError(f"reset: {int(bad.sum())} env(s) found no solvable start in "
                                 f"{16 * (max_retries + 1)} draws")
        if mask is not None and want_state:   # state of the untouched envs
            _capi.check(self._L.mapdn_get_state(self._h, _ptr(self.state), self._stream()))
        if self.history > 1:
            if self._hist is None or mask is None:
                self._hist = torch.zeros(self.batch, self.history, self.n_agents, self.obs_size, dtype=torch.float64,
                                         device=self.device)
            else:
                self._hist[mask.bool()] = 0.0
            self._hist[:, -1] = self.obs
        return self.obs, self.state

    def step(self, actions: torch.Tensor, add_noise: bool = True, want_obs: bool = True, want_info: bool = True):
        """One transition of every env. Returns (reward ``[B]``, terminated ``[B]`` uint8,
        info ``[B,11]`` in INFO_KEYS order); the new observations are in ``self.obs``."""
        if (actions.dtype is not torch.float64 or tuple(actions.shape) != self._act_shape or actions.device != self.device
                or not actions.is_contiguous()):
            self._chk(actions, self._act_shape, name="actions")
        st = self._L.mapdn_step(self._h, actions.data_ptr(), int(add_noise), self._p_reward, self._p_term,
                                self._p_info if want_info else None, self._p_obs if want_obs else None,
                                torch.cuda.current_stream(self.device).cuda_stream)
        if st:
            _capi.check(st)
        if self.history > 1 and want_obs and self._hist is not None:
            self._hist = torch.roll(self._hist, -1, dims=1)
            self._hist[:, -1] = self.obs
        return self.reward, self.terminated, self.info

    # host-buffer path (what a CPU-side caller such as the reference trainer pays end to end)
    def _host_buffers(self):
        if self._host is None:
            B, pin = self.batch, dict(pin_memory=True)
            self._host = dict(
                actions=torch.zeros(B, self.n_agents, dtype=torch.float64, **pin),
                reward=torch.zeros(B, dtype=torch.float64, **pin),
                terminated=torch.zeros(B, dtype=torch.uint8, **pin),
                info=torch.zeros(B, len(INFO_KEYS), dtype=torch.float64, **pin),
                obs=torch.zeros(B, self.n_agents, self.obs_size, dtype=torch.float64, **pin),
                obs32=torch.zeros(B, self.n_agents, self.obs_size, dtype=torch.float32, **pin))
        return self._host

    def step_host(self, actions: np.ndarray, add_noise: bool = True, obs_dtype=np.float64,
                  staged: Optional[bool] = None, sync: bool = True, layout: str = "padded"):
        """NumPy in / NumPy out. Default: the zero-copy path (``mapdn_step_host_pinned``) - the fused kernel reads the
        actions from and writes reward / terminated / info / observations straight to this object's pinned host
        buffers, so the PCIe transfer overlaps the kernel; the never-changing zero padding of the observation rows is
        not rewritten. ``staged=True``: the round-1 path (H2D copy, kernel, four D2H copies). ``obs_dtype=np.float32``
        delivers the observations in fp32 (what the reference's learners use after ``prep_obs``). ``sync=False`` returns
        right after the launch - call :meth:`wait` before reading the results. Returns views of pinned host buffers
        (overwritten by the next call).

        ``layout="compact"`` (``mapdn_step_host_compact``): the observations arrive as rows ``[B, row_len]`` without the
        zero padding of the reference's ``get_obs`` - agent ``a`` owns ``obs[:, off:off + n]`` with ``(off, n) =
        self.obs_slices[a]`` (a strided NumPy view, no copy; :meth:`expand_obs` rebuilds the padded array). The rows
        go through device memory and ONE contiguous copy-engine transfer by default (``staged=False`` makes the kernel
        write them to host memory itself, like the padded path: on an H100 about as fast, 18.7 against 18.8 M
        env-steps/s for case33 x 4096)."""
        hb = self._host_buffers()
        hb["actions"].numpy()[...] = actions
        f32 = np.dtype(obs_dtype) == np.float32
        stream = torch.cuda.current_stream(self.device).cuda_stream
        if layout == "compact":
            if self.history > 1:
                raise NotImplementedError("compact host rows carry one frame (history = 1)")
            row = self.obs_row_len
            key = "obs_c32" if f32 else "obs_c"
            if key not in hb:
                hb[key] = torch.zeros(self.batch, row, dtype=torch.float32 if f32 else torch.float64).pin_memory()
            obs = hb[key]
            _capi.check(self._L.mapdn_step_host_compact(self._h, hb["actions"].data_ptr(), int(add_noise),
                                                        hb["reward"].data_ptr(), hb["terminated"].data_ptr(),
                                                        hb["info"].data_ptr(), obs.data_ptr(), int(f32),
                                                        int(staged is False), int(sync), stream))
            return hb["reward"].numpy(), hb["terminated"].numpy(), hb["info"].numpy(), obs.numpy()
        if layout != "padded":
            raise ValueError("layout must be 'padded' or 'compact'")
        obs = hb["obs32"] if f32 else hb["obs"]
        if staged:
            fn = self._L.mapdn_step_host_f32obs if f32 else self._L.mapdn_step_host
            _capi.check(fn(self._h, hb["actions"].data_ptr(), int(add_noise), hb["reward"].data_ptr(),
                           hb["terminated"].data_ptr(), hb["info"].data_ptr(), obs.data_ptr(), stream))
        else:
            _capi.check(self._L.mapdn_step_host_pinned(self._h, hb["actions"].data_ptr(), int(add_noise),
                                                       hb["reward"].data_ptr(), hb["terminated"].data_ptr(),
                                                       hb["info"].data_ptr(), obs.data_ptr(), int(f32), 1, int(sync), stream))
        return hb["reward"].numpy(), hb["terminated"].numpy(), hb["info"].numpy(), obs.numpy()

    def wait(self):
        """Blocks until the results of a ``step_host(..., sync=False)`` are in the host buffers."""
        _capi.check(self._L.mapdn_wait(self._h, torch.cuda.current_stream(self.device).cuda_stream))

    def _compact_layout(self):
        if getattr(self, "_obs_slices", None) is None:
            off = (C.c_int32 * self.n_agents)()
            ln = (C.c_int32 * self.n_agents)()
            row = C.c_int32(0)
            _capi.check(self._L.mapdn_obs_compact_layout(self._h, off, ln, C.byref(row)))
            self._obs_slices = [(int(off[a]), int(ln[a])) for a in range(self.n_agents)]
            self._obs_row_len = int(row.value)
        return self._obs_slices, self._obs_row_len

    @property
    def obs_slices(self):
        """``[(offset, length)]`` of every agent's block in a compact observation row (``step_host(layout="compact")``)."""
        return self._compact_layout()[0]

    @property
    def obs_row_len(self) -> int:
        return self._compact_layout()[1]

    def expand_obs(self, compact: np.ndarray) -> np.ndarray:
        """Compact rows ``[B, row_len]`` -> the reference's padded ``[B, n_agents, obs_dim]`` (a host-side copy: for checks
        and for consumers that insist on the padded layout)."""
        out = np.zeros((compact.shape[0], self.n_agents, self.obs_size), dtype=compact.dtype)
        for a, (off, n) in enumerate(self.obs_slices):
            out[:, a, :n] = compact[:, off:off + n]
        return out

    @property
    def host_obs_bytes_per_env(self) -> int:
        """fp64 bytes of one env's observations that are not padding (what the zero-copy host path moves)."""
        if getattr(self, "_obs_used", None) is None:
            zones = [int((self.net.bus_zone == z).sum()) for z in self.net.sgen_zone]
            ss = set(self.args["state_space"])
            per = [nz * (2 * ("demand" in ss) + ("vm_pu" in ss) + ("va_degree" in ss)) + ("pv" in ss) + ("reactive" in ss)
                   for nz in zones]
            self._obs_used = 8 * int(sum(per))
        return self._obs_used

    def get_obs_stacked(self) -> torch.Tensor:
        """``history`` stacked observations ``[B, n_agents, history * obs_dim]``, oldest frame first and zero frames
        before the episode start (reference :303-315; one frame per reset / step, not per ``get_obs`` call)."""
        if self.history <= 1 or self._hist is None:
            return self.obs
        return self._hist.permute(0, 2, 1, 3).reshape(self.batch, self.n_agents, self.history * self.obs_size)

    # ---- getters ------------------------------------------------------------------------------
    def get_obs(self) -> torch.Tensor:
        _capi.check(self._L.mapdn_get_obs(self._h, _ptr(self.obs), self._stream()))
        return self.obs

    def get_state(self) -> torch.Tensor:
        _capi.check(self._L.mapdn_get_state(self._h, _ptr(self.state), self._stream()))
        return self.state

    def get_field(self, name: str) -> torch.Tensor:
        d = self.dims
        width = dict(vm=d["n_bus"], va_deg=d["n_bus"], p_bus=d["n_bus"], q_bus=d["n_bus"], p_sgen=d["n_sgen"],
                     q_sgen=d["n_sgen"], line_loss=d["n_line"], p_load=d["n_load"], q_load=d["n_load"],
                     sum_rewards=1, steps=1, start_row=1, nr_iters=1)[name]
        out = torch.empty(self.batch, width, dtype=torch.float64, device=self.device)
        _capi.check(self._L.mapdn_get_field(self._h, _capi.FIELDS[name], _ptr(out), self._stream()))
        return out

    def get_avail_actions(self) -> torch.Tensor:
        return torch.ones(self.batch, self.n_agents, self.n_actions, device=self.device)

    def get_env_info(self):
        return {"state_shape": self.state_size, "obs_shape": self.obs_size, "n_actions": self.n_actions,
                "n_agents": self.n_agents, "episode_limit": self.episode_limit}

    # ---- stateless batched power flow (pp.runpp on explicit element values) ---------------------
    def solve(self, p_load, q_load, p_sgen, q_sgen, want=("vm", "va_deg", "p_bus", "q_bus", "pl")):
        nb = int(p_sgen.shape[0])
        d = self.dims
        ins = []
        for t, w, nm in ((p_load, d["n_load"], "p_load"), (q_load, d["n_load"], "q_load"),
                         (p_sgen, d["n_sgen"], "p_sgen"), (q_sgen, d["n_sgen"], "q_sgen")):
            t = torch.as_tensor(t, dtype=torch.float64, device=self.device).contiguous()
            if tuple(t.shape) != (nb, w):
                raise ValueError(f"{nm}: expected shape {(nb, w)}, got {tuple(t.shape)}")
            ins.append(t)
        widths = dict(vm=d["n_bus"], va_deg=d["n_bus"], p_bus=d["n_bus"], q_bus=d["n_bus"], pl=d["n_line"])
        out = {k: (torch.empty(nb, widths[k], dtype=torch.float64, device=self.device) if k in want else None)
               for k in widths}
        out["iterations"] = torch.empty(nb, dtype=torch.int32, device=self.device)
        out["converged"] = torch.empty(nb, dtype=torch.uint8, device=self.device)
        _capi.check(self._L.mapdn_solve(self._h, nb, *[_ptr(t) for t in ins], _ptr(out["vm"]), _ptr(out["va_deg"]),
                                        _ptr(out["p_bus"]), _ptr(out["q_bus"]), _ptr(out["pl"]),
                                        _ptr(out["iterations"]), _ptr(out["converged"]), self._stream()))
        return out

    def ybus_dense(self) -> np.ndarray:
        n = self.dims["n_bus"]
        g, b = np.zeros((n, n)), np.zeros((n, n))
        _capi.check(self._L.mapdn_get_ybus_dense(self._h, g.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p)))
        return g + 1j * b


class VoltageControl:
    """Drop-in for the reference ``VoltageControl(MultiAgentEnv)`` (B = 1, NumPy in / out).

    ``kwargs`` is the reference's ``env_args`` dict / namedtuple (train.py:25-46, :62). The network
    and profiles come from ``kwargs["net"]``/``kwargs["profiles"]`` (:class:`NetDesc`,
    :class:`ProfileDesc`), from ``kwargs["scenario"]`` (synthetic stand-in, ``mapdn_b200.cases``) or
    from ``kwargs["data_path"]`` (reference file formats, ``mapdn_b200.ingest``).
    """

    def __init__(self, kwargs):
        args = kwargs
        if not isinstance(args, dict):
            args = args._asdict()
        args = dict(args)
        net, prof = args.pop("net", None), args.pop("profiles", None)
        scenario = args.pop("scenario", None)
        if net is None:
            if scenario is not None:
                from . import cases
                net, prof = cases.make_case(scenario), cases.make_profiles(scenario)
            else:
                from . import ingest
                net, prof = ingest.load_scenario(args["data_path"], pv_scale=args.get("pv_scale", 1.0),
                                                 demand_scale=args.get("demand_scale", 1.0))
        merged = dict(DEFAULT_ENV_ARGS)
        merged.update(args)
        self.args = convert({k: v for k, v in merged.items() if isinstance(k, str)})
        self.data_path = merged.get("data_path")
        self.history = int(merged.get("history", 1))
        env_args = dict(merged)
        env_args["history"] = 1
        self._env = BatchedVoltageControl(net, prof, env_args, batch=1, device=merged.get("device"))
        e = self._env
        self.base_powergrid = net
        self.episode_limit = e.episode_limit
        self.voltage_barrier_type = merged["voltage_barrier_type"]
        self.voltage_weight, self.q_weight = merged["voltage_weight"], merged["q_weight"]
        self.line_weight, self.dv_dq_weight = merged["line_weight"], merged.get("dq_dv_weight")
        self.v_upper, self.v_lower = merged["v_upper"], merged["v_lower"]
        self.pv_std, self.active_demand_std, self.reactive_demand_std = prof.pv_std, prof.load_p_std, prof.load_q_std
        self.factor = 1.2
        self.p_max = prof.pv.max(axis=0)
        self.s_max = prof.s_max
        self.action_space = e.action_space
        self.state_space = merged["state_space"]
        self.n_actions, self.n_agents = e.n_actions, e.n_agents
        self._start = torch.zeros(1, 3, dtype=torch.int32, device=e.device)
        self._act = torch.zeros(1, e.n_agents, dtype=torch.float64, device=e.device)
        agents_obs, state = self.reset()
        self.obs_size = agents_obs[0].shape[0]
        self.state_size = state.shape[0]
        self.last_v = self._get_res_bus_v()
        self.last_q = self._get_sgen_reactive()

    # ---- reset ---------------------------------------------------------------------------------
    def _after_reset(self):
        self.steps = 1
        self.sum_rewards = 0
        self.obs_history = {i: [] for i in range(self.n_agents)}
        # reset wrote obs / state of the new episode into the env's device buffers: one copy each, then get_obs() /
        # get_state() are served from the host until the next transition (no kernel, no sync per getter call)
        self._obs_host = self._env.obs[0].cpu().numpy()
        self._state_host = self._env.state[0].cpu().numpy()
        return self.get_obs(), self.get_state()

    def reset(self, reset_time=True):
        if reset_time or not hasattr(self, "_last_start"):
            self._env.reset(None, add_noise=True, check=True)
        else:
            self._env.reset(self._last_start, add_noise=True, check=True)
        start = int(self._env.get_field("start_row").item())
        sph = self._env.profiles.steps_per_hour
        self._episode_start_day, rem = divmod(start, 24 * sph)
        self._episode_start_hour, self._episode_start_interval = divmod(rem, sph)
        self._last_start = torch.tensor([[self._episode_start_day, self._episode_start_hour,
                                          self._episode_start_interval]], dtype=torch.int32, device=self._env.device)
        return self._after_reset()

    def manual_reset(self, day, hour, interval):
        sph, prof = self._env.profiles.steps_per_hour, self._env.profiles
        start = interval + hour * sph + day * 24 * sph
        if not (0 <= hour < 24 and 0 <= interval < sph and day >= 0 and start + self.episode_limit <= prof.n_rows - 1):
            # the reference would slice a short window here and fail later inside step (:440-468)
            raise ValueError(f"manual_reset({day}, {hour}, {interval}): the episode window does not fit the "
                             f"{prof.n_rows}-row profile store")
        self._episode_start_day, self._episode_start_hour, self._episode_start_interval = day, hour, interval
        self._last_start = torch.tensor([[day, hour, interval]], dtype=torch.int32, device=self._env.device)
        self._env.reset(self._last_start, add_noise=False, check=True)          # reference :159
        return self._after_reset()

    # ---- step ----------------------------------------------------------------------------------
    def step(self, actions, add_noise=True):
        a = np.asarray(actions, dtype=np.float64).reshape(1, self.n_agents)
        r, t, info, obs = self._env.step_host(a, add_noise=add_noise)      # one launch; results land in pinned host memory
        reward, terminated = float(r[0]), bool(t[0])
        info = {k: float(v) for k, v in zip(INFO_KEYS, info[0])}
        self._obs_host, self._state_host = obs[0].copy(), None
        self.steps += 1
        self.sum_rewards += reward
        if terminated:
            print(f"Episode terminated at time: {self.steps} with return: {self.sum_rewards:2.4f}.")
        return reward, terminated, info

    # ---- observations --------------------------------------------------------------------------
    def get_state(self):
        if self._state_host is None:
            self._state_host = self._env.get_state()[0].cpu().numpy()
        return self._state_host.copy()

    def get_obs(self):
        obs = self._obs_host
        agents_obs = [obs[i].copy() for i in range(self.n_agents)]
        if self.history > 1:                                          # reference :303-315
            agents_obs_ = []
            for i, o in enumerate(agents_obs):
                if len(self.obs_history[i]) >= self.history - 1:
                    o_ = np.concatenate(self.obs_history[i][-self.history + 1:] + [o], axis=0)
                else:
                    zeros = [np.zeros_like(o)] * (self.history - len(self.obs_history[i]) - 1)
                    o_ = np.concatenate(zeros + self.obs_history[i] + [o], axis=0)
                agents_obs_.append(o_.copy())
                self.obs_history[i].append(o.copy())
            agents_obs = agents_obs_
        return agents_obs

    def get_obs_agent(self, agent_id):
        return self.get_obs()[agent_id]

    def get_obs_size(self):
        return self.obs_size

    def get_state_size(self):
        return self.state_size

    def get_action(self):
        return np.random.uniform(low=self.action_space.low, high=self.action_space.high, size=(self.n_agents,))

    def get_total_actions(self):
        return self.n_actions

    def get_avail_actions(self):
        return np.expand_dims(np.array([self.get_avail_agent_actions(i) for i in range(self.n_agents)]), axis=0)

    def get_avail_agent_actions(self, agent_id):
        return [1]

    def get_num_of_agents(self):
        return self.n_agents

    def get_env_info(self):                                           # multiagentenv.py:61-67
        return {"state_shape": self.get_state_size(), "obs_shape": self.get_obs_size(),
                "n_actions": self.get_total_actions(), "n_agents": self.n_agents,
                "episode_limit": self.episode_limit}

    # ---- private getters used by the reference tester (utilities/tester.py:34-39) ---------------
    def _f(self, name):
        return self._env.get_field(name)[0].cpu().numpy()

    def _get_voltage(self):
        return self._f("vm")

    def _get_res_bus_v(self):
        return self._f("vm")

    def _get_res_bus_active(self):
        return self._f("p_bus")

    def _get_res_bus_reactive(self):
        return self._f("q_bus")

    def _get_res_line_loss(self):
        return self._f("line_loss")

    def _get_sgen_active(self):
        return self._f("p_sgen")

    def _get_sgen_reactive(self):
        return self._f("q_sgen")

    def _clip_reactive_power(self, reactive_actions, active_power):   # :568-572
        return np.sqrt(self.s_max ** 2 - active_power ** 2) * reactive_actions

    def render(self, mode="human"):
        raise NotImplementedError("rendering is out of scope (SURVEY §2 #6)")

    def res_pf_plot(self):
        raise NotImplementedError("plotting is out of scope (SURVEY §2 #6)")

    def close(self):
        self._env.close()

    def seed(self):
        return self.args.seed

    def get_stats(self):
        return {}

    def get_agg_stats(self, stats):
        return {}

    def save_replay(self):
        raise NotImplementedError
