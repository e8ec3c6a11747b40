"""Host-side mirror of the reference env API over the C-ABI.

* :class:`BatchedVoltageControl` - B independent env instances resident in HBM, tensor in/out,
  one fused CUDA launch per ``step``.
* :class:`VoltageControl` - drop-in for the reference class of the same name
  (reference ``environments/var_voltage_control/voltage_control_env.py:24``): B = 1, NumPy in/out,
  same method names, argument meaning and return shapes (PyMARL ``MultiAgentEnv`` API,
  reference ``environments/multiagentenv.py``).

There is no CPU fallback: by default both classes bind the CUDA library and need a GPU. ``BatchedVoltageControl(...,
library=L, device="cpu")`` binds another build of the C-ABI whose device memory is host memory.
"""
from __future__ import annotations

import ctypes as C
import hashlib
from collections import namedtuple
from typing import Optional

import numpy as np
import torch

from . import _capi
from ._capi import INFO_KEYS, MapdnError
from .network import NetDesc, ProfileDesc

__all__ = ["BatchedVoltageControl", "EnvSnapshot", "VoltageControl", "ActionSpace", "DEFAULT_ENV_ARGS", "INFO_KEYS"]

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


# mapdn_cfg fields that only place the envs (batch, global id of env 0) or change the last bits (lanes per env)
_PLACEMENT_FIELDS = ("batch", "env_id_offset", "lanes_per_env")


def snapshot_fingerprint(net: NetDesc, profiles: Optional[ProfileDesc], env_args: dict, history: int = 1,
                         tol: float = 0.0, max_iter: int = 0) -> str:
    """sha256 (hex) of what the dynamics of an env depend on: the net and profile arrays as ``mapdn_create`` receives
    them, every ``mapdn_cfg`` field except batch, env_id_offset and lanes_per_env (barrier, weights, voltage limits,
    episode_limit, action range, reset_action, seed, state_space, tol and max_iter with their defaults filled in) and the
    observation history. A snapshot restores only into an env with the same fingerprint."""
    h = hashlib.sha256()

    def put(tag, v):
        h.update(tag.encode() + b"=")
        if v is None:
            h.update(b"none;")
        elif isinstance(v, np.ndarray):
            a = np.ascontiguousarray(v)
            h.update(f"{a.dtype.str}{a.shape};".encode())
            h.update(memoryview(a).cast("B"))
        elif isinstance(v, float):
            h.update(v.hex().encode() + b";")
        else:
            h.update(repr(v).encode() + b";")

    for k in ("n_bus", "base_mva", "slack_bus", "slack_vm", "slack_va_deg"):
        put(k, getattr(net, k))
    put("vm_init", None if net.vm_init is None else float(net.vm_init))
    nd, keep = _capi.make_net_desc(net)
    for i, a in enumerate(keep):
        put(f"net{i}", a)
    del nd
    if profiles is None:
        put("profiles", None)
    else:
        put("rows", (profiles.n_rows, profiles.steps_per_hour, profiles.n_days))
        for i, a in enumerate(_capi.make_profile_desc(profiles)[1]):
            put(f"prof{i}", a)
    cfg = _capi.make_cfg(env_args, 1, 0, 0, tol, max_iter)
    cfg.tol = cfg.tol if cfg.tol > 0 else 1e-8                       # the defaults mapdn_create fills in
    cfg.max_iter = cfg.max_iter if cfg.max_iter > 0 else 10
    for name, _ in cfg._fields_:
        if name not in _PLACEMENT_FIELDS:
            put(name, getattr(cfg, name))
    put("history", int(history))
    return h.hexdigest()


class EnvSnapshot:
    """The device state of ``n`` envs of a :class:`BatchedVoltageControl` (``mapdn_snapshot``).

    * ``data``: uint8 ``[n, bytes_per_env]`` on the env's device, one row per env (:meth:`segment` decodes it);
    * ``env_ids``: int64 ``[n]`` (CPU) global ids of the envs the rows came from (``env_id_offset + slot``);
    * ``layout``: the segment offsets of a row (``mapdn_snapshot_layout``, last = bytes_per_env);
    * ``history`` and ``fingerprint`` of the env (:func:`snapshot_fingerprint`).

    :meth:`state_dict` holds only tensors and plain Python values, so a checkpoint with it loads with
    ``torch.load(weights_only=True)``."""

    def __init__(self, data: torch.Tensor, env_ids: torch.Tensor, layout, history: int, fingerprint: str):
        self.data, self.env_ids = data, env_ids.to(torch.int64).cpu()
        self.layout, self.history, self.fingerprint = [int(x) for x in layout], int(history), str(fingerprint)
        if data.dtype != torch.uint8 or data.dim() != 2 or data.shape[0] != self.env_ids.numel():
            raise ValueError(f"snapshot data must be uint8 [n, bytes_per_env] with n = len(env_ids), got "
                             f"{data.dtype} {tuple(data.shape)} for {self.env_ids.numel()} ids")

    def __len__(self):
        return int(self.env_ids.numel())

    def state_dict(self) -> dict:
        return dict(data=self.data, env_ids=self.env_ids, layout=list(self.layout), history=self.history,
                    fingerprint=self.fingerprint)

    @classmethod
    def from_state_dict(cls, d: dict) -> "EnvSnapshot":
        return cls(d["data"], d["env_ids"], d["layout"], d["history"], d["fingerprint"])

    def segment(self, name: str, count: int) -> torch.Tensor:
        """Segment ``name`` (``_capi.SNAPSHOT_SEGMENTS``) of every row decoded as ``[n, count]`` of its element type;
        ``count`` is the array's entries per env (``n_load``, ``n_sgen``, ``n_bus``, ``n_line`` of ``env.dims``, 1 for the
        scalars, ``history * n_agents * obs_dim`` for the frame ring)."""
        s = _capi.SNAPSHOT_SEGMENTS.index(name)
        dt = {np.int64: torch.int64, np.int32: torch.int32, np.uint32: torch.int32}.get(
            _capi.SNAPSHOT_DTYPES.get(name), torch.float64)
        size = torch.empty((), dtype=dt).element_size()
        raw = self.data[:, self.layout[s]:self.layout[s] + count * size].contiguous()
        return raw.view(dt).reshape(len(self), count)


class BatchedVoltageControl:
    """``batch`` env instances on one GPU. All tensors are fp64 CUDA tensors, row-major ``[B, ...]``.

    ``env_args``: dict with the keys of the reference's ``env_args`` (DEFAULT_ENV_ARGS).
    ``env_id_offset``: global id of env 0 (multi-GPU sharding keeps the RNG streams per env id).
    ``library``: the C-ABI library to bind (``ctypes.CDLL`` with ``_capi.bind`` applied), ``_capi.lib()`` when None.
    ``device="cpu"`` needs one whose "device" memory is host memory (such as a build of the kernel source for a CPU
    emulation of CUDA): the tensors are then CPU tensors, host buffers are not pinned and no stream is passed.
    """

    def __init__(self, net: NetDesc, profiles: Optional[ProfileDesc], env_args: Optional[dict] = None,
                 batch: int = 1, device: Optional[int] = None, env_id_offset: int = 0,
                 lanes_per_env: int = 0, tol: float = 0.0, max_iter: int = 0, library: Optional[C.CDLL] = None):
        self._cpu = str(device) == "cpu"
        if self._cpu and library is None:
            raise MapdnError("device='cpu' needs a library whose device memory is host memory (there is no CPU fallback)")
        if not self._cpu and not torch.cuda.is_available():
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
        if self._cpu:
            self.device_index, self.device = 0, torch.device("cpu")
        else:
            self.device_index = torch.cuda.current_device() if device is None else int(device)
            self.device = torch.device("cuda", self.device_index)
        L = _capi.lib() if library is None else library
        cfg = _capi.make_cfg(args, self.batch, env_id_offset, lanes_per_env, tol, max_iter)
        if args["line_weight"] is None and args["q_weight"] is None:
            raise NotImplementedError("Please at least give one weight, either q_weight or line_weight.")
        nd, keep1 = _capi.make_net_desc(net)
        pd_, keep2 = (None, None) if profiles is None else _capi.make_profile_desc(profiles)
        h = C.c_void_p()
        _capi.check(L.mapdn_create(C.byref(nd), None if pd_ is None else C.byref(pd_), C.byref(cfg),
                                   self.device_index, C.byref(h)), L)
        del keep1, keep2
        self._h, self._L = h, L
        d = _capi.DimsC()
        _capi.check(L.mapdn_get_dims(h, C.byref(d)), L)
        self.dims = {k: getattr(d, k) for k, _ in d._fields_}
        self.n_agents, self.n_actions = d.n_agents, d.n_actions
        self.obs_size, self.state_size = d.obs_dim, d.state_dim
        self.episode_limit = int(args["episode_limit"])
        self.action_space = ActionSpace(low=-args["action_scale"] + args["action_bias"],
                                        high=args["action_scale"] + args["action_bias"])
        self.s_max = None if profiles is None else profiles.s_max
        B, f64 = self.batch, torch.float64
        self.obs = torch.zeros(B, d.n_agents, d.obs_dim, dtype=f64, device=self.device)
        self.state = torch.zeros(B, d.state_dim, dtype=f64, device=self.device)
        self.reward = torch.zeros(B, dtype=f64, device=self.device)
        self.terminated = torch.zeros(B, dtype=torch.uint8, device=self.device)
        self.info = torch.zeros(B, len(INFO_KEYS), dtype=f64, device=self.device)
        self.reset_ok = torch.ones(B, dtype=torch.uint8, device=self.device)
        # history > 1 (reference :303-315): the step kernel keeps a ring of the last frames and writes the stacked rows
        # [B, n_agents, history * obs_dim] here; a learner is sized with stacked_obs_size
        self.stacked_obs_size = self.history * self.obs_size
        self.obs_stacked = self.obs
        if self.history > 1:
            _capi.check(L.mapdn_set_history(h, self.history), L)
            self.obs_stacked = torch.zeros(B, d.n_agents, self.stacked_obs_size, dtype=f64, device=self.device)
        self._host = None
        # what the snapshot fingerprint covers beyond the net and the profile store (computed on first use)
        self.env_id_offset = int(env_id_offset)
        self._cfg, self._fingerprint, self._snapshot_layout = cfg, None, None
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
        """Handle of the device's current stream (None on the CPU device); ctypes converts both for a c_void_p."""
        return None if self._cpu else torch.cuda.current_stream(self.device).cuda_stream

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
                                        p_state, _ptr(self.reset_ok), self._stream()), self._L)
        if check:
            sel = torch.ones_like(self.reset_ok) if mask is None else mask
            for _ in range(max_retries + 1):
                bad = ((self.reset_ok == 0) & (sel != 0)).to(torch.uint8)
                if not bool(bad.any()):
                    break
                if start is not None:
                    raise MapdnError("manual_reset: the power flow of the requested start does not converge")
                _capi.check(self._L.mapdn_reset(self._h, None, _ptr(bad), int(add_noise), _ptr(self.obs),
                                                p_state, _ptr(self.reset_ok), self._stream()), self._L)
                sel = bad
            else:
                raise MapdnError(f"reset: {int(bad.sum())} env(s) found no solvable start in "
                                 f"{16 * (max_retries + 1)} draws")
        if mask is not None and want_state:   # state of the untouched envs
            _capi.check(self._L.mapdn_get_state(self._h, _ptr(self.state), self._stream()), self._L)
        if self.history > 1:
            _capi.check(self._L.mapdn_get_obs_stacked(self._h, _ptr(self.obs_stacked), self._stream()), self._L)
        return self.obs, self.state

    def step(self, actions: torch.Tensor, add_noise: bool = True, want_obs: bool = True, want_info: bool = True,
             record: Optional[torch.Tensor] = None):
        """One transition of every env. Returns (reward ``[B]``, terminated ``[B]`` uint8,
        info ``[B,11]`` in INFO_KEYS order); the new observations are in ``self.obs`` and, with ``history > 1``, the
        stacked rows in ``self.obs_stacked`` (the same launch; ``want_obs=False`` skips both, the frame is still recorded).

        ``record``: an fp64 ``[B, record_len]`` view with unit column stride and any row stride (row ``t`` of a
        ``[B, T + 1, record_len]`` tensor): the same kernel launch also writes every env's tester record after the step
        (:attr:`record_slices`, ``mapdn_step_record``)."""
        if (actions.dtype is not torch.float64 or tuple(actions.shape) != self._act_shape or actions.device != self.device
                or not actions.is_contiguous()):
            self._chk(actions, self._act_shape, name="actions")
        stream = self._stream()
        if self.history > 1:
            st = self._L.mapdn_step_stacked(self._h, actions.data_ptr(), int(add_noise), self._p_reward, self._p_term,
                                            self._p_info if want_info else None, self._p_obs if want_obs else None,
                                            self.obs_stacked.data_ptr() if want_obs else None,
                                            None if record is None else record.data_ptr(),
                                            0 if record is None else self._record_stride(record), stream)
        elif record is not None:
            st = self._L.mapdn_step_record(self._h, actions.data_ptr(), int(add_noise), self._p_reward, self._p_term,
                                           self._p_info if want_info else None, self._p_obs if want_obs else None,
                                           record.data_ptr(), self._record_stride(record), stream)
        else:
            st = self._L.mapdn_step(self._h, actions.data_ptr(), int(add_noise), self._p_reward, self._p_term,
                                    self._p_info if want_info else None, self._p_obs if want_obs else None, stream)
        if st:
            _capi.check(st, self._L)
        return self.reward, self.terminated, self.info

    def step_autoreset(self, actions: torch.Tensor, add_noise: bool = True):
        """:meth:`step` in which every env that terminates starts its next episode in the same launch
        (``mapdn_step_autoreset``). Returns (reward, terminated, info) like :meth:`step`; ``self.obs`` /
        ``self.obs_stacked`` hold the observation after the step (the terminal one of an env that ended). For the envs
        with ``terminated = 1``, ``self.reset_obs`` (and ``self.reset_obs_stacked`` with ``history > 1``) hold the first
        observation of the new episode and ``self.reset_ok`` the reset outcome, as :meth:`reset` with
        ``mask=terminated`` would give them; the rows of the other envs are not written. No host sync.

        So after this call ``self.obs`` / ``self.obs_stacked`` are not the current state's observation for the envs that
        ended (``get_obs()`` / ``get_obs_stacked()`` are): a caller that resumes later keeps
        ``torch.where(terminated, reset_obs, obs)`` as its current observation."""
        if (actions.dtype is not torch.float64 or tuple(actions.shape) != self._act_shape or actions.device != self.device
                or not actions.is_contiguous()):
            self._chk(actions, self._act_shape, name="actions")
        if getattr(self, "reset_obs", None) is None:
            self.reset_obs = torch.zeros_like(self.obs)
            self.reset_obs_stacked = torch.zeros_like(self.obs_stacked) if self.history > 1 else self.reset_obs
        hist = self.history > 1
        st = self._L.mapdn_step_autoreset(self._h, actions.data_ptr(), int(add_noise), self._p_reward, self._p_term,
                                          self._p_info, self._p_obs, self.obs_stacked.data_ptr() if hist else None,
                                          self.reset_obs.data_ptr(), self.reset_obs_stacked.data_ptr() if hist else None,
                                          self.reset_ok.data_ptr(), self._stream())
        if st:
            _capi.check(st, self._L)
        return self.reward, self.terminated, self.info

    # host-buffer path (what a CPU-side caller such as the reference trainer pays end to end)
    def _host_buffers(self):
        if self._host is None:
            B, pin = self.batch, dict(pin_memory=not self._cpu)
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
        stream = self._stream()
        if layout == "compact":
            row = self.obs_row_len
            key = "obs_c32" if f32 else "obs_c"
            if key not in hb:
                hb[key] = torch.zeros(self.batch, row, dtype=torch.float32 if f32 else torch.float64,
                                      pin_memory=not self._cpu)
            obs = hb[key]
            _capi.check(self._L.mapdn_step_host_compact(self._h, hb["actions"].data_ptr(), int(add_noise),
                                                        hb["reward"].data_ptr(), hb["terminated"].data_ptr(),
                                                        hb["info"].data_ptr(), obs.data_ptr(), int(f32),
                                                        int(staged is False), int(sync), stream), self._L)
            return hb["reward"].numpy(), hb["terminated"].numpy(), hb["info"].numpy(), obs.numpy()
        if layout != "padded":
            raise ValueError("layout must be 'padded' or 'compact'")
        obs = hb["obs32"] if f32 else hb["obs"]
        if staged:
            fn = self._L.mapdn_step_host_f32obs if f32 else self._L.mapdn_step_host
            _capi.check(fn(self._h, hb["actions"].data_ptr(), int(add_noise), hb["reward"].data_ptr(),
                           hb["terminated"].data_ptr(), hb["info"].data_ptr(), obs.data_ptr(), stream), self._L)
        else:
            _capi.check(self._L.mapdn_step_host_pinned(self._h, hb["actions"].data_ptr(), int(add_noise),
                                                       hb["reward"].data_ptr(), hb["terminated"].data_ptr(),
                                                       hb["info"].data_ptr(), obs.data_ptr(), int(f32), 1, int(sync),
                                                       stream), self._L)
        return hb["reward"].numpy(), hb["terminated"].numpy(), hb["info"].numpy(), obs.numpy()

    def wait(self):
        """Blocks until the results of a ``step_host(..., sync=False)`` are in the host buffers."""
        _capi.check(self._L.mapdn_wait(self._h, self._stream()), self._L)

    def _compact_layout(self):
        if getattr(self, "_obs_slices", None) is None:
            off = (C.c_int32 * self.n_agents)()
            ln = (C.c_int32 * self.n_agents)()
            row = C.c_int32(0)
            _capi.check(self._L.mapdn_obs_compact_layout(self._h, off, ln, C.byref(row)), self._L)
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
        before the episode start (reference :303-315; one frame per reset / step, not per ``get_obs`` call), in a new
        tensor gathered from the device's frame ring: current after every reset and step, host-path steps included."""
        if self.history <= 1:
            return self.obs
        out = torch.empty_like(self.obs_stacked)
        _capi.check(self._L.mapdn_get_obs_stacked(self._h, _ptr(out), self._stream()), self._L)
        return out

    # ---- getters ------------------------------------------------------------------------------
    def get_obs(self) -> torch.Tensor:
        _capi.check(self._L.mapdn_get_obs(self._h, _ptr(self.obs), self._stream()), self._L)
        return self.obs

    def get_state(self) -> torch.Tensor:
        _capi.check(self._L.mapdn_get_state(self._h, _ptr(self.state), self._stream()), self._L)
        return self.state

    def get_field(self, name: str) -> torch.Tensor:
        out = torch.empty(self.batch, self.dims.get(_capi.FIELD_DIMS.get(name), 1), dtype=torch.float64, device=self.device)
        _capi.check(self._L.mapdn_get_field(self._h, _capi.FIELDS[name], _ptr(out), self._stream()), self._L)
        return out

    # ---- env state snapshots (mapdn_snapshot / mapdn_restore) ----------------------------------------
    @property
    def fingerprint(self) -> str:
        """:func:`snapshot_fingerprint` of this env, computed on first use (it hashes the whole profile store)."""
        if self._fingerprint is None:
            c = self._cfg
            self._fingerprint = snapshot_fingerprint(self.net, self.profiles, self.args, self.history, c.tol, c.max_iter)
        return self._fingerprint

    @property
    def snapshot_layout(self):
        """Byte offsets of the ``MAPDN_N_SNAPSHOT`` segments of a snapshot row, then bytes_per_env."""
        if self._snapshot_layout is None:
            off = (C.c_int64 * (len(_capi.SNAPSHOT_SEGMENTS) + 1))()
            _capi.check(self._L.mapdn_snapshot_layout(self._h, off), self._L)
            self._snapshot_layout = [int(x) for x in off]
        return self._snapshot_layout

    def _slots(self, idx, what: str, unique: bool) -> torch.Tensor:
        """``idx`` as an int64 CPU tensor of slots in [0, batch), checked on the host (a CUDA tensor costs one sync)."""
        t = torch.as_tensor(idx).reshape(-1)
        if t.dtype.is_floating_point or t.dtype == torch.bool:
            raise ValueError(f"{what}: slot indices must be integers, got {t.dtype}")
        t = t.to("cpu", torch.int64)
        if t.numel() == 0 or t.numel() > self.batch:
            raise ValueError(f"{what}: need 1 to {self.batch} slots, got {t.numel()}")
        if int(t.min()) < 0 or int(t.max()) >= self.batch:
            raise ValueError(f"{what}: slots must be in [0, {self.batch}), got {t.min().item()}..{t.max().item()}")
        if unique and torch.unique(t).numel() != t.numel():
            raise ValueError(f"{what}: duplicate slots")
        return t

    def snapshot(self, idx=None) -> EnvSnapshot:
        """The state of the envs in slots ``idx`` (all envs in order when None; repeats allowed) as an
        :class:`EnvSnapshot` whose rows live on this env's device. One launch, stream-ordered; ``idx`` is checked on
        the host, so a CUDA index tensor costs one sync."""
        L = self.snapshot_layout
        slots = torch.arange(self.batch) if idx is None else self._slots(idx, "snapshot", unique=False)
        data = torch.empty(slots.numel(), L[-1], dtype=torch.uint8, device=self.device)
        ids = None if idx is None else slots.to(self.device, torch.int32)
        _capi.check(self._L.mapdn_snapshot(self._h, _ptr(ids), slots.numel(), _ptr(data), self._stream()), self._L)
        return EnvSnapshot(data, slots + self.env_id_offset, L, self.history, self.fingerprint)

    def restore(self, snap: EnvSnapshot, idx=None) -> torch.Tensor:
        """Puts the rows of ``snap`` back and returns the slots written (int64, CPU). ``idx``: the slot of each row (no
        repeats). Without it every row goes to the slot of its global id (``env_id - env_id_offset``) and rows of ids
        outside this env are skipped, so a snapshot of one env of B envs restores into N shards of B / N. Refuses a
        snapshot of an env with another fingerprint, layout or history. Then ``obs``, ``state`` and (``history > 1``)
        ``obs_stacked`` are gathered again from the restored state, for all envs. Stream-ordered, no host sync unless
        ``idx`` is a CUDA tensor (one)."""
        if snap.history != self.history or snap.layout != self.snapshot_layout:
            raise ValueError(f"restore: snapshot layout {snap.layout} (history {snap.history}) does not match this env's "
                             f"{self.snapshot_layout} (history {self.history})")
        if snap.fingerprint != self.fingerprint:
            raise ValueError("restore: the snapshot comes from an env with another net, profile store or env_args")
        data = snap.data
        if idx is None:
            slots = snap.env_ids - self.env_id_offset
            rows = torch.nonzero((slots >= 0) & (slots < self.batch)).reshape(-1)
            if rows.numel() == 0:
                return rows
            if rows.numel() != len(snap):
                data, slots = data[rows.to(data.device)], slots[rows]
            slots = self._slots(slots, "restore", unique=True)
        else:
            slots = self._slots(idx, "restore", unique=True)
            if slots.numel() != len(snap):
                raise ValueError(f"restore: {slots.numel()} slots for {len(snap)} snapshot rows")
        data = data.to(self.device).contiguous()
        whole = slots.numel() == self.batch and bool(torch.equal(slots, torch.arange(self.batch)))
        ids = None if whole else slots.to(self.device, torch.int32)
        st = self._stream()
        _capi.check(self._L.mapdn_restore(self._h, _ptr(ids), slots.numel(), _ptr(data), st), self._L)
        _capi.check(self._L.mapdn_get_obs(self._h, _ptr(self.obs), st), self._L)
        _capi.check(self._L.mapdn_get_state(self._h, _ptr(self.state), st), self._L)
        if self.history > 1:
            _capi.check(self._L.mapdn_get_obs_stacked(self._h, _ptr(self.obs_stacked), st), self._L)
        return slots

    def fork(self, src, dst) -> torch.Tensor:
        """Copies the state of slots ``src`` into slots ``dst`` (``restore(snapshot(src), dst)``: two launches through a
        temporary, so ``src`` and ``dst`` may overlap). One source into K slots: ``fork([s] * K, dst)``. The copies draw
        the noise of their own slots from the next profile row on (see the header's noise rules)."""
        return self.restore(self.snapshot(src), dst)

    # ---- tester records (reference utilities/tester.py:26-55) ---------------------------------------
    @property
    def record_slices(self):
        """``{key: (offset, length)}`` of the six blocks of a tester record row, in the reference tester's key order
        (``RECORD_KEYS``: pv_active, pv_reactive, bus_active, bus_reactive, bus_voltage, line_loss)."""
        if getattr(self, "_record_slices", None) is None:
            off, row = (C.c_int32 * len(_capi.RECORD_KEYS))(), C.c_int32(0)
            _capi.check(self._L.mapdn_record_layout(self._h, off, C.byref(row)), self._L)
            ends = [int(o) for o in off][1:] + [int(row.value)]
            self._record_slices = {k: (int(o), e - int(o)) for k, o, e in zip(_capi.RECORD_KEYS, off, ends)}
            self._record_len = int(row.value)
        return self._record_slices

    @property
    def record_len(self) -> int:
        """Entries of one tester record row."""
        self.record_slices
        return self._record_len

    def _record_stride(self, out: torch.Tensor) -> int:
        if (out.dtype is not torch.float64 or out.device != self.device or out.dim() != 2
                or tuple(out.shape) != (self.batch, self.record_len) or out.stride(1) != 1):
            raise ValueError(f"record: expected a float64 [{self.batch}, {self.record_len}] view with unit column stride on "
                             f"{self.device}, got {out.dtype} {tuple(out.shape)} strides {out.stride()} on {out.device}")
        return out.stride(0)

    def record(self, out: torch.Tensor) -> torch.Tensor:
        """The current tester record row of every env into ``out`` (``[B, record_len]`` view, any row stride): one gather
        launch. After a step, :meth:`step` with ``record=`` writes the same rows without it."""
        _capi.check(self._L.mapdn_record(self._h, out.data_ptr(), self._record_stride(out), self._stream()), self._L)
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
                                        _ptr(out["iterations"]), _ptr(out["converged"]), self._stream()), self._L)
        return out

    def ybus_dense(self) -> np.ndarray:
        n = self.dims["n_bus"]
        g, b = np.zeros((n, n)), np.zeros((n, n))
        _capi.check(self._L.mapdn_get_ybus_dense(self._h, g.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p)),
                    self._L)
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
