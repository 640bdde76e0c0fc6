"""Vector envs stepped on the host: any gymnasium-style env (a real simulator, a user's own env) behind the
collector, with the actor, the action-noise stream and the replay ring kept on the device.

:class:`HostVectorEnv` takes tianshou's constructor (a list of callables returning envs) and steps the envs in
this process, in order, as ``DummyVectorEnv`` does; :meth:`HostVectorEnv.from_vector_env` adopts an object that
already speaks tianshou's ``BaseVectorEnv`` protocol (``len``, ``step(action, id)``, ``reset(id, **kw)``), such as
a ``SubprocVectorEnv``.  What envs return is normalised as the reference's collector does
(fsrl/data/fast_collector.py:135-137,287-303,325): 5-tuple or 4-tuple ``step`` results (``TimeLimit.truncated``
in ``info``), ``reset`` returning ``obs`` or ``(obs, info)``, and ``cost`` read from ``info`` given as a Batch, a
list of dicts or a dict of arrays (0 when absent).  ``truncated`` is kept only where the step did not terminate,
the convention of the device ring.

The device state (the per-env action-noise counters ``act_ctr``, the scratch of the collect step and the pinned
staging buffers) is allocated on first use, so construction and the protocol handling need no GPU.
:class:`~fsrl_b200.data.FastCollector` drives the per-step device work through ``fsrl_host_collect_step``
(csrc/rollout_host.cu).
"""
from __future__ import annotations

import ctypes
from typing import Any, Callable, List, Optional, Sequence

import numpy as np
import torch

from . import _lib

MAX_A = 8                                   # the widest action the collect kernel is instantiated for
MAX_DA = int(_lib.lib.fsrl_engine_dx_ld())  # FSRL_ENG_DX_LD: the widest obs + act input the learners' engine takes


class _Spec:
    """An env's ``spec``: its id and horizon."""

    def __init__(self, id, max_episode_steps):
        self.id, self.max_episode_steps = id, max_episode_steps


def _per_env(value, n: int) -> list:
    """A vector env's attribute as one entry per env (tianshou returns lists, a single object stands for all)."""
    if isinstance(value, (list, tuple)) or (isinstance(value, np.ndarray) and value.dtype == object):
        return list(value)
    return [value] * n


def _box_width(space, what: str) -> int:
    if type(space).__name__ != "Box" or not hasattr(space, "low") or not hasattr(space, "high"):
        raise ValueError(f"HostVectorEnv takes Box {what} spaces only (got {type(space).__name__})")
    shape = tuple(space.shape)
    if len(shape) != 1:
        raise ValueError(f"HostVectorEnv takes flat (1-D) {what}s only (got shape {shape})")
    return shape[0]


def _same_space(a, b) -> bool:
    return (type(a) is type(b) and tuple(a.shape) == tuple(b.shape) and np.array_equal(np.asarray(a.low), np.asarray(b.low))
            and np.array_equal(np.asarray(a.high), np.asarray(b.high)))


def _is_dict_seq(info) -> bool:
    return isinstance(info, (list, tuple, np.ndarray)) and len(info) > 0 and (info[0] is None or isinstance(info[0], dict))


def _info_column(info, key: str, n: int, default, dtype) -> np.ndarray:
    """``info[key]`` per env for an info given as a dict of arrays, a Batch or a list of dicts."""
    if _is_dict_seq(info):
        return np.array([default if d is None else d.get(key, default) for d in info], dtype=dtype)
    if info is not None and hasattr(info, "get"):
        v = info.get(key, None)
        if v is not None:
            if isinstance(v, torch.Tensor):
                v = v.detach().cpu().numpy()
            return np.broadcast_to(np.asarray(v, dtype=dtype), (n,)).copy()
    return np.full(n, default, dtype=dtype)


def normalize_step(result, n: int, D: int):
    """A vector ``step`` result of n rows -> (obs_next [n, D] f32, rew f64, terminated, truncated, cost f64).  Rewards and
    costs keep the env's values (widened, never rounded), so the collect statistics sum what the env reported; the
    ring stores them as float32."""
    if not isinstance(result, (tuple, list)) or len(result) not in (4, 5):
        raise ValueError(f"env.step must return a 4- or 5-tuple (got {type(result).__name__} of "
                         f"{len(result) if isinstance(result, (tuple, list)) else '?'} items)")
    if len(result) == 5:
        obs, rew, term, trunc, info = result
        term = np.asarray(term, dtype=bool).reshape(n)
        trunc = np.asarray(trunc, dtype=bool).reshape(n)
    else:                                  # gym's done + TimeLimit.truncated (fast_collector.py:290-301)
        obs, rew, done, info = result
        trunc = _info_column(info, "TimeLimit.truncated", n, False, bool)
        term = np.asarray(done, dtype=bool).reshape(n) & ~trunc
    trunc = trunc & ~term
    obs = _obs(obs, n, D)
    rew = np.asarray(rew, dtype=np.float64).reshape(n)
    cost = _info_column(info, "cost", n, 0.0, np.float64)
    return obs, rew, term, trunc, cost


def normalize_reset(rval, n: int, D: int) -> np.ndarray:
    """A vector ``reset`` result (``obs`` or ``(obs, info)``, fast_collector.py:134-152) -> obs [n, D] f32."""
    if isinstance(rval, (tuple, list)) and len(rval) == 2:
        info = rval[1]
        if isinstance(info, dict) or _is_dict_seq(info) or type(info).__name__ == "Batch":
            rval = rval[0]
    return _obs(rval, n, D)


def _obs(obs, n: int, D: int) -> np.ndarray:
    if isinstance(obs, torch.Tensor):
        obs = obs.detach().cpu().numpy()
    o = np.asarray(obs, dtype=np.float32)
    if o.size != n * D:
        raise ValueError(f"expected {n} observations of {D} floats, got an array of shape {o.shape}")
    return np.ascontiguousarray(o.reshape(n, D))


def _single_reset(rval):
    if isinstance(rval, tuple) and len(rval) == 2 and isinstance(rval[1], dict):
        return rval[0]
    return rval


class HostVectorEnv:
    """E host envs of one observation / action shape behind the vector-env protocol the collector consumes."""

    def __init__(self, env_fns: Sequence[Callable[[], Any]], device="cuda", seed: int = 0):
        self._setup([fn() for fn in env_fns], None, device, seed)

    @classmethod
    def from_vector_env(cls, venv, device="cuda", seed: int = 0) -> "HostVectorEnv":
        """Adopt an object with tianshou's ``BaseVectorEnv`` protocol; its own ``step`` / ``reset`` step the envs."""
        self = cls.__new__(cls)
        self._setup(None, venv, device, seed)
        return self

    @classmethod
    def _from_envs(cls, envs: List[Any], device="cuda", seed: int = 0) -> "HostVectorEnv":
        self = cls.__new__(cls)
        self._setup(list(envs), None, device, seed)
        return self

    def _setup(self, envs, venv, device, seed) -> None:
        self._envs, self._venv = envs, venv
        if envs is not None:
            if not envs:
                raise ValueError("HostVectorEnv needs at least one env")
            E = len(envs)
            obs_sp = [e.observation_space for e in envs]
            act_sp = [e.action_space for e in envs]
            spec = getattr(envs[0], "spec", None)
        else:
            E = len(venv)
            if E < 1:
                raise ValueError("HostVectorEnv needs at least one env")
            obs_sp = _per_env(venv.observation_space, E)
            act_sp = _per_env(venv.action_space, E)
            spec = _per_env(getattr(venv, "spec", None), E)[0]
        self.env_num = E
        D, A = _box_width(obs_sp[0], "observation"), _box_width(act_sp[0], "action")
        for i in range(1, E):
            if not (_same_space(obs_sp[i], obs_sp[0]) and _same_space(act_sp[i], act_sp[0])):
                raise ValueError(f"every env of a HostVectorEnv must have the same spaces; env {i} differs from env 0")
        if A > MAX_A:
            raise ValueError(f"HostVectorEnv takes actions of at most {MAX_A} dimensions (got A = {A})")
        if D + A > MAX_DA:
            raise ValueError(f"HostVectorEnv takes obs + action widths of at most D + A = {MAX_DA} "
                             f"(got D = {D}, A = {A})")
        self.D, self.A = D, A
        self.observation_space, self.action_space = obs_sp[0], act_sp[0]
        T = getattr(spec, "max_episode_steps", None)
        self.max_episode_steps = T
        self.spec = _Spec(getattr(spec, "id", None), T) if spec is not None else None
        self.device = torch.device(device)
        self.seed_value = int(seed) & 0xFFFFFFFF
        self._dev = None          # device state, allocated by the first collect step
        self._parity = 0

    def __len__(self) -> int:
        return self.env_num

    # ---- the gym vector protocol over the host envs ------------------------------------------------------
    def _rows(self, id) -> np.ndarray:
        if id is None:
            return np.arange(self.env_num)
        if isinstance(id, torch.Tensor):
            id = id.cpu().numpy()
        ids = np.atleast_1d(np.asarray(id))
        if ids.ndim != 1 or not np.issubdtype(ids.dtype, np.integer) or ids.size == 0:
            raise ValueError(f"env ids must be a non-empty 1-D integer array (got {ids!r})")
        if ids.min() < 0 or ids.max() >= self.env_num:
            raise ValueError(f"env ids must lie in [0, {self.env_num}) (got {ids.tolist()})")
        return ids

    def reset_obs(self, id=None, **kwargs) -> np.ndarray:
        """Fresh episodes in the envs ``id`` lists (all by default); their observations [n, D] float32."""
        ids = self._rows(id)
        if self._venv is not None:
            rval = self._venv.reset(None if id is None else ids, **kwargs)
            return normalize_reset(rval, len(ids), self.D)
        return _obs([_single_reset(self._envs[i].reset(**kwargs)) for i in ids], len(ids), self.D)

    def step_envs(self, action, id=None):
        """env.step with env-range actions [n, A] for the envs ``id`` lists; returns the normalised
        (obs_next [n, D] f32, rew f64, terminated, truncated, cost f64) of normalize_step."""
        ids = self._rows(id)
        act = np.asarray(action, dtype=np.float32).reshape(len(ids), self.A)
        if self._venv is not None:
            return normalize_step(self._venv.step(act, None if id is None else ids), len(ids), self.D)
        res = [self._envs[i].step(act[k]) for k, i in enumerate(ids)]
        if any(len(r) != len(res[0]) for r in res):
            raise ValueError("the envs of one HostVectorEnv must return step results of one length")
        cols = list(zip(*res))
        info = list(cols[-1])
        return normalize_step(tuple(cols[:-1]) + (info,), len(ids), self.D)

    def reset(self, id=None, **kwargs):
        """tianshou's ``reset(id)``: (obs [n, D] float32, one info dict per env)."""
        obs = self.reset_obs(id, **kwargs)
        return obs, [{} for _ in range(len(obs))]

    def step(self, action, id=None):
        """tianshou's ``step(action, id)``: (obs_next, rew, terminated, truncated, info), numpy, with the cost of
        every row in ``info["cost"]``."""
        obs, rew, term, trunc, cost = self.step_envs(action, id)
        return obs, rew, term, trunc, {"cost": cost, "env_id": self._rows(id)}

    def seed(self, seed=None):
        """Pass ``seed + i`` to env i (``seed(None)`` to every env); returns what the envs return."""
        if seed is not None:
            self.seed_value = int(seed) & 0xFFFFFFFF
        if self._venv is not None:
            return self._venv.seed(seed) if hasattr(self._venv, "seed") else None
        out = []
        for i, e in enumerate(self._envs):
            s = None if seed is None else int(seed) + i
            out.append(e.seed(s) if hasattr(e, "seed") else s)
        return out

    def render(self, **kwargs):
        if self._venv is not None:
            return self._venv.render(**kwargs)
        return [e.render(**kwargs) for e in self._envs]

    def close(self) -> None:
        if self._venv is not None:
            self._venv.close()
        else:
            for e in self._envs:
                if hasattr(e, "close"):
                    e.close()

    # ---- device state of the collect ------------------------------------------------------------------------
    @property
    def act_ctr(self) -> torch.Tensor:
        """[E] int32 action samples drawn per env: the counter of the Philox noise stream keyed by env id, so a
        second collector over the same envs continues the stream."""
        return self._device_state()["act_ctr"]

    def _device_state(self) -> dict:
        if self._dev is None:
            if self.device.type != "cuda":
                raise RuntimeError(f"HostVectorEnv collects on CUDA devices only (device={self.device})")
            E, D, A, dev = self.env_num, self.D, self.A, self.device
            nbytes = int(_lib.lib.fsrl_host_pack_norm_bytes(D, E, E, E))   # room for a wrapped env's fresh rows
            pack_host = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
            act_host = torch.empty((E, A), dtype=torch.float32).pin_memory()
            self._dev = dict(
                act_ctr=torch.zeros(E, dtype=torch.int32, device=dev),
                scratch=torch.zeros(2 * E * (D + A + 1), dtype=torch.float32, device=dev),
                pack_dev=torch.empty(nbytes, dtype=torch.uint8, device=dev),
                act_dev=torch.empty((E, A), dtype=torch.float32, device=dev),
                pack_host=pack_host, pack_np=pack_host.numpy(), act_host=act_host, act_np=act_host.numpy())
        return self._dev

    def fill(self, r: "_lib.Rollout") -> None:
        """The env half of a rollout descriptor: E, the noise counters and the action bounds of map_action."""
        s = self._device_state()
        r.kind, r.E, r.max_steps = -1, self.env_num, 0
        r.seed_env = self.seed_value
        r.act_ctr = s["act_ctr"].data_ptr()
        low, high = np.asarray(self.action_space.low), np.asarray(self.action_space.high)
        for j in range(self.A):
            r.act_low[j], r.act_high[j] = float(low[j]), float(high[j])

    def device_step(self, r: "_lib.Rollout", act_ids: np.ndarray, obs: np.ndarray, store=None, norm=None,
                    fresh=None) -> np.ndarray:
        """One ``fsrl_host_collect_step``: store ``store`` = (ids, obs_next, rew, cost, terminated, truncated) of
        the previous call into r's ring, then act on obs [n, D] of the envs act_ids.  Returns the env-range
        actions [n, A].  One H2D copy, one launch, one D2H copy and one stream synchronisation.  ``norm``: the
        VectorEnvNormObs wrapping this env; the statistics then take the stored obs_next rows, then ``fresh`` =
        (ids, reset obs) of the envs restarted since the previous call, and the actor and the ring see normalized
        rows (the act rows come from the wrapper's ``obs_norm``)."""
        s = self._device_state()
        D, A = self.D, self.A
        n_a = len(act_ids)
        n_s = 0 if store is None else len(store[0])
        buf = s["pack_np"]
        o = 0
        parts = []
        if n_s:
            parts.append((store[0], np.int32))
        parts += [(act_ids, np.int32), (obs, np.float32)]
        if n_s:
            parts += [(store[1], np.float32), (store[2], np.float32), (store[3], np.float32),
                      (store[4], np.uint8), (store[5], np.uint8)]
        n_f = 0
        if norm is not None:
            if fresh is not None and len(fresh[0]):
                n_f = len(fresh[0])
                parts += [(np.zeros(int(_lib.lib.fsrl_host_pack_norm_bytes(D, n_s, n_a, 0))
                                    - int(_lib.lib.fsrl_host_pack_bytes(D, n_s, n_a)), np.uint8), np.uint8),
                          (fresh[0], np.int32), (fresh[1], np.float32)]
        for arr, dt in parts:
            b = np.ascontiguousarray(arr, dtype=dt).reshape(-1).view(np.uint8)
            buf[o:o + b.size] = b
            o += b.size
        h = _lib.HostStep(D=D, A=A, n_store=n_s, n_act=n_a, parity=self._parity,
                          pack_host=s["pack_host"].data_ptr(), pack_dev=s["pack_dev"].data_ptr(),
                          scratch=s["scratch"].data_ptr(), act_dev=s["act_dev"].data_ptr(),
                          act_host=s["act_host"].data_ptr())
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device)
            if norm is not None:
                desc = norm.descriptor()
                hn = _lib.HostNorm(obs_rms=ctypes.addressof(desc), obs_norm=norm.obs_norm.data_ptr(), n_fresh=n_f)
                _lib.check(_lib.lib.fsrl_host_collect_step_norm(ctypes.byref(r), ctypes.byref(h), ctypes.byref(hn),
                                                                stream.cuda_stream))
            else:
                _lib.check(_lib.lib.fsrl_host_collect_step(ctypes.byref(r), ctypes.byref(h), stream.cuda_stream))
            stream.synchronize()
        self._parity ^= 1
        return s["act_np"][:n_a].copy()


def is_vector_env(obj) -> bool:
    """Whether obj speaks the vector-env protocol the collector needs: ``len``, ``step(action, id)``, ``reset``."""
    return hasattr(obj, "__len__") and callable(getattr(obj, "step", None)) and callable(getattr(obj, "reset", None))
