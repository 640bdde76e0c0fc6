"""Observation normalization for vector envs: tianshou 0.5's ``VectorEnvNormObs`` with the running statistics on
the GPU (csrc/obsnorm.cu).

:class:`VectorEnvNormObs` wraps a :class:`DeviceVectorEnv` or a :class:`HostVectorEnv` (any other object with the
vector-env protocol is first adopted by ``HostVectorEnv.from_vector_env``).  With ``update_obs_rms=True`` every
``reset`` (all envs or ``id``) and every ``step(action, id)`` first updates the statistics with exactly the rows
it returns, then returns those rows normalized with the updated statistics; with ``update_obs_rms=False`` it only
normalizes.  ``FastCollector`` runs the same sequence on every collect path (see DESIGN.md §7).

The statistics (:class:`ObsRunningMeanStd`) are float64 on the device with an integer count, and each normalized
value is computed in float64 and rounded to float32 once; tianshou keeps them in the observation dtype.
[UNVERIFIED: tianshou 0.5's wrapper is restated from memory, its source is not installed.]
"""
from __future__ import annotations

import contextlib
import ctypes
from typing import Optional

import numpy as np
import torch

from . import _lib
from .host_envs import HostVectorEnv, is_vector_env


class ObsRunningMeanStd:
    """Running ``mean[D]``, ``var[D]`` (float64) and ``count`` (int64) of observations, on ``device``.  Starts at
    mean 0, var 1, count 0.  ``.mean``, ``.var`` and ``.count`` read host numpy values (a device sync).  The device
    tensors are allocated on first use, so construction needs no GPU."""

    def __init__(self, D: int, device="cuda", clip_max: float = 10.0,
                 epsilon: float = float(np.finfo(np.float32).eps)):
        self.D = int(D)
        self.device = torch.device(device)
        self.clip_max = float(clip_max)
        self.eps = float(epsilon)
        self._host = (np.zeros(self.D, np.float64), np.ones(self.D, np.float64), 0)
        self._t = None

    def tensors(self):
        """(mean [D] f64, var [D] f64, count [1] i64) on the device."""
        if self._t is None:
            m, v, c = self._host
            self._t = (torch.from_numpy(m.copy()).to(self.device), torch.from_numpy(v.copy()).to(self.device),
                       torch.tensor([c], dtype=torch.int64, device=self.device))
        return self._t

    @property
    def mean(self) -> np.ndarray:
        return self._host[0].copy() if self._t is None else self._t[0].cpu().numpy()

    @property
    def var(self) -> np.ndarray:
        return self._host[1].copy() if self._t is None else self._t[1].cpu().numpy()

    @property
    def count(self) -> int:
        return self._host[2] if self._t is None else int(self._t[2].item())

    def state_dict(self) -> dict:
        return {"mean": self.mean, "var": self.var, "count": self.count, "clip_max": self.clip_max, "eps": self.eps}

    def load_state_dict(self, state: dict) -> None:
        self.copy_from(state["mean"], state["var"], state["count"])
        self.clip_max = float(state.get("clip_max", self.clip_max))
        self.eps = float(state.get("eps", self.eps))

    def copy_from(self, mean, var, count) -> None:
        mean = np.broadcast_to(np.asarray(mean, dtype=np.float64), (self.D,)).copy()
        var = np.broadcast_to(np.asarray(var, dtype=np.float64), (self.D,)).copy()
        if self._t is None:
            self._host = (mean, var, int(count))
            return
        self._t[0].copy_(torch.from_numpy(mean))
        self._t[1].copy_(torch.from_numpy(var))
        self._t[2].fill_(int(count))

    def descriptor(self, work: torch.Tensor, update: bool) -> "_lib.ObsRms":
        m, v, c = self.tensors()
        return _lib.ObsRms(mean=m.data_ptr(), var=v.data_ptr(), count=c.data_ptr(), work=work.data_ptr(), D=self.D,
                           update=int(update), clip_max=self.clip_max, eps=self.eps)


class VectorEnvNormObs:
    """tianshou's ``VectorEnvNormObs(venv, update_obs_rms=True)`` over a device or host vector env."""

    def __init__(self, venv, update_obs_rms: bool = True):
        # imported here: envs re-exports this module's classes, so a module-level import would make
        # `import fsrl_b200.obs_norm` in a fresh interpreter fail on the cycle
        from .envs import DeviceVectorEnv
        if isinstance(venv, VectorEnvNormObs):
            raise TypeError("VectorEnvNormObs wraps a DeviceVectorEnv or a HostVectorEnv, not another VectorEnvNormObs")
        if not isinstance(venv, (DeviceVectorEnv, HostVectorEnv)):
            if not is_vector_env(venv):
                raise TypeError("VectorEnvNormObs wraps a DeviceVectorEnv, a HostVectorEnv or an object with the "
                                f"vector-env protocol (len, step(action, id), reset(id)); got {type(venv).__name__}")
            venv = HostVectorEnv.from_vector_env(venv)
        self.venv = venv
        self.update_obs_rms = bool(update_obs_rms)
        self.obs_rms = ObsRunningMeanStd(venv.D, venv.device)
        self._work = None
        self._obs_norm = None        # host envs: [E, D] normalized current observations on the device

    # ---- forwarding --------------------------------------------------------------------------------------
    def __len__(self) -> int:
        return len(self.venv)

    @property
    def env_num(self) -> int:
        return self.venv.env_num

    @property
    def observation_space(self):
        return self.venv.observation_space

    @property
    def action_space(self):
        return self.venv.action_space

    @property
    def spec(self):
        return self.venv.spec

    @property
    def max_episode_steps(self):
        return self.venv.max_episode_steps

    @property
    def D(self) -> int:
        return self.venv.D

    @property
    def A(self) -> int:
        return self.venv.A

    @property
    def device(self):
        return self.venv.device

    def seed(self, seed=None):
        return self.venv.seed(seed)

    def render(self, **kwargs):
        return self.venv.render(**kwargs)

    def close(self):
        return self.venv.close()

    # ---- statistics ----------------------------------------------------------------------------------------
    def get_obs_rms(self) -> ObsRunningMeanStd:
        return self.obs_rms

    def set_obs_rms(self, obs_rms) -> None:
        """Share ``obs_rms`` (an :class:`ObsRunningMeanStd`: later updates by any wrapper sharing it reach this
        one), or copy in any object with ``mean``, ``var`` and ``count``."""
        if isinstance(obs_rms, ObsRunningMeanStd):
            if obs_rms.D != self.D or obs_rms.device != torch.device(self.device):
                raise ValueError(f"obs_rms holds D = {obs_rms.D} on {obs_rms.device}; this env has D = {self.D} "
                                 f"on {self.device}")
            self.obs_rms = obs_rms
            return
        self.obs_rms.copy_from(obs_rms.mean, obs_rms.var, obs_rms.count)

    @contextlib.contextmanager
    def frozen(self):
        """Normalize without updating the statistics inside the block (evaluation)."""
        old = self.update_obs_rms
        self.update_obs_rms = False
        try:
            yield self
        finally:
            self.update_obs_rms = old

    # ---- device plumbing -----------------------------------------------------------------------------------
    @property
    def host(self) -> bool:
        return isinstance(self.venv, HostVectorEnv)

    def _stream(self) -> int:
        if self.device.type != "cuda":
            raise RuntimeError(f"VectorEnvNormObs normalizes on CUDA devices only (device={self.device})")
        return torch.cuda.current_stream(self.device).cuda_stream

    def descriptor(self) -> "_lib.ObsRms":
        """The statistics and this wrapper's workspace as the C descriptor (update flag included)."""
        if self._work is None:
            nbytes = int(_lib.lib.fsrl_obs_rms_work_bytes(self.env_num, self.D))
            self._work = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)
        return self.obs_rms.descriptor(self._work, self.update_obs_rms)

    @property
    def obs_norm(self) -> torch.Tensor:
        """Host envs: every env's current normalized observation [E, D] on the device."""
        if self._obs_norm is None:
            self._obs_norm = torch.zeros((self.env_num, self.D), dtype=torch.float32, device=self.device)
        return self._obs_norm

    def _rows(self, x: torch.Tensor, ids: Optional[np.ndarray], n: int, rows_in: Optional[torch.Tensor],
              out: Optional[torch.Tensor]) -> None:
        desc = self.descriptor()
        with torch.cuda.device(self.device):
            stream = self._stream()
            _lib.check(_lib.lib.fsrl_obs_rms_rows(
                ctypes.byref(desc), x.data_ptr(), self.env_num, None if ids is None else ids.ctypes.data, n,
                None if rows_in is None else rows_in.data_ptr(), None if out is None else out.data_ptr(), stream))

    def _host_rows(self, ids: Optional[np.ndarray], raw: np.ndarray) -> torch.Tensor:
        """Update with / normalize the host rows ``raw`` of envs ``ids`` (None: all) into ``obs_norm``."""
        self._stream()
        rows_in = torch.from_numpy(np.ascontiguousarray(raw, dtype=np.float32)).to(self.device)
        out = torch.empty_like(rows_in)
        self._rows(self.obs_norm, ids, len(raw), rows_in, out)
        return out

    @staticmethod
    def _ids32(ids) -> Optional[np.ndarray]:
        return None if ids is None else np.ascontiguousarray(ids, dtype=np.int32)

    # ---- the gym vector protocol ---------------------------------------------------------------------------
    def reset(self, id=None, **kwargs):
        """Fresh episodes in every env or in the envs ``id`` lists; the statistics take their observations first
        (with ``update_obs_rms``), the rows come back normalized.  Device envs return device tensors, host envs
        numpy arrays, as the wrapped env does."""
        if self.host:
            raw = self.venv.reset_obs(id, **kwargs)
            ids = None if id is None else self._ids32(self.venv._rows(id))
            out = self._host_rows(ids, raw)
            return out.cpu().numpy(), [{} for _ in range(len(raw))]
        obs, info = self.venv.reset(id, **kwargs)
        ids = self._ids32(self.venv._ids(id if id is not None else kwargs.get("ids")))
        if ids is None:
            self._rows(self.venv.obs_cur, None, self.env_num, None, None)
            return self.venv.obs_cur, info
        self._rows(self.venv.obs_cur, ids, len(ids), None, obs)
        return obs, info

    def step(self, action, id=None):
        """The wrapped env's ``step`` with ``obs_next`` normalized after the statistics took it."""
        if self.host:
            obs, rew, term, trunc, info = self.venv.step(action, id)
            ids = None if id is None else self._ids32(self.venv._rows(id))
            out = self._host_rows(ids, obs)
            return out.cpu().numpy(), rew, term, trunc, info
        obs_next, rew, term, trunc, info = self.venv.step(action, id)
        ids = self._ids32(self.venv._ids(id))
        self._rows(self.venv.obs_cur, ids, len(obs_next), None, obs_next)
        return obs_next, rew, term, trunc, info

    # ---- collector hooks -------------------------------------------------------------------------------------
    def host_reset_all(self, **kwargs) -> np.ndarray:
        """Host envs: reset every env, update and normalize into ``obs_norm``; returns the raw rows."""
        raw = self.venv.reset_obs(None, **kwargs)
        self._host_rows(None, raw)
        return raw
