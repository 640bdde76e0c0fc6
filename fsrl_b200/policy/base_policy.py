"""``BasePolicy`` with the reference's constructor and hooks
(/root/reference/fsrl/policy/base_policy.py:83-512), backed by the flat device arena and the
CUDA kernels instead of eager PyTorch + numba:

* ``forward``              -> csrc/mlpfwd.cu (API compatibility; the fused collector runs the
                               actor inside the rollout kernel; an actor the arena cannot hold runs as
                               its own torch module, called per step by the generic collector)
* ``compute_gae_returns``  -> batched critic forward + csrc/gae.cu dual scan (:384-451)
* ``compute_nstep_returns``-> csrc/nstep.cu (:453-512)
* ``soft_update``          -> csrc/polyak (:220-224)
* ``map_action`` / ``map_action_inverse`` keep their numpy semantics (:226-283) for callers
  that hold host actions; the rollout kernel applies the same mapping on the device.
"""
from __future__ import annotations

import ctypes
from abc import ABC, abstractmethod
from typing import Any, Dict, List, Optional, Union

import numpy as np
import torch
from torch import nn

from .. import _lib, ops
from ..data.batch import Batch, to_numpy
from ..nets import Actor, ActorProb, Arena, Critic, slot_from_module, slots_from_module
from ..spaces import Box, Discrete, MultiBinary, MultiDiscrete
from ..utils.logger import BaseLogger, DummyLogger
from ..utils.optim_util import RunningMeanStd


class ActorCritic(nn.Module):
    """Parameter container (reference: fsrl/utils/net/common.py:6-18)."""

    def __init__(self, actor: nn.Module, critics) -> None:
        super().__init__()
        self.actor = actor
        self.critics = critics if isinstance(critics, nn.ModuleList) else nn.ModuleList(
            critics if isinstance(critics, (list, tuple)) else [critics])


class DeviceBatch:
    """The processed on-policy batch, SoA on the device, in the reference's batch order
    (env-major, chronological).  ``values/rets/advs`` are exposed as (N, C) views like the
    reference's ``batch.values/rets/advs``; the kernels read the (C, N) bases."""

    def __init__(self):
        self.n = 0

    def __len__(self):
        return self.n


class BasePolicy(ABC, nn.Module):
    def __init__(self, actor: nn.Module, critics: Union[nn.Module, List[nn.Module]],
                 dist_fn=None, logger: BaseLogger = DummyLogger(), gamma: float = 0.99,
                 max_batchsize: Optional[int] = 99999, reward_normalization: bool = False,
                 deterministic_eval: bool = True, action_scaling: bool = True,
                 action_bound_method: str = "clip", observation_space=None, action_space=None,
                 lr_scheduler=None) -> None:
        super().__init__()
        self.actor = actor
        if isinstance(critics, nn.Module):
            self.critics = nn.ModuleList([critics])
        elif isinstance(critics, List):
            self.critics = nn.ModuleList(critics)
        else:
            raise TypeError("critics should not be %s" % (type(critics)))
        self.critics_num = len(self.critics)
        self.dist_fn = dist_fn
        self.logger = logger
        assert 0.0 <= gamma <= 1.0, "discount factor should be in [0, 1]."
        self._gamma = gamma
        self._rew_norm = reward_normalization
        self.ret_rms = [RunningMeanStd() for _ in range(self.critics_num)]              # :111
        self._eps = 1e-8
        self._deterministic_eval = deterministic_eval
        self._max_batchsize = max_batchsize
        self._actor_critic = ActorCritic(self.actor, self.critics)
        self.observation_space = observation_space
        self.action_space = action_space
        self.action_type = ""
        if isinstance(action_space, (Discrete, MultiDiscrete, MultiBinary)):
            self.action_type = "discrete"
        elif isinstance(action_space, Box):
            self.action_type = "continuous"
        else:
            print("Warning! The action sapce type is unclear, regard it as continuous.")
            self.action_type = "continuous"
        if self.action_type == "discrete":
            raise NotImplementedError("the device path covers the continuous-control tasks of the hot path")
        self.updating = False
        self.action_scaling = action_scaling
        assert action_bound_method in ("", "clip", "tanh")
        self.action_bound_method = action_bound_method
        self.lr_scheduler = lr_scheduler
        self.gradient_steps = 0
        self.last_stats: Dict[str, Any] = {}
        self._arena: Optional[Arena] = None

    # ---- arena ------------------------------------------------------------------------------------
    def _net_list(self) -> List[nn.Module]:
        return [self.actor] + list(self.critics)

    def _build_arena(self, device=None) -> Arena:
        if device is None:
            device = getattr(self.actor, "device", None) or "cuda"
        if torch.device(device).type != "cuda":
            raise RuntimeError("fsrl_b200 runs on CUDA devices only (got device=%r); there is no "
                               "CPU fallback" % (device,))
        slots, self._slot_groups = [], []
        for i, m in enumerate(self._net_list()):
            ss = slots_from_module("net%d" % i, m)
            self._slot_groups.append(ss)
            slots += ss
        self._arena = Arena(slots, device)
        return self._arena

    def _arena_holds_nets(self) -> bool:
        """Whether every network of the policy fits the flat device arena (tianshou Actor / ActorProb / Critic
        with two equal hidden layers of width 64, 128, 256 or 512), which the rollout kernel and the fused
        learners need.  Checked without allocating."""
        if self._arena is not None:
            return True
        try:
            for i, m in enumerate(self._net_list()):
                slots_from_module("net%d" % i, m)
        except (TypeError, ValueError, NotImplementedError, AttributeError):
            return False
        return True

    @property
    def arena(self) -> Arena:
        if self._arena is None:
            self._build_arena()
        return self._arena

    @property
    def device(self):
        return self.arena.device

    def _stream(self) -> int:
        return torch.cuda.current_stream().cuda_stream

    def net_forward(self, slot_index: int, x: torch.Tensor, idx: Optional[torch.Tensor] = None,
                    out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """y = net(x[idx]) through csrc/mlpfwd.cu."""
        ar = self.arena
        s = ar.slots[slot_index]
        m = ar.mlp3(s)
        n = x.shape[0] if idx is None else idx.shape[0]
        if out is None:
            out = torch.empty((n, s.out), dtype=torch.float32, device=ar.device)
        assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and x.shape[1] == s.D
        ip = None
        if idx is not None:
            assert idx.dtype == torch.int32 and idx.is_contiguous()
            ip = idx.data_ptr()
        with torch.cuda.device(ar.device):
            _lib.check(_lib.lib.fsrl_mlp_forward(ctypes.byref(m), x.data_ptr(), ip, n, out.data_ptr(), self._stream()))
        return out

    def load_state_dict(self, state_dict, strict: bool = True, **kw):
        """Parameters alias the device arena, so loading writes straight into it; derived copies (the
        out-major W2 mirrors used by the backward kernels) are refreshed afterwards."""
        self.arena
        out = super().load_state_dict(state_dict, strict=strict, **kw)
        if hasattr(self, "_mirror_dirty"):
            self._mirror_dirty = True
        eng = getattr(self, "_eng", None)
        if eng is not None:
            eng.sync_mirror(self.arena.slots)
        return out

    # ---- rollout descriptor (consumed by FastCollector) ----------------------------------------------
    def _rollout_mode(self) -> int:
        if self._deterministic_eval and not self.training:
            return _lib.MODE_EVAL
        return _lib.MODE_TRAIN

    def fill_rollout(self, r: "_lib.Rollout", exploration_noise: bool = False) -> None:
        ar = self.arena
        s = ar.slots[0]
        r.actor = ar.mlp3(s)
        r.mode = self._rollout_mode()
        r.action_bound = {"": _lib.BOUND_NONE, "clip": _lib.BOUND_CLIP, "tanh": _lib.BOUND_TANH}[self.action_bound_method]
        r.action_scaling = int(self.action_scaling)
        a = self.actor
        r.max_action = float(getattr(a, "_max", 1.0))
        r.tanh_eps = float(np.finfo(np.float32).eps)
        r.seed_act = int(getattr(self, "_act_seed", 0)) & 0xFFFFFFFF
        if isinstance(a, ActorProb):
            r.bounded = int(not a._unbounded)
            if a._c_sigma:
                from ..nets import SIGMA_MAX, SIGMA_MIN
                r.head = _lib.HEAD_GAUSS_COND
                r.sigma_min, r.sigma_max = SIGMA_MIN, SIGMA_MAX
            else:
                r.head = _lib.HEAD_GAUSS_INDEP
                r.log_sigma = ar.extra_ptr(s)
        elif isinstance(a, Actor):
            r.head = _lib.HEAD_DETERMINISTIC
            r.bounded = 1
        else:
            raise TypeError(f"unsupported actor type {type(a)}")
        r.expl_sigma = 0.0

    def set_action_seed(self, seed: int) -> None:
        """Key of the Philox action-noise stream (documented RNG; oracle/philox.py)."""
        self._act_seed = int(seed)

    # ---- learner plumbing ----------------------------------------------------------------------------
    def _expand_cost_limit(self, cost_limit) -> list:
        """One limit per cost critic: a scalar applies to every cost stream."""
        return [cost_limit] * (self.critics_num - 1) if np.isscalar(cost_limit) else cost_limit

    def _record(self, stats: Dict[str, float]) -> None:
        """One gradient step's ``tab/key`` scalars: appended to ``last_stats`` and stored in the logger, in
        the dict's order."""
        for k, v in stats.items():
            self.last_stats.setdefault(k, []).append(v)
            tab, key = k.split("/", 1)
            self.logger.store(tab, **{key: v})

    def _record_many(self, out: Dict[str, np.ndarray]) -> None:
        """Columns of per-step ``tab/key`` values from one device->host copy: they become ``last_stats`` and are
        stored in the logger, in the dict's order."""
        self.last_stats = out
        for k, v in out.items():
            tab, key = k.split("/", 1)
            self.logger.store_many(tab, key, v)

    # ---- reference hooks -----------------------------------------------------------------------------
    def forward(self, batch: Batch, state=None, **kwargs: Any) -> Batch:
        """API-compatible policy forward on a device batch (base_policy.py:178-190).  The actor runs through
        csrc/mlpfwd.cu when the arena holds the policy's networks; any other actor (more hidden layers,
        LayerNorm, a user's own module) is the torch module the user wrote and runs as one, as in the
        reference -- FastCollector then takes its generic path."""
        if not self._arena_holds_nets():
            return self._module_forward(batch, state)
        obs = torch.as_tensor(batch.obs, dtype=torch.float32, device=self.device).contiguous()
        out = self.net_forward(0, obs)
        a = self.actor
        A = out.shape[1] if not (isinstance(a, ActorProb) and a._c_sigma) else out.shape[1] // 2
        if isinstance(a, ActorProb):
            mu = out[:, :A]
            if not a._unbounded:
                mu = a._max * torch.tanh(mu)
            if a._c_sigma:
                from ..nets import SIGMA_MAX, SIGMA_MIN
                sigma = out[:, A:].clamp(SIGMA_MIN, SIGMA_MAX).exp()
            else:
                sigma = a.sigma_param.view(1, -1).exp().expand_as(mu)
            logits = (mu, sigma)
            dist = self.dist_fn(*logits) if self.dist_fn is not None else None
            if self._deterministic_eval and not self.training:
                act = mu
            else:
                act = dist.sample() if dist is not None else mu + sigma * torch.randn_like(mu)
        else:
            logits = a._max * torch.tanh(out)
            dist, act = None, logits
        return Batch(logits=logits, act=act, state=None, dist=dist)

    def _module_forward(self, batch: Batch, state=None) -> Batch:
        """The reference's forward (base_policy.py:178-190) with the actor module itself; without a dist_fn a
        (mu, sigma) head samples mu + sigma * N(0, 1) as forward() does."""
        logits, hidden = self.actor(batch.obs, state=state)
        if self.dist_fn is not None:
            dist = self.dist_fn(*logits) if isinstance(logits, tuple) else self.dist_fn(logits)
        else:
            dist = None
        mean = logits[0] if isinstance(logits, tuple) else logits
        if (self._deterministic_eval and not self.training) or (dist is None and not isinstance(logits, tuple)):
            act = mean
        elif dist is not None:
            act = dist.sample()
        else:
            act = mean + logits[1] * torch.randn_like(mean)
        return Batch(logits=logits, act=act, state=hidden, dist=dist)

    def pre_update_fn(self, **kwarg: Any) -> Any:
        pass

    def post_update_fn(self, **kwarg: Any) -> Any:
        pass

    def exploration_noise(self, act, batch):
        return act

    def soft_update(self, tgt: nn.Module, src: nn.Module, tau: float) -> None:
        for tp, sp in zip(tgt.parameters(), src.parameters()):
            tp.data.copy_(tau * sp.data + (1 - tau) * tp.data)

    def map_action(self, act):
        """Policy output -> what the env receives (base_policy.py:226-256): bound to [-1, 1] by clipping or
        tanh, then stretch affinely onto [low, high].  Host twin of the epilogue fused into the rollout
        kernel (csrc/rollout.cu); only ndarray actions of Box spaces are touched."""
        if not (isinstance(self.action_space, Box) and isinstance(act, np.ndarray)):
            return act
        bound = {"clip": lambda a: np.clip(a, -1.0, 1.0), "tanh": np.tanh}.get(self.action_bound_method)
        unit = bound(act) if bound is not None else act
        if not self.action_scaling:
            return unit
        assert np.min(unit) >= -1.0 and np.max(unit) <= 1.0, "action scaling only accepts raw action range = [-1, 1]"
        lo, hi = self.action_space.low, self.action_space.high
        return lo + (hi - lo) * (unit + 1.0) / 2.0

    def map_action_inverse(self, act):
        """Env-range action (e.g. ``action_space.sample()`` during random warm-up) -> the policy's own range
        (base_policy.py:258-283): undo the affine stretch (degenerate dimensions get an epsilon width), then
        undo tanh bounding with atanh."""
        if not isinstance(self.action_space, Box):
            return act
        raw = to_numpy(act)
        if not isinstance(raw, np.ndarray):
            return raw
        if self.action_scaling:
            lo = self.action_space.low
            width = self.action_space.high - lo
            tiny = np.finfo(np.float32).eps.item()
            width[width < tiny] += tiny
            raw = (raw - lo) * 2.0 / width - 1.0
        if self.action_bound_method == "tanh":
            raw = (np.log(1.0 + raw) - np.log(1.0 - raw)) / 2.0
        return raw

    def process_fn(self, batch, buffer, indices):
        return batch

    @abstractmethod
    def learn(self, batch, **kwargs: Any) -> Dict[str, Any]:
        pass

    def post_process_fn(self, batch, buffer, indices) -> None:
        pass

    def update(self, sample_size: int, buffer, **kwargs: Any) -> Dict[str, Any]:
        """process_fn -> learn -> post_process_fn (base_policy.py:332-355)."""
        if buffer is None:
            return {}
        indices = buffer.sample_indices(sample_size)
        self.updating = True
        batch = self.process_fn(None, buffer, indices)
        self.learn(batch, **kwargs)
        self.post_process_fn(batch, buffer, indices)
        if self.lr_scheduler is not None:
            self.lr_scheduler.step()
        self.updating = False

    @staticmethod
    def value_mask(buffer, indices):
        return buffer.terminated[indices] == 0

    @staticmethod
    def get_metrics(batch):
        """[reward, cost] streams of a batch (base_policy.py:377-382).  The reference re-reads the cost from
        ``batch.info["cost"]`` because tianshou's buffer drops the collector's ``cost`` key; the device buffer
        stores it as a first-class array, and a host ``Batch`` with an ``info`` entry is accepted as well."""
        cost = getattr(batch, "cost", None)
        if cost is None:
            info = getattr(batch, "info", None)
            cost = info.get("cost", None) if info is not None and hasattr(info, "get") else None
        if cost is None:
            cost = np.zeros(np.shape(batch.rew))
        if isinstance(cost, np.ndarray):
            cost = cost.astype(np.asarray(batch.rew).dtype)
        return [batch.rew, cost]

    # ---- GAE ---------------------------------------------------------------------------------------------
    def gather_batch(self, buffer, indices: torch.Tensor) -> DeviceBatch:
        """buffer[indices] as SoA device arrays; zero-copy when the valid transitions are the
        whole dense buffer (every env filled its sub-buffer, the headline configuration)."""
        b = DeviceBatch()
        n = int(indices.numel())
        b.n = n
        dense = (n == buffer.maxsize)
        b.indices = indices
        if dense:
            b.obs, b.obs_next, b.act = buffer.obs, buffer.obs_next, buffer.act
            b.rew, b.cost, b.logp_old = buffer.rew, buffer.cost, buffer.logp
            b.terminated, b.truncated = buffer.terminated, buffer.truncated
        else:
            b.obs, b.obs_next, b.act = buffer.obs[indices], buffer.obs_next[indices], buffer.act[indices]
            b.rew, b.cost, b.logp_old = buffer.rew[indices], buffer.cost[indices], buffer.logp[indices]
            b.terminated, b.truncated = buffer.terminated[indices], buffer.truncated[indices]
        return b

    def compute_gae_returns(self, batch: Optional[DeviceBatch], buffer, indices: torch.Tensor,
                            gae_lambda: float = 0.95) -> DeviceBatch:
        assert 0.0 <= gae_lambda <= 1.0, "GAE lambda should be in [0, 1]."
        if batch is None:
            batch = self.gather_batch(buffer, indices)
        n, C, dev = batch.n, self.critics_num, self.device
        end_flag = (batch.terminated | batch.truncated)                               # :410
        unfinished = buffer.unfinished_index()
        if unfinished.numel():
            end_flag = end_flag.clone()
            end_flag[torch.isin(indices, unfinished)] = 1                               # :411
        batch.end_flag = end_flag
        v = torch.empty((C, n), dtype=torch.float32, device=dev)
        vnext = torch.empty((C, n), dtype=torch.float32, device=dev)
        # V(obs_next[i]) == V(obs[i+1]) wherever the collector stored the same row twice (inside an
        # episode segment), so only the other rows need a second critic pass: segment ends, the last
        # row, and every row whose successor in the batch is NOT its obs_next (an abandoned partial
        # episode after a second collect without reset_buffer, or caller-chosen `indices`).  The test is
        # on the data itself, so it holds for any index set (the reference always evaluates
        # critic(obs_next), base_policy.py:427-428).
        need = end_flag.to(torch.bool).clone()
        need[-1] = True
        if n > 1:
            need[:-1] |= (batch.obs_next[:-1] != batch.obs[1:]).any(dim=1)
        ends = torch.nonzero(need, as_tuple=False).flatten().to(torch.int32)
        for i in range(C):
            vi = self.net_forward(1 + i, batch.obs).flatten()
            v[i] = vi
            vnext[i, :-1] = vi[1:]
            if ends.numel():
                ve = self.net_forward(1 + i, batch.obs_next, idx=ends).flatten()
                vnext[i, ends.long()] = ve
        v_scan, vnext_scan = v, vnext
        if self._rew_norm:
            # un-normalise V(s), V(s') by the running std of the returns (no mean shift, :430-436)
            scale = torch.tensor([float(np.sqrt(r.var + self._eps)) for r in self.ret_rms],
                                 dtype=torch.float32, device=dev).view(C, 1)
            v_scan, vnext_scan = v * scale, vnext * scale
        adv, ret = ops.gae_dual(v_scan, vnext_scan, batch.rew, batch.cost if C > 1 else None, end_flag,
                                batch.terminated, self._gamma, gae_lambda)
        if self._rew_norm:
            ret = ret / scale                                                           # :442-443
            r64 = ret.double()
            means, variances = r64.mean(dim=1).cpu().numpy(), r64.var(dim=1, unbiased=False).cpu().numpy()
            for i in range(C):                                                          # :444
                self.ret_rms[i].update_moments(float(means[i]), float(variances[i]), n)
        batch.v, batch.adv, batch.ret = v, adv, ret
        batch.values, batch.rets, batch.advs = v.t(), ret.t(), adv.t()
        return batch
