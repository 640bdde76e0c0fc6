"""Shared device machinery of the off-policy learners: ``OffPolicyEngine`` holds what SAC, DDPG and CVPO
all need (engine context, work arrays, replay-buffer half of the csrc/offpolicy.cu descriptor, batch-index
sampling, n-step returns); ``OffPolicyLagrangian`` adds the PID-Lagrangian multiplier and the batched gradient
steps of SAC / DDPG.

Reference call path being replaced: OffpolicyTrainer.policy_update_fn
(fsrl/trainer/offpolicy.py:93-106) -> BasePolicy.update (base_policy.py:332-355) ->
process_fn = compute_nstep_returns (:453-512) -> learn (sac_lag.py:260-269 /
ddpg_lag.py:215-223)."""
from __future__ import annotations

import ctypes
from copy import deepcopy
from typing import Any, Dict, List, Optional

import numpy as np
import torch

from .. import _lib
from ..data.batch import Batch
from ..engine import EngineCtx
from ..nets import SIGMA_MAX, SIGMA_MIN
from .base_policy import BasePolicy
from .lagrangian_base import LagrangianPolicy


class OffPolicyEngine(BasePolicy):
    _algo = _lib.ALGO_SAC

    def _init_offpolicy(self, tau, n_step, actor_lr, critic_lr):
        assert 0.0 <= tau <= 1.0, "tau should be in [0, 1]"
        self.tau = tau
        self._n_step = n_step
        self._actor_lr, self._critic_lr = actor_lr, critic_lr
        self._eng: Optional[EngineCtx] = None
        self._critic_t = 0
        self._actor_t = 0
        self._noise_t = 0
        self._upd_seed = 0
        self.last_stats: Dict[str, np.ndarray] = {}

    def set_update_seed(self, seed: int) -> None:
        self._upd_seed = int(seed) & 0xFFFFFFFF

    # groups of arena slots ---------------------------------------------------------------------------
    def _groups(self):
        raise NotImplementedError

    def _ensure_engine(self, bmax: int):
        if self._eng is None or self._eng.bmax < bmax:
            self._eng = EngineCtx(self.arena, max(bmax, 256), grown_from=self._eng)
            B, dev = self._eng.bmax, self.device
            A = int(self.actor.output_dim)
            self._A = A
            self._w = dict(
                term_idx=torch.zeros(B, dtype=torch.int32, device=dev),
                partial=torch.zeros(2 * B, dtype=torch.float64, device=dev),
                gpow=torch.zeros(B, dtype=torch.float64, device=dev),
                vmask=torch.zeros(B, dtype=torch.float32, device=dev),
                target=torch.zeros(2 * B, dtype=torch.float32, device=dev),
                act_next=torch.zeros((B, A), dtype=torch.float32, device=dev),
                logp_next=torch.zeros(B, dtype=torch.float32, device=dev),
                act=torch.zeros((B, A), dtype=torch.float32, device=dev),
                logp=torch.zeros(B, dtype=torch.float32, device=dev),
                keep=torch.zeros((B, 24), dtype=torch.float32, device=dev),
            )
            self._alloc_work(B)
        return self._eng

    def _alloc_work(self, bmax: int) -> None:
        pass

    def _descriptor(self, buffer) -> "_lib.OffPolicy":
        eng = self._eng
        g = self._groups()
        d = _lib.OffPolicy()
        d.eng = eng.engine()
        d.actor = eng.netlist(g["actor"])
        d.critics = eng.netlist(g["critics"])
        d.critics_old = eng.netlist(g["critics_old"])
        if g.get("actor_old"):
            d.actor_old = eng.netlist(g["actor_old"])
        d.algo = self._algo
        d.D, d.A, d.C = self.arena.slots[0].D, self._A, self.critics_num
        d.twin = int(self._twin)
        d.n_step = self._n_step
        d.bounded = int(not getattr(self.actor, "_unbounded", False))
        d.seed = self._upd_seed
        d.gamma, d.tau = self._gamma, self.tau
        # learning rates are read from the caller's optimizers every time (an lr scheduler stepping them takes effect); the
        # engine's Adam uses torch's default betas / eps -- anything else is rejected loudly instead of being ignored
        a_opt, c_opt = getattr(self, "actor_optim", None), getattr(self, "critics_optim", None)
        for opt in (a_opt, c_opt):
            if opt is not None and hasattr(opt, "param_groups"):
                g0 = opt.param_groups[0]
                if tuple(g0.get("betas", (0.9, 0.999))) != (0.9, 0.999) or g0.get("eps", 1e-8) != 1e-8 or g0.get("weight_decay", 0) != 0:
                    raise ValueError("the off-policy engine runs Adam with betas=(0.9, 0.999), eps=1e-8, weight_decay=0; got %r"
                                     % {k: g0.get(k) for k in ("betas", "eps", "weight_decay")})
        if a_opt is not None and hasattr(a_opt, "param_groups"):
            self._actor_lr = float(a_opt.param_groups[0]["lr"])
        if c_opt is not None and hasattr(c_opt, "param_groups"):
            self._critic_lr = float(c_opt.param_groups[0]["lr"])
        d.critic_lr, d.actor_lr = self._critic_lr, self._actor_lr
        d.max_action = float(self.actor._max)
        d.sigma_min, d.sigma_max = SIGMA_MIN, SIGMA_MAX
        d.tanh_eps = float(np.finfo(np.float32).eps)
        d.rescaling = 1.0
        self._fill_lagrangian(d)
        d.b_obs, d.b_obs_next, d.b_act = buffer.obs.data_ptr(), buffer.obs_next.data_ptr(), buffer.act.data_ptr()
        d.b_rew, d.b_cost = buffer.rew.data_ptr(), buffer.cost.data_ptr()
        d.b_term, d.b_trunc = buffer.terminated.data_ptr(), buffer.truncated.data_ptr()
        d.b_ptr, d.b_len, d.cap = buffer.ptr.data_ptr(), buffer.len.data_ptr(), buffer.cap
        w = self._w
        d.w_term_idx, d.w_partial, d.w_gpow = w["term_idx"].data_ptr(), w["partial"].data_ptr(), w["gpow"].data_ptr()
        d.w_vmask, d.w_target = w["vmask"].data_ptr(), w["target"].data_ptr()
        d.w_act_next, d.w_logp_next = w["act_next"].data_ptr(), w["logp_next"].data_ptr()
        d.w_act, d.w_logp, d.w_keep = w["act"].data_ptr(), w["logp"].data_ptr(), w["keep"].data_ptr()
        a = g["actor"][0]
        d.actor_out = eng.slot_view(a, "out").data_ptr()
        d.actor_dout = eng.slot_view(a, "dout").data_ptr()
        if g.get("actor_old"):
            d.actor_old_out = eng.slot_view(g["actor_old"][0], "out").data_ptr()
        for i, s in enumerate(g["critics"]):
            d.q_out[i] = eng.slot_view(s, "out").data_ptr()
            d.q_dout[i] = eng.slot_view(s, "dout").data_ptr()
            d.q_dx[i] = eng.slot_view(s, "dx").data_ptr()
        for i, s in enumerate(g["critics_old"]):
            d.q_old_out[i] = eng.slot_view(s, "out").data_ptr()
        dp = getattr(self, "_dp", None)
        if dp is not None and dp.world > 1:
            d.comm, d.world = dp.comm, dp.world
        self._fill_algo(d)
        return d

    def _fill_algo(self, d) -> None:
        pass

    def _fill_lagrangian(self, d) -> None:
        pass

    # ---- reference hooks ---------------------------------------------------------------------------------
    def train(self, mode: bool = True):
        self.training = mode
        self.actor.train(mode)
        self.critics.train(mode)
        return self

    def sample_batch_indices(self, buffer, n_steps: int, batch_size: int) -> torch.Tensor:
        """[n_steps][batch_size] flat buffer indices, drawn on the host with NumPy's global RNG
        like tianshou's buffer.sample (one randint stream, row k = the k-th update's batch)."""
        lens = buffer.len.cpu().numpy().astype(np.int64)
        total = int(lens.sum())
        if total == 0:
            raise ValueError("cannot sample from an empty buffer")
        offsets = np.concatenate([[0], np.cumsum(lens)])
        draw = np.random.randint(0, total, size=(n_steps, batch_size))
        env = np.searchsorted(offsets, draw, side="right") - 1
        k = draw - offsets[env]
        ptr = buffer.ptr.cpu().numpy().astype(np.int64)
        start = np.where(lens == buffer.cap, ptr, 0)
        flat = env * buffer.cap + (start[env] + k) % buffer.cap
        return torch.as_tensor(flat.astype(np.int32), device=self.device)

    def compute_nstep_returns(self, batch, buffer, indice, target_q_fn, n_step: int = 1):
        """API twin of BasePolicy.compute_nstep_returns (base_policy.py:453-512) for callers that drive the
        pieces themselves (the built-in update path fuses this into ``fsrl_offpolicy_steps``): the n-step walk,
        the discounted reward / cost sums, gamma^k and the value mask come from ``fsrl_nstep_prepare``;
        ``target_q_fn(buffer, terminal_indices)`` returns one tensor per critic stream, and
        ``batch.rets[b, i] = partial_i[b] + gamma^k[b] * ~terminated[terminal[b]] * target_q_i[b]``."""
        idx = torch.as_tensor(indice, device=self.device).to(torch.int32).contiguous()
        B = int(idx.numel())
        self._ensure_engine(max(B, 256))
        d = self._descriptor(buffer)
        d.n_step = int(n_step)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib.fsrl_nstep_prepare(ctypes.byref(d), idx.data_ptr(), B, self._stream()))
        w = self._w
        terminal = w["term_idx"][:B]
        with torch.no_grad():
            target_q_list = target_q_fn(buffer, terminal)
        partial = w["partial"][:2 * B].view(2, B)
        rets = []
        for i in range(self.critics_num):
            tq = torch.as_tensor(target_q_list[i], device=self.device).reshape(B, -1).float() * w["vmask"][:B, None]
            rets.append((tq.double() * w["gpow"][:B, None] + partial[i][:, None]).float())
        if batch is None:
            batch = Batch()
        batch.rets = torch.stack(rets, dim=-1)
        return batch


    # ---- batched gradient steps: one C call per chunk, parameterised by the learner --------------------------
    _stats_width = _lib.OFF_STATS

    def _run_steps(self, buffer, idx: torch.Tensor, n: int, batch_size: int, stats: torch.Tensor) -> None:
        d = self._descriptor(buffer)
        _lib.check(_lib.lib.fsrl_offpolicy_steps(ctypes.byref(d), idx.data_ptr(), n, int(batch_size), self._critic_t,
                                                 self._actor_t, self._noise_t, stats.data_ptr(), self._stream()))

    def _engine_rows(self, batch_size: int) -> int:
        return batch_size

    def _actor_steps_per_update(self) -> int:
        return 1

    def update_many(self, n_updates: int, batch_size: int, buffer, chunk: int = 4096) -> None:
        """`n_updates` x policy.update(batch_size, buffer) without returning to Python per step."""
        if buffer is None or n_updates <= 0:
            return
        self._ensure_engine(self._engine_rows(batch_size))
        self.updating = True
        stats_all = []
        done = 0
        while done < n_updates:
            n = min(chunk, n_updates - done)
            idx = self.sample_batch_indices(buffer, n, batch_size)
            stats = torch.zeros((n, self._stats_width), dtype=torch.float32, device=self.device)
            with torch.cuda.device(self.device):
                self._run_steps(buffer, idx, n, batch_size, stats)
            self._critic_t += n; self._actor_t += n * self._actor_steps_per_update(); self._noise_t += n
            self.gradient_steps += n
            stats_all.append(stats)
            done += n
        st = torch.cat(stats_all, 0).cpu().numpy()
        self._log_stats(st)
        if self.lr_scheduler is not None:
            for _ in range(n_updates):
                self.lr_scheduler.step()
        self.updating = False

    def update(self, sample_size: int, buffer, **kwargs: Any):
        self.update_many(1, sample_size, buffer)

    def learn(self, batch, **kwargs):
        raise RuntimeError("off-policy learners are driven through update()/update_many() on the device")

    def _log_stats(self, st: np.ndarray) -> None:
        raise NotImplementedError


class OffPolicyLagrangian(OffPolicyEngine, LagrangianPolicy):
    def _fill_lagrangian(self, d) -> None:
        d.use_lagrangian = int(self.use_lagrangian and self.critics_num > 1)
        lags = self.lagrangians()
        d.lagrangian = lags[0] if lags else 0.0
        d.rescaling = self.rescaling_factor() if self.use_lagrangian else 1.0

    def _log_stats(self, st: np.ndarray) -> None:
        resc = self.rescaling_factor() if self.use_lagrangian else 1.0
        out = {"loss/q0": st[:, 0], "loss/q_total": st[:, 0] + (st[:, 1] if self.critics_num > 1 else 0.0),
               "loss/actor_rew": st[:, 2], "loss/actor_total": resc * (st[:, 2] + st[:, 3]),
               "loss/rescaling": np.full(len(st), resc)}
        if self.critics_num > 1:
            out["loss/q1"] = st[:, 1]
        if self.use_lagrangian and self.critics_num > 1:
            out["loss/lagrangian"] = np.full(len(st), self.lagrangians()[0])
            out["loss/actor_safety"] = st[:, 3]
        self._extra_stats(out, st)
        self.last_stats = out
        for k, v in out.items():
            tab, key = k.split("/", 1)
            self.logger.store_many(tab, key, v)

    def _extra_stats(self, out, st):
        pass
