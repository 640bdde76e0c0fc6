"""First Order Constrained Optimization in Policy Space (reference:
/root/reference/fsrl/policy/focops.py; SURVEY.md 8f-2).

process_fn (:135-155): dual GAE + the old log-prob / mean / std of the collecting policy.
learn (:217-251): one dual step on nu (:157-162), then per repeat and per minibatch of
tianshou's ``Batch.split`` a critic regression step (MSE + L2 over the critic
parameters, :164-180) and an actor step (:182-215) on

    mean( (KL(new || old) - ratio (A_r - nu A_c) / lambda) * 1[KL <= eta] )

with per-minibatch advantage normalisation and clip_grad_norm_ on the actor; the repeat loop stops
early when the mean KL exceeds delta.  Forward / backward / weight gradients / Adam run on the
generic device engine (csrc/engine.cu), the loss head is csrc/cpo.cu::focops_head_kernel.
"""
from __future__ import annotations

import ctypes
from typing import Any, Dict, List, Optional, Tuple, Union

import numpy as np
import torch

from .. import _lib
from ..nets import ActorProb
from ..optim import FusedAdam
from ..utils.logger import BaseLogger, DummyLogger
from .base_policy import BasePolicy, DeviceBatch
from .trust_region import TrustRegionMixin


class FOCOPS(TrustRegionMixin, BasePolicy):
    def __init__(self, actor, critics, actor_optim, critic_optim, dist_fn=None,
                 logger: BaseLogger = DummyLogger(), cost_limit: float = 10,
                 nu: Union[float, Tuple[float, float, Any]] = 0.01, l2_reg: float = 1e-3, delta: float = 0.02,
                 eta: float = 0.02, tem_lambda: float = 0.95, gae_lambda: float = 0.95,
                 max_grad_norm: Optional[float] = 0.5, advantage_normalization: bool = True,
                 recompute_advantage: bool = False, gamma: float = 0.99, max_batchsize: int = 99999,
                 reward_normalization: bool = False, deterministic_eval: bool = True,
                 action_scaling: bool = True, action_bound_method: str = "clip", observation_space=None,
                 action_space=None, lr_scheduler=None) -> None:
        super().__init__(actor, critics, dist_fn, logger, gamma, max_batchsize, reward_normalization,
                         deterministic_eval, action_scaling, action_bound_method, observation_space,
                         action_space, lr_scheduler)
        self.actor_optim = FusedAdam.from_optimizer(actor_optim)
        self.critics_optim = FusedAdam.from_optimizer(critic_optim)
        self.optim = self.critics_optim              # TrustRegionMixin.critics_loss steps this one
        self.cost_limit = cost_limit
        self._gae_lambda = gae_lambda
        self._tem_lambda = tem_lambda
        self._grad_norm = max_grad_norm
        self._is_auto_nu = isinstance(nu, tuple)
        if self._is_auto_nu:                          # (nu_max, nu_lr, initial nu): :108-110
            self._nu_max, self._nu_lr, nu0 = nu
            self._nu = float(nu0.item()) if torch.is_tensor(nu0) else float(nu0)
        else:
            self._nu = float(nu)
        self._l2_reg = l2_reg
        self._delta = delta
        self._eta = eta
        self._norm_adv = advantage_normalization
        self._recompute_adv = recompute_advantage
        if not isinstance(actor, ActorProb) or actor._c_sigma:
            raise TypeError("FOCOPS needs a state-independent-sigma ActorProb")
        assert self.critics_num == 2, "FOCOPS uses a reward critic and one cost critic"
        self._actor_t = 0
        self._ave_cost_return = 0.0
        self._norm_sq: Optional[torch.Tensor] = None

    def pre_update_fn(self, stats_train: Dict, **kwarg) -> Any:
        self._ave_cost_return = stats_train["cost"]

    def update_cost_limit(self, cost_limit: float) -> None:
        self.cost_limit = self._expand_cost_limit(cost_limit)

    def process_fn(self, batch, buffer, indices) -> DeviceBatch:
        if self._recompute_adv:
            self._buffer, self._indices = buffer, indices
        batch = self.compute_gae_returns(batch, buffer, indices, self._gae_lambda)       # :143
        mu, std = self._old_dist(batch.obs)                                             # :146-152
        batch.mean_old, batch.std_old = mu.contiguous(), std.contiguous()
        return batch

    def nu_loss(self) -> dict:
        """Dual ascent on the cost multiplier (:157-162); a fixed nu is left untouched by the clamp only
        when it already lies in range -- the reference clamps through ``_nu_max``, which exists only in
        auto mode, so a fixed nu is reported as is."""
        limit = self.cost_limit[0] if isinstance(self.cost_limit, (list, tuple)) else self.cost_limit
        loss_nu = float(limit) - float(self._ave_cost_return)
        if self._is_auto_nu:
            self._nu = float(np.clip(np.float32(self._nu) + np.float32(-self._nu_lr * loss_nu), 0.0, self._nu_max))
        return {"loss/nu_loss": loss_nu, "loss/nu_value": float(self._nu)}

    # ---- actor step (:182-215) ------------------------------------------------------------------------------
    def _normalised_adv(self, batch: DeviceBatch, perm: torch.Tensor) -> torch.Tensor:
        if getattr(self, "_adv_n", None) is None or self._adv_n.shape != batch.adv.shape:
            self._adv_n = torch.empty_like(batch.adv)
        idx = perm.long()
        for c in range(self.critics_num):
            a = batch.adv[c][idx]
            self._adv_n[c][idx] = (a - a.mean()) / a.std() if self._norm_adv else a
        return self._adv_n

    def policy_loss(self, batch: DeviceBatch, perm: torch.Tensor, n: int) -> dict:
        eng, lib, s = self._eng, _lib.lib, self._stream()
        a = self.arena.slots[0]
        ent = self._entropy()
        adv_n = self._normalised_adv(batch, perm)
        d = self._descriptor(batch, perm, n)
        d.adv = adv_n.data_ptr()
        inp = eng.make_input(batch.obs, perm)
        eng.forward([a], inp, n, save=True)
        _lib.check(lib.fsrl_focops_head(ctypes.byref(d), 1.0 / self._tem_lambda, float(self._nu), float(self._eta),
                                        self._sums.data_ptr(), s))
        eng.backward([a], n)
        clip = float(self._grad_norm) if self._grad_norm else 0.0
        if self._norm_sq is None:
            self._norm_sq = torch.zeros(1, dtype=torch.float32, device=self.device)
        self._norm_sq.zero_()
        eng.wgrad([a], inp, n, norm_sq=self._norm_sq if clip > 0 else None)
        self._actor_t += 1
        g = self.actor_optim.param_groups[0]
        eng.adam([a], g["lr"], self._actor_t, betas=g["betas"], eps=g["eps"],
                 norm_sq=self._norm_sq if clip > 0 else None, max_grad_norm=clip)
        eng.sync_mirror([a])
        sm = self._sums.cpu().numpy()
        return {"loss/actor_loss": float(sm[0] / n), "loss/kl": float(sm[1] / n), "loss/entropy": ent}

    def learn(self, batch: DeviceBatch, batch_size: int, repeat: int, **kwargs: Any) -> Dict[str, List[float]]:
        n_all = batch.n
        self._ensure_engine(n_all)
        self.last_stats = {}
        stats_nu = self.nu_loss()                                                       # :221
        with torch.cuda.device(self.device):
            for step in range(repeat):
                if self._recompute_adv and step > 0:                                    # :224-227
                    batch = self.compute_gae_returns(batch, self._buffer, self._indices, self._gae_lambda)
                iter_counts, approx_kl = 0, 0.0
                for perm, n in self._minibatches(n_all, batch_size):
                    stats_critic = self.critics_loss(batch, perm, n)                    # :231
                    stats_actor = self.policy_loss(batch, perm, n)                      # :234
                    approx_kl += stats_actor["loss/kl"]
                    iter_counts += 1
                    self.gradient_steps += 1
                    self._record({**stats_nu, **stats_actor, **stats_critic})
                approx_kl /= iter_counts + 1e-7                                         # :246
                if approx_kl > self._delta:
                    self.logger.print("Early stop at step %d due to reaching max kl." % step)
                    break
        self.logger.store(gradient_steps=self.gradient_steps, tab="update")
