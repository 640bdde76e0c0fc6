"""Constrained Variational Policy Optimization (reference: /root/reference/fsrl/policy/cvpo.py).

Gaussian actor without a tanh squash (conditioned or state-independent sigma), one SingleCritic or
DoubleCritic per return stream with Polyak targets, n-step targets whose next action is sampled from the
current actor.  ``update_many`` runs whole gradient steps on the device (csrc/cvpo.cu,
``fsrl_cvpo_steps``): critic regression, the E-step (K particles of ``actor_old`` scored by the updated
critics, Adam on the dual ``[eta, lambda]``, softmax weights) and the M-step (weighted maximum likelihood
with decoupled KL multipliers).  Every dual and its Adam moments stay on the device, so a batch of steps
never synchronises with the host.  Like the reference, ``estep_dual`` is not part of the state_dict."""
from __future__ import annotations

import ctypes
from copy import deepcopy
from typing import Any, List, Optional, Union

import numpy as np
import torch
from torch.distributions import Independent, Normal

from .. import _lib
from ..data.batch import Batch
from ..nets import SIGMA_MAX, SIGMA_MIN, ActorProb, DoubleCritic, SingleCritic
from ..utils.logger import BaseLogger, DummyLogger
from .offpolicy_base import OffPolicyEngine


class CVPO(OffPolicyEngine):
    def __init__(self, actor, critics, actor_optim, critic_optim, action_space, dist_fn, max_episode_steps: int,
                 logger: Optional[BaseLogger] = DummyLogger(), cost_limit: Union[List, float] = np.inf,
                 tau: float = 0.05, gamma: float = 0.99, n_step: int = 2,
                 estep_iter_num: int = 1, estep_kl: float = 0.02, estep_dual_max: float = 20,
                 estep_dual_lr: float = 0.02, sample_act_num: int = 16,
                 mstep_iter_num: int = 1, mstep_kl_mu: float = 0.005, mstep_kl_std: float = 0.0005,
                 mstep_dual_max: float = 0.5, mstep_dual_lr: float = 0.1,
                 deterministic_eval: bool = True, action_scaling: bool = True, action_bound_method: str = "clip",
                 lr_scheduler=None) -> None:
        super().__init__(actor, critics, dist_fn, logger, gamma, 99999, False, deterministic_eval, action_scaling,
                         action_bound_method, None, action_space, lr_scheduler)
        if not isinstance(actor, ActorProb):
            raise TypeError("CVPO needs a Gaussian ActorProb")
        if all(isinstance(c, DoubleCritic) for c in self.critics):
            self._twin = True
        elif all(isinstance(c, SingleCritic) for c in self.critics):
            self._twin = False
        else:
            raise TypeError("CVPO critics must be all SingleCritic or all DoubleCritic")
        self.actor_old = deepcopy(self.actor)
        self.actor_old.eval()
        self.actor_optim = actor_optim
        self.critics_old = deepcopy(self.critics)
        self.critics_old.eval()
        self.critics_optim = critic_optim
        self.dtype = torch.float32
        self.max_episode_steps = max_episode_steps
        self.update_cost_limit(cost_limit)
        self._estep_kl, self._estep_iter_num = estep_kl, estep_iter_num
        self._estep_dual_max, self._estep_dual_lr = estep_dual_max, estep_dual_lr
        self._sample_act_num = sample_act_num
        self._mstep_kl_mu, self._mstep_kl_std = mstep_kl_mu, mstep_kl_std
        self._mstep_iter_num, self._mstep_dual_max, self._mstep_dual_lr = mstep_iter_num, mstep_dual_max, mstep_dual_lr
        a_lr = actor_optim.param_groups[0]["lr"] if hasattr(actor_optim, "param_groups") else 5e-4
        c_lr = critic_optim.param_groups[0]["lr"] if hasattr(critic_optim, "param_groups") else 1e-3
        self._init_offpolicy(tau, n_step, a_lr, c_lr)
        self._estep_state: Optional[torch.Tensor] = None   # eta, lambda, adam m[2], v[2], step, -
        self._mstep_state: Optional[torch.Tensor] = None   # dual_mu, dual_std, adam m[2], v[2], step, -

    # ---- arena -------------------------------------------------------------------------------------------
    def _net_list(self):
        return [self.actor] + list(self.critics) + [self.actor_old] + list(self.critics_old)

    def _groups(self):
        g, C = self._slot_groups, self.critics_num
        return {"actor": g[0], "critics": [s for grp in g[1:1 + C] for s in grp], "actor_old": g[1 + C],
                "critics_old": [s for grp in g[2 + C:2 + 2 * C] for s in grp]}

    def _states(self):
        if self._estep_state is None:
            dev = self.device
            self._estep_state = torch.zeros(8, dtype=torch.float32, device=dev)
            self._estep_state[0] = 1.0                                      # eta = 1, lambda = 0 (cvpo.py:142-146)
            self._mstep_state = torch.zeros(8, dtype=torch.float32, device=dev)
        return self._estep_state, self._mstep_state

    def _alloc_work(self, bmax: int) -> None:
        dev, A = self.device, self._A
        self._cw = dict(particles=torch.zeros((bmax, A), dtype=torch.float32, device=dev),
                        part_idx=torch.zeros(bmax, dtype=torch.int32, device=dev),
                        mu_old=torch.zeros((bmax, A), dtype=torch.float32, device=dev),
                        std_old=torch.zeros((bmax, A), dtype=torch.float32, device=dev),
                        comb=torch.zeros(bmax, dtype=torch.float32, device=dev),
                        weights=torch.zeros(bmax, dtype=torch.float32, device=dev))

    def _cvpo_descriptor(self, buffer) -> "_lib.Cvpo":
        es, ms = self._states()
        d = _lib.Cvpo()
        d.off = self._descriptor(buffer)
        d.K, d.estep_iters, d.mstep_iters = self._sample_act_num, self._estep_iter_num, self._mstep_iter_num
        d.cond_sigma = int(self.actor._c_sigma)
        d.estep_kl, d.estep_dual_max, d.estep_dual_lr = self._estep_kl, self._estep_dual_max, self._estep_dual_lr
        d.qc_thres = float(self.qc_thres[0]) if self.critics_num > 1 else 0.0
        d.mstep_kl_mu, d.mstep_kl_std = self._mstep_kl_mu, self._mstep_kl_std
        d.mstep_dual_max, d.mstep_dual_lr = self._mstep_dual_max, self._mstep_dual_lr
        d.estep_state, d.mstep_state = es.data_ptr(), ms.data_ptr()
        w = self._cw
        d.particles, d.part_idx = w["particles"].data_ptr(), w["part_idx"].data_ptr()
        d.mu_old, d.std_old = w["mu_old"].data_ptr(), w["std_old"].data_ptr()
        d.comb, d.weights = w["comb"].data_ptr(), w["weights"].data_ptr()
        if not self.actor._c_sigma:
            g = self._groups()
            d.log_sigma, d.log_sigma_old = self.arena.extra_ptr(g["actor"][0]), self.arena.extra_ptr(g["actor_old"][0])
        return d

    # ---- rollout: the conditioned-sigma head without SAC's squash ------------------------------------------
    def fill_rollout(self, r, exploration_noise: bool = False) -> None:
        super().fill_rollout(r, exploration_noise)
        if self.actor._c_sigma:
            r.head = _lib.HEAD_GAUSS_COND_RAW

    # ---- reference hooks -----------------------------------------------------------------------------------
    @property
    def estep_dual(self) -> torch.Tensor:
        """[eta, lambda_1..] on the device (cvpo.py:142-146)."""
        return self._states()[0][:self.critics_num]

    @property
    def mstep_dual_mu(self) -> torch.Tensor:
        return self._states()[1][0:1]

    @property
    def mstep_dual_std(self) -> torch.Tensor:
        return self._states()[1][1:2]

    @property
    def estep_optim(self) -> dict:
        """The E-step dual's Adam state, device resident (torch.optim.Adam(lr=estep_dual_lr) in the reference)."""
        es = self._states()[0]
        C = self.critics_num
        return {"lr": self._estep_dual_lr, "exp_avg": es[2:2 + C], "exp_avg_sq": es[4:4 + C], "step": es[6:7]}

    @property
    def mstep_optim(self) -> dict:
        """The M-step duals' Adam state, device resident; pre_update_fn resets it."""
        ms = self._states()[1]
        return {"lr": self._mstep_dual_lr, "exp_avg": ms[2:4], "exp_avg_sq": ms[4:6], "step": ms[6:7]}

    def update_cost_limit(self, cost_limit) -> None:
        self.cost_limit = [cost_limit] * (self.critics_num - 1) if np.isscalar(cost_limit) else cost_limit
        T = self.max_episode_steps
        self.qc_thres = [c * (1 - self._gamma ** T) / (1 - self._gamma) / T for c in self.cost_limit]

    def pre_update_fn(self, **kwarg: Any) -> None:
        """Fresh M-step duals and Adam state for this collect cycle (cvpo.py:178-188)."""
        self._states()[1].zero_()

    def post_update_fn(self, **kwarg: Any) -> None:
        """actor_old <- actor (cvpo.py:190-193): arena copy plus the W2 mirror of actor_old."""
        g = self._groups()
        src, dst = g["actor"][0], g["actor_old"][0]
        th = self.arena.theta
        with torch.no_grad():
            th[dst.offset:dst.offset + dst.size].copy_(th[src.offset:src.offset + src.size])
        if self._eng is not None:
            self._eng.sync_mirror([dst])

    def sync_weight(self) -> None:
        g = self._groups()
        self._ensure_engine(256).polyak(g["critics_old"], g["critics"], self.tau)

    def get_extra_state(self):
        """None, like the reference (cvpo.py:432-439): estep_dual is not checkpointed."""
        return None

    def set_extra_state(self, state) -> None:
        pass

    @staticmethod
    def gaussian_kl(mu_old, std_old, mu, std):
        """Decoupled KL (cvpo.py:289-317): kl_mu under the old variance, kl_std at the old mean."""
        var_old, var = torch.clamp_min(std_old ** 2, 1e-6), torch.clamp_min(std ** 2, 1e-6)
        kl_mu = torch.sum(0.5 * (mu_old - mu) ** 2 / var_old, dim=-1).mean()
        kl_std = torch.sum(0.5 * (torch.log(var / var_old) + var_old / var - 1), dim=-1).mean()
        return kl_mu, kl_std

    def forward(self, batch: Batch, state=None, model: str = "actor", input: str = "obs", **kwargs: Any) -> Batch:
        """API-compatible forward (cvpo.py:224-246) on a device batch: unsquashed Gaussian of ``actor`` or
        ``actor_old``."""
        g = self._groups()
        slot = g[model][0]
        obs = torch.as_tensor(batch[input], dtype=torch.float32, device=self.device).contiguous()
        out = self.net_forward(self.arena.slots.index(slot), obs)
        net = getattr(self, model)
        A = self._action_dim()
        mu = out[:, :A]
        if not net._unbounded:
            mu = net._max * torch.tanh(mu)
        if net._c_sigma:
            sigma = out[:, A:2 * A].clamp(SIGMA_MIN, SIGMA_MAX).exp()
        else:
            sigma = net.sigma_param.detach().view(1, -1).exp().expand_as(mu)
        dist = self.dist_fn(mu, sigma) if self.dist_fn is not None else Independent(Normal(mu, sigma), 1)
        act = mu if (self._deterministic_eval and not self.training) else dist.sample()
        return Batch(logits=(mu, sigma), act=act, state=None, dist=dist)

    def _action_dim(self) -> int:
        return int(self.actor.output_dim)

    # ---- gradient steps --------------------------------------------------------------------------------------
    _stats_width = _lib.CVPO_STATS

    def _run_steps(self, buffer, idx: torch.Tensor, n: int, batch_size: int, stats: torch.Tensor) -> None:
        d = self._cvpo_descriptor(buffer)
        _lib.check(_lib.lib.fsrl_cvpo_steps(ctypes.byref(d), idx.data_ptr(), n, int(batch_size), self._critic_t,
                                            self._actor_t, self._noise_t, stats.data_ptr(), self._stream()))

    def _engine_rows(self, batch_size: int) -> int:
        return self._sample_act_num * batch_size          # the E-step Q pass covers K particles per state

    def _actor_steps_per_update(self) -> int:
        return self._mstep_iter_num

    def _log_stats(self, st: np.ndarray) -> None:
        C, n = self.critics_num, len(st)
        out = {"loss/q_total": st[:, 0] + (st[:, 1] if C > 1 else 0.0), "loss/estep_loss": st[:, 4]}
        for i in range(C):
            out[f"loss/loss_q{i}"] = st[:, i]
            out[f"estep/dual{i}"] = st[:, 5 + i]
            out[f"estep/val_q{i}"] = st[:, 2 + i]
            if i >= 1:
                out[f"estep/thres_q{i}"] = np.full(n, self.qc_thres[i - 1])
        for k, col in (("mstep_kl_mu", 7), ("mstep_kl_std", 8), ("mstep_loss_kl", 9), ("mstep_loss_mle", 10),
                       ("mstep_loss_total", 11), ("mstep_dual_mu", 12), ("mstep_dual_std", 13), ("entropy", 14)):
            out["mstep/" + k] = st[:, col]
        self.last_stats = out
        for k, v in out.items():
            tab, key = k.split("/", 1)
            self.logger.store_many(tab, key, v)
