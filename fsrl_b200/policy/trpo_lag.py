"""TRPO with PID Lagrangian (reference: /root/reference/fsrl/policy/trpo_lag.py; SURVEY.md 8f-1).
Shares CPO's device machinery: the surrogate gradient is a linear combination of the two head
gradients CPO already computes, the Fisher-vector product is the same R-op kernel evaluated with
the OLD distribution re-taken at the current parameters (:189-190, so H is the pure Fisher
matrix), conjugate gradients use tol 1e-10 (:265), the step is -H^-1 g * sqrt(2 delta / d^T H d)
with plain backtracking on `kl < delta and loss decreased` (:195-231)."""
from __future__ import annotations

import ctypes
from typing import Any, Dict, List, Optional, Tuple, Union

import numpy as np
import torch

from .. import _lib
from ..nets import ActorProb
from ..optim import FusedAdam
from ..utils.logger import BaseLogger, DummyLogger
from .base_policy import DeviceBatch
from .lagrangian_base import LagrangianPolicy
from .trust_region import TrustRegionMixin


class TRPOLagrangian(TrustRegionMixin, LagrangianPolicy):
    def __init__(self, actor, critics, optim, dist_fn=None, logger: BaseLogger = DummyLogger(),
                 target_kl: float = 0.001, backtrack_coeff: float = 0.8, max_backtracks: int = 10,
                 optim_critic_iters: int = 5, gae_lambda: float = 0.95, advantage_normalization: bool = True,
                 use_lagrangian: bool = True, lagrangian_pid: Tuple = (0.05, 0.0005, 0.1),
                 cost_limit: Union[List, float] = np.inf, rescaling: bool = True, gamma: float = 0.99,
                 max_batchsize: int = 99999, reward_normalization: bool = False,
                 deterministic_eval: bool = True, action_scaling: bool = True,
                 action_bound_method: str = "clip", observation_space=None, action_space=None,
                 lr_scheduler=None) -> None:
        super().__init__(actor, critics, dist_fn, logger, use_lagrangian, lagrangian_pid, cost_limit,
                         rescaling, gamma, max_batchsize, reward_normalization, deterministic_eval,
                         action_scaling, action_bound_method, observation_space, action_space, lr_scheduler)
        self.optim = FusedAdam.from_optimizer(optim)
        self._lambda = gae_lambda
        self._norm_adv = advantage_normalization
        self._max_backtracks = max_backtracks
        self._delta = target_kl
        self._backtrack_coeff = backtrack_coeff
        self._optim_critic_iters = optim_critic_iters
        self._damping_coeff = 0.1                       # hard-coded in the reference (:115)
        self._l2_reg = 0.0
        if not isinstance(actor, ActorProb) or actor._c_sigma:
            raise TypeError("TRPOLagrangian needs a state-independent-sigma ActorProb")
        assert self.critics_num == 2

    def process_fn(self, batch, buffer, indices) -> DeviceBatch:
        batch = self.compute_gae_returns(batch, buffer, indices, self._lambda)
        if self._norm_adv:                                                   # :129-133
            for c in range(self.critics_num):
                self._standardize(batch.adv[c], batch.n)
        batch.mean_old = torch.empty((batch.n, self.arena.slots[0].out), dtype=torch.float32, device=self.device)
        batch.std_old = torch.empty_like(batch.mean_old)
        return batch

    def _refresh_old_dist(self, batch: DeviceBatch) -> None:
        """old_dist = self(minibatch).dist under no_grad at the CURRENT parameters (:189-190)."""
        mu, std = self._old_dist(batch.obs)
        batch.mean_old.copy_(mu)
        batch.std_old.copy_(std)

    def learn(self, batch: DeviceBatch, batch_size: int, repeat: int, **kwargs: Any) -> Dict[str, List[float]]:
        n_all = batch.n
        eng = self._ensure_engine(n_all)
        lib, a = _lib.lib, self.arena.slots[0]
        P = a.size
        v = self._vec
        self.last_stats = {}
        theta_a = self.arena.theta[a.offset:a.offset + P]
        with torch.cuda.device(self.device):
            s = self._stream()
            for _ in range(repeat):
                minibatches = self._minibatches(n_all, batch_size)
                self._dp_same_count(len(minibatches), "minibatch count")
                for perm, n in minibatches:
                    lag = self.lagrangians()[0] if (self.use_lagrangian and self.lag_optims) else 0.0
                    resc = self.rescaling_factor() if self.use_lagrangian else 1.0
                    self._refresh_old_dist(batch)
                    d = self._descriptor(batch, perm, n)
                    inp = eng.make_input(batch.obs, perm)
                    e, nl = eng.engine(), eng.netlist([a])

                    n_g = self._dp_begin(n)     # rows of the global minibatch (== n on one GPU)

                    def loss_of(sm):            # policy_loss (:158-180) from the batch sums
                        return resc * (-(sm[0] / n_g) + lag * (sm[1] / n_g))

                    eng.forward([a], inp, n, save=True)
                    self._head(d, 1)
                    sm = self._gsums()
                    eng.backward([a], n)
                    _lib.check(lib.fsrl_engine_wgrad_to(ctypes.byref(e), ctypes.byref(nl), ctypes.byref(inp), n, v["g"].data_ptr(), s))
                    self._gvec(v["g"])
                    self._head(d, 2)
                    eng.backward([a], n)
                    _lib.check(lib.fsrl_engine_wgrad_to(ctypes.byref(e), ctypes.byref(nl), ctypes.byref(inp), n, v["b"].data_ptr(), s))
                    self._gvec(v["b"])
                    loss_actor = loss_of(sm)
                    # flat_grads = rescaling * (-grad objective + lambda * grad cost ratio term)
                    flat = v["step"]
                    _lib.check(lib.fsrl_vec_add_scaled(v["g"].data_ptr(), lag, v["b"].data_ptr(), flat.data_ptr(), P, s))
                    flat.mul_(-resc)
                    self._head(d, 3)
                    eng.backward([a], n)
                    self._cg(d, flat, v["Hinv_g"], nsteps=10, residual_tol=1e-10)
                    sd = v["Hinv_g"]
                    sd.neg_()                                                 # search_direction (:194)
                    self._hvp(d, sd, v["hv"])
                    shs = self._dotp(sd, v["hv"])
                    step_size = float(np.sqrt(2 * self._delta / shs)) if shs > 0 else float("nan")
                    v["theta0"].copy_(theta_a)
                    kl = float("nan")
                    for i in range(self._max_backtracks):
                        _lib.check(lib.fsrl_vec_add_scaled(v["theta0"].data_ptr(), step_size, sd.data_ptr(), theta_a.data_ptr(), P, s))
                        eng.forward([a], inp, n, save=False)
                        self._head(d, 0)
                        sm2 = self._gsums()
                        kl = float(sm2[2] / n_g)
                        if kl < self._delta and loss_of(sm2) < loss_actor:
                            break
                        elif i < self._max_backtracks - 1:
                            step_size = step_size * self._backtrack_coeff
                        else:
                            step_size = 0.0                                   # last tried params stay (:223-231)
                            self.logger.print("Line search failed! It seems hyperparamters"
                                              " are poor and need to be changed.")
                    eng.sync_mirror([a])
                    for _ in range(self._optim_critic_iters):                 # :233-238
                        stats_critic = self.critics_loss(batch, perm, n)
                        self.gradient_steps += 1
                    stats = {"loss/actor_rew": float(-(sm[0] / n_g)), "loss/actor_total": float(loss_actor),
                             "loss/rescaling": resc, "loss/kl": kl, "loss/step_size": step_size,
                             "loss/entropy": self._entropy(), **stats_critic}
                    if self.use_lagrangian:
                        stats["loss/lagrangian"] = lag
                        stats["loss/actor_safety"] = float(lag * sm[1] / n_g)
                    self._record(stats)
        self.logger.store(gradient_steps=self.gradient_steps, tab="update")
