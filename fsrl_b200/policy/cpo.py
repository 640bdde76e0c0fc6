"""Constrained Policy Optimization (reference: /root/reference/fsrl/policy/cpo.py).

process_fn (:123-145): dual GAE, whole-batch advantage normalisation, old log-prob / mean / std.
learn (:353-370): per minibatch, ``optim_critic_iters`` critic regression steps (MSE + L2 over
the critic parameters, :147-162) then one policy step (:234-351): surrogate / cost gradients,
two conjugate-gradient solves with exact Hessian-vector products of the mean KL, the analytic
dual (lambda*, nu*) case analysis (transcribed from :257-304, SURVEY.md Appendix F), and the
backtracking line search -- everything batched on the device (csrc/cpo.cu, engine.cu); the
host only sees the handful of scalars the case analysis needs.
"""
from __future__ import annotations

import ctypes
from typing import Any, Dict, List, Optional, Union

import numpy as np
import torch

from .. import _lib
from ..engine import EngineCtx
from ..nets import ActorProb
from ..optim import FusedAdam
from ..utils.logger import BaseLogger, DummyLogger
from .base_policy import BasePolicy, DeviceBatch
from .trust_region import TrustRegionMixin


class CPO(TrustRegionMixin, BasePolicy):
    def __init__(self, actor, critics, optim, dist_fn=None, logger: BaseLogger = DummyLogger(),
                 target_kl: float = 0.01, backtrack_coeff: float = 0.8, damping_coeff: float = 0.1,
                 max_backtracks: int = 10, optim_critic_iters: int = 20, l2_reg: float = 0.001,
                 gae_lambda: float = 0.95, advantage_normalization: bool = True,
                 cost_limit: Union[List, float] = np.inf, gamma: float = 0.99,
                 max_batchsize: int = 99999, reward_normalization: bool = False,
                 deterministic_eval: bool = True, action_scaling: bool = True,
                 action_bound_method: str = "clip", observation_space=None, action_space=None,
                 lr_scheduler=None) -> None:
        super().__init__(actor, critics, dist_fn, logger, gamma, max_batchsize, reward_normalization,
                         deterministic_eval, action_scaling, action_bound_method, observation_space,
                         action_space, lr_scheduler)
        self.optim = FusedAdam.from_optimizer(optim)
        self._cost_limit = cost_limit
        self._lambda = gae_lambda
        self._norm_adv = advantage_normalization
        self._max_backtracks = max_backtracks
        self._optim_critic_iters = optim_critic_iters
        self._l2_reg = l2_reg
        self._delta = target_kl
        self._backtrack_coeff = backtrack_coeff
        self._damping_coeff = damping_coeff
        if not isinstance(actor, ActorProb) or actor._c_sigma:
            raise TypeError("CPO needs a state-independent-sigma ActorProb")
        assert self.critics_num == 2, "CPO uses a reward critic and one cost critic"
        self._eng: Optional[EngineCtx] = None
        self._critic_t = 0
        self._ave_cost_return = 0.0

    def pre_update_fn(self, stats_train: Dict, **kwarg) -> Any:
        self._ave_cost_return = stats_train["cost"]

    def update_cost_limit(self, cost_limit: float) -> None:
        # reference quirk (SURVEY.md App. A.12): writes `cost_limit`, the algorithm reads `_cost_limit`
        self.cost_limit = self._expand_cost_limit(cost_limit)

    def process_fn(self, batch, buffer, indices) -> DeviceBatch:
        batch = self.compute_gae_returns(batch, buffer, indices, self._lambda)          # :126
        if self._norm_adv:                                                             # :127-131
            for c in range(self.critics_num):
                self._standardize(batch.adv[c], batch.n)
        mu, std = self._old_dist(batch.obs)                                             # :133-144
        batch.mean_old, batch.std_old = mu.contiguous(), std.contiguous()
        return batch

    # ---- policy step (:234-351) ----------------------------------------------------------------------------------
    def policy_loss(self, batch: DeviceBatch, perm: Optional[torch.Tensor], n: int) -> dict:
        eng, lib, s = self._eng, _lib.lib, self._stream()
        a = self.arena.slots[0]
        P = a.size
        v = self._vec
        d = self._descriptor(batch, perm, n)
        inp = eng.make_input(batch.obs, perm)
        e, nl = eng.engine(), eng.netlist([a])
        theta_a = self.arena.theta[a.offset:a.offset + P]

        n_g = self._dp_begin(n)          # rows of the global minibatch (== n on one GPU)

        def sums():
            return self._gsums()

        def grad_into(mode, dst):
            self._head(d, mode)
            sm = sums()
            eng.backward([a], n)
            _lib.check(lib.fsrl_engine_wgrad_to(ctypes.byref(e), ctypes.byref(nl), ctypes.byref(inp), n, dst.data_ptr(), s))
            self._gvec(dst)
            return sm

        # entropy of the state-independent Gaussian BEFORE the step (:239)
        ent = self._entropy()
        eng.forward([a], inp, n, save=True)
        sm = grad_into(1, v["g"])                                                   # :252
        adv_c = batch.adv[1] if perm is None else batch.adv[1][perm.long()]
        mean_adv_c = self._gscalar(float(adv_c.sum().item())) / n_g if self._dpw is not None else float(adv_c.mean().item())
        objective = np.float32(sm[0] / n_g)
        cost_surrogate = np.float32(self._ave_cost_return + sm[1] / n_g - mean_adv_c)  # :169-175
        kl = np.float32(sm[2] / n_g)
        grad_into(2, v["b"])                                                         # :253
        self._head(d, 3)                                                             # :254 (graph of grad kl)
        eng.backward([a], n)
        self._cg(d, v["g"], v["Hinv_g"])                                             # :255
        self._hvp(d, v["Hinv_g"], v["hv"])                                           # :256 approx_g
        approx_g = v["hv"].clone()
        c_value = np.float32(cost_surrogate - np.float32(self._cost_limit))          # :257
        EPS = 1e-8
        f32 = np.float32
        bb = self._dotp(v["b"], v["b"])
        if bb <= EPS and c_value < 0:                                                # :261-266
            v["Hinv_b"].zero_()
            scalar_r = scalar_s = A_value = B_value = f32(0)
            scalar_q = f32(self._dotp(approx_g, v["Hinv_g"]))
            optim_case = 4
        else:
            self._cg(d, v["b"], v["Hinv_b"])                                         # :268
            self._hvp(d, v["Hinv_b"], v["hv"])                                       # :269 approx_b
            scalar_q = f32(self._dotp(approx_g, v["Hinv_g"]))
            scalar_r = f32(self._dotp(approx_g, v["Hinv_b"]))
            scalar_s = f32(self._dotp(v["hv"], v["Hinv_b"]))
            A_value = f32(scalar_q - scalar_r ** 2 / scalar_s)                       # :275
            B_value = f32(2 * self._delta - c_value ** 2 / scalar_s)                 # :277
            if c_value < 0 and B_value < 0:
                optim_case = 3
            elif c_value < 0 and B_value >= 0:
                optim_case = 2
            elif c_value >= 0 and B_value >= 0:
                optim_case = 1
            else:
                optim_case = 0
        with np.errstate(invalid="ignore", divide="ignore"):
            if optim_case in [3, 4]:                                                 # :287-289
                lam = f32(np.sqrt(scalar_q / (2 * self._delta)))
                nu = f32(0)
            elif optim_case in [1, 2]:                                               # :291-301
                LA, LB = [0, scalar_r / c_value], [scalar_r / c_value, np.inf]
                LA, LB = (LA, LB) if c_value < 0 else (LB, LA)
                proj = lambda x, L: max(L[0], min(L[1], x))
                lam_a = proj(f32(np.sqrt(A_value / B_value)), LA)
                lam_b = proj(f32(np.sqrt(scalar_q / (2 * self._delta))), LB)
                f_a = lambda lam: -0.5 * (A_value / (lam + EPS) + B_value * lam) - scalar_r * c_value / (scalar_s + EPS)
                f_b = lambda lam: -0.5 * (scalar_q / (lam + EPS) + 2 * self._delta * lam)
                lam = f32(lam_a if f_a(lam_a) >= f_b(lam_b) else lam_b)
                nu = f32(max(0, float(lam * c_value - scalar_r)) / (scalar_s + EPS))
            else:                                                                    # :303-304
                nu = f32(np.sqrt(2 * self._delta / (scalar_s + EPS)))
                lam = f32(0)
        # ---- line search (:306-333) --------------------------------------------------------------------------
        step = v["step"]
        if optim_case > 0:
            _lib.check(lib.fsrl_vec_add_scaled(v["Hinv_g"].data_ptr(), float(nu), v["Hinv_b"].data_ptr(), step.data_ptr(), P, s))
            step.mul_(float(1.0 / (lam + EPS)))
        else:
            step.copy_(v["Hinv_b"]).mul_(float(nu))
        nrm = np.sqrt(self._dotp(step, step))
        step.div_(float(nrm))                                                        # :310
        beta = 1.0
        if not np.isnan(lam):
            v["theta0"].copy_(theta_a)
            for _ in range(self._max_backtracks):
                _lib.check(lib.fsrl_vec_add_scaled(v["theta0"].data_ptr(), beta, step.data_ptr(), theta_a.data_ptr(), P, s))
                eng.forward([a], inp, n, save=False)
                self._head(d, 0)
                sm2 = sums()
                new_kl = f32(sm2[2] / n_g)
                new_obj = f32(sm2[0] / n_g)
                new_cost = f32(self._ave_cost_return + sm2[1] / n_g - mean_adv_c)
                if new_kl <= self._delta and (new_obj > objective if optim_case > 1 else True) and \
                        new_cost - cost_surrogate <= max(-float(c_value), 0):
                    break
                beta *= self._backtrack_coeff
            eng.sync_mirror([a])
        return {"loss/kl": float(kl), "loss/entropy": ent, "loss/rew_loss": float(objective),
                "loss/cost_loss": float(cost_surrogate), "loss/optim_A": float(A_value),
                "loss/optim_B": float(B_value), "loss/optim_C": float(c_value), "loss/optim_Q": float(scalar_q),
                "loss/optim_R": float(scalar_r), "loss/optim_S": float(scalar_s), "loss/optim_lam": float(lam),
                "loss/optim_nu": float(nu), "loss/optim_case": optim_case, "loss/step_size": beta}

    def learn(self, batch: DeviceBatch, batch_size: int, repeat: int, **kwargs: Any) -> Dict[str, List[float]]:
        n_all = batch.n
        self._ensure_engine(n_all)
        self.last_stats = {}
        with torch.cuda.device(self.device):
            for _ in range(repeat):
                minibatches = self._minibatches(n_all, batch_size)
                self._dp_same_count(len(minibatches), "minibatch count")
                for perm, n in minibatches:
                    for _ in range(self._optim_critic_iters):                        # :360-361
                        stats_critic = self.critics_loss(batch, perm, n)
                    stats_actor = self.policy_loss(batch, perm, n)                   # :364
                    self.gradient_steps += 1
                    self._record({**stats_actor, **stats_critic})
        self.logger.store(gradient_steps=self.gradient_steps, tab="update")
