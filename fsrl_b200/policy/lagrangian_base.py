"""PID-Lagrangian policy base (reference: /root/reference/fsrl/policy/lagrangian_base.py).
The multiplier is a host scalar updated once per collect (:98-120); the fused loss kernels
receive lambda and the rescaling factor 1/(sum(lambda)+1) (:156) as launch arguments, and the
``loss/*`` statistics of ``safety_loss`` (:158-165) are reconstructed from the per-minibatch
device statistics."""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple, Union

import numpy as np

from ..utils.logger import BaseLogger, DummyLogger
from ..utils.optim_util import LagrangianOptimizer
from .base_policy import BasePolicy


class LagrangianPolicy(BasePolicy):
    def __init__(self, actor, critics, dist_fn=None, logger: BaseLogger = DummyLogger(),
                 use_lagrangian: bool = True, lagrangian_pid: Tuple = (0.05, 0.0005, 0.1),
                 cost_limit: Union[List, float] = np.inf, rescaling: bool = True,
                 gamma: float = 0.99, max_batchsize: int = 99999,
                 reward_normalization: bool = False, deterministic_eval: bool = True,
                 action_scaling: bool = True, action_bound_method: str = "clip",
                 observation_space=None, action_space=None, lr_scheduler=None) -> None:
        super().__init__(actor, critics, dist_fn, logger, gamma, max_batchsize,
                         reward_normalization, deterministic_eval, action_scaling,
                         action_bound_method, observation_space, action_space, lr_scheduler)
        self.rescaling = rescaling
        self.use_lagrangian = use_lagrangian
        self.cost_limit = self._expand_cost_limit(cost_limit)
        if self.use_lagrangian:
            assert len(self.cost_limit) == (self.critics_num - 1), \
                "cost_limit must has equal len of critics_num"
            self.lag_optims = [LagrangianOptimizer(lagrangian_pid) for _ in range(self.critics_num - 1)]
        else:
            self.lag_optims = []

    def pre_update_fn(self, stats_train: Dict, **kwarg) -> None:
        self.update_lagrangian(stats_train["cost"])

    def update_cost_limit(self, cost_limit: float) -> None:
        self.cost_limit = self._expand_cost_limit(cost_limit)

    def update_lagrangian(self, cost_values: Union[List, float]) -> None:
        if np.isscalar(cost_values):
            cost_values = [cost_values]
        for i, lag_optim in enumerate(self.lag_optims):
            lag_optim.step(cost_values[i], self.cost_limit[i])

    def get_extra_state(self):
        if len(self.lag_optims):
            return [optim.state_dict() for optim in self.lag_optims]
        return None

    def set_extra_state(self, state):
        # torch hands us exactly what get_extra_state returned; the reference additionally
        # accepts a dict holding it under "_extra_state" (:139-143)
        if isinstance(state, dict) and "_extra_state" in state:
            state = state["_extra_state"]
        if state and self.lag_optims:
            for i, sd in enumerate(state):
                self.lag_optims[i].load_state_dict(sd)

    def safety_loss(self, values: List) -> Tuple["torch.Tensor", dict]:
        """Host-side twin of the term the fused update kernels apply (lagrangian_base.py:145-166): the
        lambda-weighted means of the constrained quantities ``values`` (one tensor per cost stream), plus
        the statistics the reference logs -- the rescaling factor 1 / (sum(lambda) + 1) (Stooke et al.,
        Alg. 1) and, per stream, the multiplier and its loss term (suffix "_i" for i >= 1)."""
        import torch
        lams = [opt.get_lag() for opt in self.lag_optims]
        assert len(values) == len(lams), "lags and values length must be equal"
        stats = {"loss/rescaling": 1. / (np.sum(lams) + 1) if self.rescaling else 1}
        total = 0.
        for i, (value, lam) in enumerate(zip(values, lams)):
            term = torch.mean(value * lam)
            total = total + term
            tag = "" if i == 0 else f"_{i}"
            stats["loss/lagrangian" + tag] = lam
            stats["loss/actor_safety" + tag] = term.item()
        return total, stats

    def lagrangians(self) -> List[float]:
        return [float(o.get_lag()) for o in self.lag_optims]

    def rescaling_factor(self) -> float:
        lags = self.lagrangians()
        return 1.0 / (float(np.sum(lags)) + 1.0) if self.rescaling else 1.0
