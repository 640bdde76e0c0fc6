"""FOCOPS agent preset (reference: /root/reference/fsrl/agent/focops_agent.py:71-198): actor and
the two critics as 2-layer MLPs (orthogonal init, log sigma = -0.5), separate Adam optimisers for
the actor and the critics, automatic nu when ``auto_nu``."""
from __future__ import annotations

from typing import Optional, Tuple

import torch
from torch.distributions import Independent, Normal

from ..nets import ActorProb, Critic, Net
from ..optim import FusedAdam
from ..policy.focops import FOCOPS
from ..utils.logger import BaseLogger, DummyLogger
from .base_agent import OnpolicyAgent
from .ppo_lag_agent import init_actor_critic


class FOCOPSAgent(OnpolicyAgent):
    name = "FOCOPSAgent"

    def __init__(self, env, logger: BaseLogger = DummyLogger(), cost_limit: float = 10, device: str = "cuda",
                 thread: int = 4, seed: int = 10, actor_lr: float = 5e-4, critic_lr: float = 1e-3,
                 hidden_sizes: Tuple[int, ...] = (128, 128), unbounded: bool = False,
                 last_layer_scale: bool = False, auto_nu: bool = True, nu: float = 0.01, nu_max: float = 2.0,
                 nu_lr: float = 1e-2, l2_reg: float = 1e-3, delta: float = 0.02, eta: float = 0.02,
                 tem_lambda: float = 0.95, gae_lambda: float = 0.95, max_grad_norm: Optional[float] = 0.5,
                 advantage_normalization: bool = True, recompute_advantage: bool = False, gamma: float = 0.99,
                 max_batchsize: int = 100000, reward_normalization: bool = False,
                 deterministic_eval: bool = True, action_scaling: bool = True,
                 action_bound_method: str = "clip", lr_scheduler=None) -> None:
        super().__init__()
        device = self._prologue(logger, cost_limit, seed, thread, device)
        state_shape, action_shape = env.observation_space.shape, env.action_space.shape
        max_action = float(env.action_space.high[0])
        actor = ActorProb(Net(state_shape, hidden_sizes=hidden_sizes, device=device), action_shape,
                          max_action=max_action, unbounded=unbounded, device=device)
        critics = [Critic(Net(state_shape, hidden_sizes=hidden_sizes, device=device), device=device)
                   for _ in range(2)]
        torch.nn.init.constant_(actor.sigma_param, -0.5)
        init_actor_critic(actor, critics, last_layer_scale)
        if auto_nu:                       # the reference starts the multiplier at 0 in auto mode (:168-170)
            nu = (nu_max, nu_lr, 0.0)
        self._adopt_policy(FOCOPS(
            actor, critics, FusedAdam(lr=actor_lr), FusedAdam(lr=critic_lr),
            lambda *l: Independent(Normal(*l), 1), logger=logger, cost_limit=cost_limit, nu=nu, l2_reg=l2_reg,
            delta=delta, eta=eta, tem_lambda=tem_lambda, gae_lambda=gae_lambda, max_grad_norm=max_grad_norm,
            advantage_normalization=advantage_normalization, recompute_advantage=recompute_advantage,
            gamma=gamma, max_batchsize=max_batchsize, reward_normalization=reward_normalization,
            deterministic_eval=deterministic_eval, action_scaling=action_scaling,
            action_bound_method=action_bound_method, observation_space=env.observation_space,
            action_space=env.action_space, lr_scheduler=lr_scheduler), seed)
