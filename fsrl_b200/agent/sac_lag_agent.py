"""SAC-Lagrangian agent preset (reference: /root/reference/fsrl/agent/sac_lag_agent.py:75-200)."""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np
import torch

from ..nets import ActorProb, DoubleCritic, Net
from ..optim import FusedAdam
from ..policy import SACLagrangian
from ..utils.logger import BaseLogger, DummyLogger
from .base_agent import OffpolicyAgent
from .ppo_lag_agent import init_actor_critic


class SACLagAgent(OffpolicyAgent):
    name = "SACLagAgent"

    def __init__(self, env, logger: BaseLogger = DummyLogger(), cost_limit: float = 10,
                 device: str = "cuda", thread: int = 4, seed: int = 10, actor_lr: float = 5e-4,
                 critic_lr: float = 1e-3, hidden_sizes: Tuple[int, ...] = (128, 128),
                 auto_alpha: bool = True, alpha_lr: float = 3e-4, alpha: float = 0.002, tau: float = 0.05,
                 n_step: int = 2, use_lagrangian: bool = True,
                 lagrangian_pid: Tuple = (0.05, 0.0005, 0.1), rescaling: bool = True, gamma: float = 0.99,
                 conditioned_sigma: bool = True, unbounded: bool = True, last_layer_scale: bool = False,
                 deterministic_eval: bool = False, action_scaling: bool = True,
                 action_bound_method: str = "clip", lr_scheduler=None) -> None:
        super().__init__()
        device = self._prologue(logger, cost_limit, seed, thread, device)
        cost_dim = 1 if np.isscalar(cost_limit) else len(cost_limit)
        state_shape, action_shape = env.observation_space.shape, env.action_space.shape
        max_action = float(env.action_space.high[0])
        actor = ActorProb(Net(state_shape, hidden_sizes=hidden_sizes, device=device), action_shape,
                          max_action=max_action, device=device, conditioned_sigma=conditioned_sigma,
                          unbounded=unbounded)
        critics = [DoubleCritic(Net(state_shape, action_shape, hidden_sizes=hidden_sizes, concat=True, device=device),
                                Net(state_shape, action_shape, hidden_sizes=hidden_sizes, concat=True, device=device),
                                device=device) for _ in range(1 + cost_dim)]
        init_actor_critic(actor, critics, last_layer_scale)
        a = alpha
        if auto_alpha:
            target_entropy = -float(np.prod(env.action_space.shape))
            a = (target_entropy, torch.zeros(1), FusedAdam(lr=alpha_lr))
        self._adopt_policy(SACLagrangian(
            actor=actor, critics=critics, actor_optim=FusedAdam(lr=actor_lr), critic_optim=FusedAdam(lr=critic_lr),
            logger=logger, alpha=a, tau=tau, gamma=gamma, exploration_noise=None, n_step=n_step,
            use_lagrangian=use_lagrangian, lagrangian_pid=lagrangian_pid, cost_limit=cost_limit,
            rescaling=rescaling, reward_normalization=False, deterministic_eval=deterministic_eval,
            action_scaling=action_scaling, action_bound_method=action_bound_method,
            observation_space=env.observation_space, action_space=env.action_space,
            lr_scheduler=lr_scheduler), seed)
        self.policy.set_update_seed(seed + 1)
