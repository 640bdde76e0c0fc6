"""DDPG-Lagrangian agent preset (reference: /root/reference/fsrl/agent/ddpg_lag_agent.py:66-160)."""
from __future__ import annotations

from typing import Tuple

import numpy as np

from ..nets import Actor, Critic, Net
from ..optim import FusedAdam
from ..policy import DDPGLagrangian, GaussianNoise
from ..utils.logger import BaseLogger, DummyLogger
from .base_agent import OffpolicyAgent
from .ppo_lag_agent import init_actor_critic


class DDPGLagAgent(OffpolicyAgent):
    name = "DDPGLagAgent"

    def __init__(self, env, logger: BaseLogger = DummyLogger(), cost_limit: float = 10,
                 device: str = "cuda", thread: int = 4, seed: int = 10, actor_lr: float = 1e-4,
                 critic_lr: float = 1e-3, hidden_sizes: Tuple[int, ...] = (128, 128), tau: float = 0.005,
                 exploration_noise: float = 0.1, n_step: int = 3, use_lagrangian: bool = True,
                 lagrangian_pid: Tuple = (0.5, 0.001, 0.1), rescaling: bool = True, gamma: float = 0.99,
                 deterministic_eval: bool = True, action_scaling: bool = True,
                 action_bound_method: str = "clip", lr_scheduler=None) -> None:
        super().__init__()
        device = self._prologue(logger, cost_limit, seed, thread, device)
        cost_dim = 1 if np.isscalar(cost_limit) else len(cost_limit)
        state_shape, action_shape = env.observation_space.shape, env.action_space.shape
        max_action = float(env.action_space.high[0])
        actor = Actor(Net(state_shape, hidden_sizes=hidden_sizes, device=device), action_shape,
                      max_action=max_action, device=device)
        critics = [Critic(Net(state_shape, action_shape, hidden_sizes=hidden_sizes, concat=True, device=device),
                          device=device) for _ in range(cost_dim + 1)]
        init_actor_critic(actor, critics)
        self._adopt_policy(DDPGLagrangian(
            actor=actor, critics=critics, actor_optim=FusedAdam(lr=actor_lr), critic_optim=FusedAdam(lr=critic_lr),
            logger=logger, tau=tau, exploration_noise=GaussianNoise(sigma=exploration_noise), n_step=n_step,
            use_lagrangian=use_lagrangian, lagrangian_pid=lagrangian_pid, cost_limit=cost_limit,
            rescaling=rescaling, gamma=gamma, reward_normalization=False,
            deterministic_eval=deterministic_eval, action_scaling=action_scaling,
            action_bound_method=action_bound_method, observation_space=env.observation_space,
            action_space=env.action_space, lr_scheduler=lr_scheduler), seed)
        self.policy.set_update_seed(seed + 1)
