"""CPO agent preset (reference: /root/reference/fsrl/agent/cpo_agent.py:69-175): the optimiser
holds ONLY the critic parameters (:148); the actor moves by the trust-region step."""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np
import torch
from torch.distributions import Independent, Normal

from ..nets import ActorProb, Critic, Net
from ..optim import FusedAdam
from ..policy import CPO
from ..utils.logger import BaseLogger, DummyLogger
from .base_agent import OnpolicyAgent
from .ppo_lag_agent import init_actor_critic


class CPOAgent(OnpolicyAgent):
    name = "CPOAgent"

    def __init__(self, env, logger: BaseLogger = DummyLogger(), cost_limit: float = 10,
                 device: str = "cuda", thread: int = 4, seed: int = 10, lr: float = 1e-3,
                 hidden_sizes: Tuple[int, ...] = (128, 128), unbounded: bool = False,
                 last_layer_scale: bool = False, target_kl: float = 0.01, backtrack_coeff: float = 0.8,
                 damping_coeff: float = 0.1, max_backtracks: int = 10, optim_critic_iters: int = 10,
                 l2_reg: float = 0.001, gae_lambda: float = 0.95, advantage_normalization: bool = True,
                 gamma: float = 0.99, max_batchsize: int = 99999, reward_normalization: bool = False,
                 deterministic_eval: bool = True, action_scaling: bool = True,
                 action_bound_method: str = "clip", lr_scheduler=None) -> None:
        super().__init__()
        device = self._prologue(logger, cost_limit, seed, thread, device)
        state_shape, action_shape = env.observation_space.shape, env.action_space.shape
        max_action = float(env.action_space.high[0])
        actor = ActorProb(Net(state_shape, hidden_sizes=hidden_sizes, device=device), action_shape,
                          max_action=max_action, unbounded=unbounded, device=device)
        critics = [Critic(Net(state_shape, hidden_sizes=hidden_sizes, device=device), device=device) for _ in range(2)]
        torch.nn.init.constant_(actor.sigma_param, -0.5)
        init_actor_critic(actor, critics, last_layer_scale)
        self._adopt_policy(CPO(
            actor, critics, FusedAdam(lr=lr), lambda *l: Independent(Normal(*l), 1), logger=logger,
            target_kl=target_kl, backtrack_coeff=backtrack_coeff, damping_coeff=damping_coeff,
            max_backtracks=max_backtracks, optim_critic_iters=optim_critic_iters, l2_reg=l2_reg,
            gae_lambda=gae_lambda, advantage_normalization=advantage_normalization,
            cost_limit=cost_limit, gamma=gamma, max_batchsize=max_batchsize,
            reward_normalization=reward_normalization, deterministic_eval=deterministic_eval,
            action_scaling=action_scaling, action_bound_method=action_bound_method,
            observation_space=env.observation_space, action_space=env.action_space,
            lr_scheduler=lr_scheduler), seed)

    def learn(self, train_envs, test_envs=None, epoch: int = 300, episode_per_collect: int = 20,
              step_per_epoch: int = 10000, repeat_per_collect: int = 4, buffer_size: int = 100000,
              testing_num: int = 2, batch_size: int = 99999, reward_threshold: float = 450,
              save_interval: int = 4, resume: bool = False, save_ckpt: bool = True,
              verbose: bool = True, show_progress: bool = True):
        """Same protocol as OnpolicyAgent.learn; the trust-region step wants the whole collect as ONE batch, hence
        the reference's default batch_size = 99999 (cpo_agent.py:183-206)."""
        return super().learn(train_envs, test_envs, epoch, episode_per_collect, step_per_epoch, repeat_per_collect,
                             buffer_size, testing_num, batch_size, reward_threshold, save_interval, resume, save_ckpt,
                             verbose, show_progress)
