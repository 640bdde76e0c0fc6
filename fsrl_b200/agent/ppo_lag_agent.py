"""PPO-Lagrangian agent preset (reference: /root/reference/fsrl/agent/ppo_lag_agent.py:82-200):
2x hidden MLP actor (tanh-bounded mean, state-independent log-sigma initialised to -0.5) and
one critic per return stream, orthogonal init with zero bias, one Adam over everything."""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np
import torch
from torch.distributions import Independent, Normal

from ..nets import ActorProb, Critic, Net
from ..optim import FusedAdam
from ..policy import PPOLagrangian
from ..utils.logger import BaseLogger, DummyLogger
from .base_agent import OnpolicyAgent


def init_actor_critic(actor, critics, last_layer_scale: bool = False) -> None:
    """ppo_lag_agent.py:150-161: orthogonal weights, zero biases, optional 0.01 scale of mu."""
    for mod in [actor] + list(critics):
        for m in mod.modules():
            if isinstance(m, torch.nn.Linear):
                torch.nn.init.orthogonal_(m.weight)
                torch.nn.init.zeros_(m.bias)
    if last_layer_scale:
        for m in actor.mu.modules():
            if isinstance(m, torch.nn.Linear):
                torch.nn.init.zeros_(m.bias)
                m.weight.data.copy_(0.01 * m.weight.data)


class PPOLagAgent(OnpolicyAgent):
    name = "PPOLagAgent"

    def __init__(self, env, logger: BaseLogger = DummyLogger(), cost_limit: float = 10,
                 device: str = "cuda", thread: int = 4, seed: int = 10, lr: float = 5e-4,
                 hidden_sizes: Tuple[int, ...] = (128, 128), unbounded: bool = False,
                 last_layer_scale: bool = False, target_kl: float = 0.02, vf_coef: float = 0.25,
                 max_grad_norm: Optional[float] = None, gae_lambda: float = 0.95,
                 eps_clip: float = 0.2, dual_clip: Optional[float] = None, value_clip: bool = False,
                 advantage_normalization: bool = True, recompute_advantage: bool = False,
                 use_lagrangian: bool = True, lagrangian_pid: Tuple = (0.05, 0.0005, 0.1),
                 rescaling: bool = True, gamma: float = 0.99, max_batchsize: int = 99999,
                 reward_normalization: bool = False, deterministic_eval: bool = True,
                 action_scaling: bool = True, action_bound_method: str = "clip",
                 lr_scheduler=None) -> None:
        super().__init__()
        device = self._prologue(logger, cost_limit, seed, thread, device)
        cost_dim = 1 if np.isscalar(cost_limit) else len(cost_limit)
        state_shape = env.observation_space.shape
        action_shape = env.action_space.shape
        max_action = float(env.action_space.high[0])
        actor = ActorProb(Net(state_shape, hidden_sizes=hidden_sizes, device=device), action_shape,
                          max_action=max_action, unbounded=unbounded, device=device)
        critics = [Critic(Net(state_shape, hidden_sizes=hidden_sizes, device=device), device=device)
                   for _ in range(1 + cost_dim)]
        torch.nn.init.constant_(actor.sigma_param, -0.5)
        init_actor_critic(actor, critics, last_layer_scale)
        optim = FusedAdam(lr=lr)

        def dist(*logits):
            return Independent(Normal(*logits), 1)

        self._adopt_policy(PPOLagrangian(
            actor, critics, optim, dist, logger=logger, target_kl=target_kl, vf_coef=vf_coef,
            max_grad_norm=max_grad_norm, gae_lambda=gae_lambda, eps_clip=eps_clip,
            dual_clip=dual_clip, value_clip=value_clip,
            advantage_normalization=advantage_normalization,
            recompute_advantage=recompute_advantage, use_lagrangian=use_lagrangian,
            lagrangian_pid=lagrangian_pid, cost_limit=cost_limit, rescaling=rescaling, gamma=gamma,
            max_batchsize=max_batchsize, reward_normalization=reward_normalization,
            deterministic_eval=deterministic_eval, action_scaling=action_scaling,
            action_bound_method=action_bound_method, observation_space=env.observation_space,
            action_space=env.action_space, lr_scheduler=lr_scheduler), seed)
