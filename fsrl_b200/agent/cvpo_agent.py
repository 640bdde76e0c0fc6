"""CVPO agent preset (reference: /root/reference/fsrl/agent/cvpo_agent.py:81-230).  Networks are built and
initialised in the reference's order (actor Net, ActorProb, critics, orthogonal init over the ActorCritic,
last-layer scaling), so a seed gives the reference's initial parameters."""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np
import torch
from torch.distributions import Independent, Normal

from ..nets import ActorProb, DoubleCritic, Net, SingleCritic
from ..policy import CVPO
from ..policy.base_policy import ActorCritic
from ..utils.exp_util import seed_all
from ..utils.logger import BaseLogger, DummyLogger
from .base_agent import OffpolicyAgent


def _dist(*logits):
    return Independent(Normal(*logits), 1)


class CVPOAgent(OffpolicyAgent):
    name = "CVPOAgent"

    def __init__(self, env, logger: BaseLogger = DummyLogger(), cost_limit: float = 10, device: str = "cuda",
                 thread: int = 4, seed: int = 10, estep_iter_num: int = 1, estep_kl: float = 0.02,
                 estep_dual_max: float = 20, estep_dual_lr: float = 0.02, sample_act_num: int = 16,
                 mstep_iter_num: int = 1, mstep_kl_mu: float = 0.005, mstep_kl_std: float = 0.0005,
                 mstep_dual_max: float = 0.5, mstep_dual_lr: float = 0.1, actor_lr: float = 5e-4,
                 critic_lr: float = 1e-3, gamma: float = 0.98, n_step: int = 2, tau: float = 0.05,
                 hidden_sizes: Tuple[int, ...] = (128, 128), double_critic: bool = False,
                 conditioned_sigma: bool = True, unbounded: bool = False, last_layer_scale: bool = False,
                 deterministic_eval: bool = True, action_scaling: bool = True, action_bound_method: str = "clip",
                 lr_scheduler: Optional[torch.optim.lr_scheduler.LambdaLR] = None) -> None:
        super().__init__()
        self.logger, self.cost_limit = logger, cost_limit
        cost_dim = 1 if np.isscalar(cost_limit) else len(cost_limit)
        seed_all(seed)
        torch.set_num_threads(thread)
        if device == "cpu":
            import warnings
            warnings.warn("fsrl_b200 runs on CUDA devices only: device='cpu' is mapped to 'cuda'", RuntimeWarning, stacklevel=2)
            device = "cuda"
        state_shape, action_shape = env.observation_space.shape, env.action_space.shape
        max_action = float(env.action_space.high[0])
        assert hasattr(env.spec, "max_episode_steps"), \
            "Please use an env wrapper to provide 'max_episode_steps' for CVPO"
        actor = ActorProb(Net(state_shape, hidden_sizes=hidden_sizes, device=device), action_shape,
                          max_action=max_action, device=device, conditioned_sigma=conditioned_sigma, unbounded=unbounded)
        actor_optim = torch.optim.Adam(actor.parameters(), lr=actor_lr)
        critics = []
        for _ in range(1 + cost_dim):
            if double_critic:
                critics.append(DoubleCritic(Net(state_shape, action_shape, hidden_sizes=hidden_sizes, concat=True, device=device),
                                            Net(state_shape, action_shape, hidden_sizes=hidden_sizes, concat=True, device=device),
                                            device=device))
            else:
                critics.append(SingleCritic(Net(state_shape, action_shape, hidden_sizes=hidden_sizes, concat=True,
                                                device=device), device=device))
        critic_optim = torch.optim.Adam(torch.nn.ModuleList(critics).parameters(), lr=critic_lr)
        if not conditioned_sigma:
            torch.nn.init.constant_(actor.sigma_param, -0.5)
        for m in ActorCritic(actor, critics).modules():
            if isinstance(m, torch.nn.Linear):
                torch.nn.init.orthogonal_(m.weight)
                torch.nn.init.zeros_(m.bias)
        if last_layer_scale:
            for m in actor.mu.modules():
                if isinstance(m, torch.nn.Linear):
                    torch.nn.init.zeros_(m.bias)
                    m.weight.data.copy_(0.01 * m.weight.data)
        self.policy = CVPO(
            actor=actor, critics=critics, actor_optim=actor_optim, critic_optim=critic_optim, logger=logger,
            action_space=env.action_space, dist_fn=_dist, max_episode_steps=env.spec.max_episode_steps,
            cost_limit=cost_limit, tau=tau, gamma=gamma, n_step=n_step, estep_iter_num=estep_iter_num,
            estep_kl=estep_kl, estep_dual_max=estep_dual_max, estep_dual_lr=estep_dual_lr,
            sample_act_num=sample_act_num, mstep_iter_num=mstep_iter_num, mstep_kl_mu=mstep_kl_mu,
            mstep_kl_std=mstep_kl_std, mstep_dual_max=mstep_dual_max, mstep_dual_lr=mstep_dual_lr,
            deterministic_eval=deterministic_eval, action_scaling=action_scaling,
            action_bound_method=action_bound_method, lr_scheduler=lr_scheduler)
        self.policy.arena
        self.policy.set_action_seed(seed)
        self.policy.set_update_seed(seed + 1)
