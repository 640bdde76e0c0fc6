"""Optimizer state for the fused Adam kernel (csrc/ppo.cu adam_kernel).  Keeps the
``torch.optim.Adam`` hyper-parameter surface (lr, betas, eps; ``param_groups`` for lr
schedulers) while the moments live in two flat device tensors next to the parameter arena."""
from __future__ import annotations

import torch


class FusedAdam:
    def __init__(self, params=None, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8):
        self.defaults = dict(lr=lr, betas=tuple(betas), eps=eps)
        self.param_groups = [dict(self.defaults, params=list(params) if params is not None else [])]
        self.step_count = 0
        self.m = None
        self.v = None

    @classmethod
    def from_optimizer(cls, opt) -> "FusedAdam":
        """``opt`` itself if it is a FusedAdam; otherwise a FusedAdam with the lr, betas and eps of its first
        parameter group, so that a ``torch.optim.Adam`` built by reference-style agent code keeps its
        hyper-parameters while the update runs in the fused kernel."""
        if isinstance(opt, FusedAdam):
            return opt
        g = opt.param_groups[0]
        return cls(lr=g["lr"], betas=g.get("betas", (0.9, 0.999)), eps=g.get("eps", 1e-8))

    @property
    def lr(self):
        return self.param_groups[0]["lr"]

    def attach(self, arena):
        self.m = torch.zeros_like(arena.theta)
        self.v = torch.zeros_like(arena.theta)

    def zero_grad(self, set_to_none: bool = False):
        pass   # gradients are fully overwritten by the wgrad kernel each step

    def state_dict(self):
        return {"step": self.step_count, "exp_avg": self.m, "exp_avg_sq": self.v,
                "param_groups": [{k: v for k, v in g.items() if k != "params"} for g in self.param_groups]}

    def load_state_dict(self, sd):
        self.step_count = int(sd["step"])
        self.m.copy_(sd["exp_avg"]); self.v.copy_(sd["exp_avg_sq"])
        for g, s in zip(self.param_groups, sd["param_groups"]):
            g.update(s)
