"""Training configurations with the reference's field names and defaults
(/root/reference/fsrl/config/{ppol,cpo,sacl,ddpgl,trpol,focosp,cvpo}_cfg.py, SURVEY.md Appendix E), generated from
one compact table so that the CLI/YAML surface of ``examples/`` keeps working.  Pure data."""
from __future__ import annotations

import types
from dataclasses import field, make_dataclass
from typing import Any, Dict, Tuple

_COMMON_TAIL = dict(buffer_size=100000, worker="ShmemVectorEnv", testing_num=2, reward_threshold=10000,
                    save_interval=4, resume=False, save_ckpt=True, verbose=True, render=False, logdir="logs",
                    project="fast-safe-rl", group=None, name=None, suffix="")
_HEAD = dict(task="SafetyCarCircle-v0", cost_limit=10, device="cpu", thread=4, seed=10)

_TABLES: Dict[str, Dict[str, Any]] = {
    "ppol": dict(_HEAD, lr=5e-4, hidden_sizes=(128, 128), unbounded=False, last_layer_scale=False,
                 target_kl=0.02, vf_coef=0.25, max_grad_norm=0.5, gae_lambda=0.95, eps_clip=0.2,
                 dual_clip=None, value_clip=False, norm_adv=True, recompute_adv=False, use_lagrangian=True,
                 lagrangian_pid=(0.05, 0.0005, 0.1), rescaling=True, gamma=0.99, max_batchsize=100000,
                 rew_norm=False, deterministic_eval=True, action_scaling=True, action_bound_method="clip",
                 epoch=200, episode_per_collect=20, step_per_epoch=10000, repeat_per_collect=4,
                 training_num=20, batch_size=256, prefix="ppol", **_COMMON_TAIL),
    "cpo": dict(_HEAD, lr=1e-3, hidden_sizes=(128, 128), unbounded=False, last_layer_scale=False,
                target_kl=0.01, backtrack_coeff=0.8, damping_coeff=0.1, max_backtracks=100,
                optim_critic_iters=10, l2_reg=0.001, gae_lambda=0.95, norm_adv=True, gamma=0.99,
                max_batchsize=99999, rew_norm=False, deterministic_eval=True, action_scaling=True,
                action_bound_method="clip", epoch=200, episode_per_collect=20, step_per_epoch=10000,
                repeat_per_collect=4, training_num=20, batch_size=99999, prefix="cpo", **_COMMON_TAIL),
    "sacl": dict(_HEAD, actor_lr=5e-4, critic_lr=1e-3, hidden_sizes=(128, 128), auto_alpha=True,
                 alpha_lr=3e-4, alpha=0.005, tau=0.05, n_step=2, conditioned_sigma=True, unbounded=False,
                 last_layer_scale=False, use_lagrangian=True, lagrangian_pid=(0.05, 0.0005, 0.1),
                 rescaling=True, gamma=0.97, deterministic_eval=True, action_scaling=True,
                 action_bound_method="clip", epoch=200, episode_per_collect=2, step_per_epoch=10000,
                 update_per_step=0.2, training_num=10, batch_size=256, prefix="sacl", **_COMMON_TAIL),
    "ddpgl": dict(_HEAD, actor_lr=5e-4, critic_lr=1e-3, hidden_sizes=(128, 128), tau=0.05,
                  exploration_noise=0.1, n_step=2, use_lagrangian=True, lagrangian_pid=(0.05, 0.0005, 0.1),
                  rescaling=True, gamma=0.97, deterministic_eval=True, action_scaling=True,
                  action_bound_method="clip", epoch=200, episode_per_collect=2, step_per_epoch=10000,
                  update_per_step=0.2, training_num=10, batch_size=256, prefix="ddpgl", **_COMMON_TAIL),
    "trpol": dict(_HEAD, lr=5e-4, hidden_sizes=(128, 128), unbounded=False, last_layer_scale=False,
                  target_kl=0.001, backtrack_coeff=0.8, max_backtracks=10, optim_critic_iters=20,
                  gae_lambda=0.95, norm_adv=True, use_lagrangian=True, lagrangian_pid=(0.05, 0.0005, 0.1),
                  rescaling=True, gamma=0.99, max_batchsize=99999, rew_norm=False, deterministic_eval=True,
                  action_scaling=True, action_bound_method="clip", epoch=200, episode_per_collect=20,
                  step_per_epoch=10000, repeat_per_collect=4, training_num=20, batch_size=99999,
                  prefix="trpol", **_COMMON_TAIL),
    # the reference spells this module `focosp_cfg` (fsrl/config/focosp_cfg.py); both names resolve
    "focops": dict(_HEAD, actor_lr=5e-4, critic_lr=1e-3, hidden_sizes=(128, 128), unbounded=False,
                   last_layer_scale=False, auto_nu=True, nu=0, nu_max=2.0, nu_lr=1e-2, l2_reg=0.001,
                   delta=0.02, eta=0.02, max_grad_norm=0.5, tem_lambda=0.95, gae_lambda=0.95, norm_adv=True,
                   recompute_adv=False, gamma=0.99, max_batchsize=100000, rew_norm=False,
                   deterministic_eval=True, action_scaling=True, action_bound_method="clip", epoch=200,
                   episode_per_collect=20, step_per_epoch=10000, repeat_per_collect=4, training_num=20,
                   batch_size=256, prefix="focops", **_COMMON_TAIL),
    "cvpo": dict(_HEAD, estep_iter_num=1, estep_kl=0.02, estep_dual_max=20, estep_dual_lr=0.02, sample_act_num=16,
                 mstep_iter_num=1, mstep_kl_mu=0.005, mstep_kl_std=0.0005, mstep_dual_max=0.5, mstep_dual_lr=0.1,
                 actor_lr=5e-4, critic_lr=1e-3, gamma=0.97, n_step=2, tau=0.05, hidden_sizes=(128, 128),
                 double_critic=False, conditioned_sigma=True, unbounded=False, last_layer_scale=False, epoch=200,
                 episode_per_collect=10, step_per_epoch=10000, update_per_step=0.2, buffer_size=200000,
                 worker="ShmemVectorEnv", training_num=20, testing_num=2, batch_size=256, reward_threshold=10000,
                 save_interval=4, deterministic_eval=True, action_scaling=True, action_bound_method="clip",
                 resume=False, save_ckpt=True, verbose=False, render=False, logdir="logs", project="fast-safe-rl",
                 group=None, name=None, prefix="cvpo", suffix=""),
}
# per-suite overrides (class name -> changed fields); off-policy Mujoco adds gamma / n_step / buffer
_ON_MUJOCO = dict(task="SafetyPointCircle1Gymnasium-v0", epoch=250, cost_limit=25, episode_per_collect=20,
                  step_per_epoch=20000, repeat_per_collect=4)
_OFF_MUJOCO = dict(task="SafetyPointCircle1Gymnasium-v0", epoch=250, cost_limit=25, gamma=0.99, n_step=3,
                   step_per_epoch=20000, buffer_size=800000)
# CVPO's Mujoco suite (cvpo_cfg.py) has its own base and per-class overrides, and a Mujoco5MCfg
_CVPO_MUJOCO = dict(task="SafetyPointCircle1Gymnasium-v0", epoch=250, cost_limit=25, unbounded=True, gamma=0.995,
                    n_step=3, step_per_epoch=20000, buffer_size=200000)
_CVPO_MUJOCO_CLASSES = (("Mujoco2MCfg", dict(epoch=100)),
                        ("Mujoco5MCfg", dict(epoch=250, unbounded=False, gamma=0.98, n_step=3, buffer_size=40000)),
                        ("Mujoco20MCfg", dict(epoch=1000, sample_act_num=64)),
                        ("Mujoco10MCfg", dict(epoch=500, unbounded=False, gamma=0.98, sample_act_num=32)))


def _dc(name, fields: Dict[str, Any], base=None):
    spec = []
    for k, v in fields.items():
        default = field(default_factory=(lambda v=v: v)) if isinstance(v, (list, dict)) else v
        spec.append((k, Any if v is None else type(v), default))
    return make_dataclass(name, spec, bases=(base,) if base else ())


def _module(key: str) -> types.ModuleType:
    m = types.ModuleType(f"fsrl_b200.config.{key}_cfg")
    base = _dc("TrainCfg", _TABLES[key])
    m.TrainCfg = base
    for nm, ep in (("Bullet1MCfg", 100), ("Bullet5MCfg", 500), ("Bullet10MCfg", 1000)):
        setattr(m, nm, _dc(nm, {"epoch": ep}, base))
    if key == "cvpo":
        mj = m.MujocoBaseCfg = _dc("MujocoBaseCfg", _CVPO_MUJOCO, base)
        for nm, over in _CVPO_MUJOCO_CLASSES:
            setattr(m, nm, _dc(nm, over, mj))
        return m
    mj = _dc("MujocoBaseCfg", _ON_MUJOCO if key in ("ppol", "cpo", "trpol", "focops") else _OFF_MUJOCO, base)
    m.MujocoBaseCfg = mj
    for nm, ep in (("Mujoco2MCfg", 100), ("Mujoco10MCfg", 500), ("Mujoco20MCfg", 1000)):
        setattr(m, nm, _dc(nm, {"epoch": ep}, mj))
    return m


ppol_cfg, cpo_cfg, sacl_cfg, ddpgl_cfg, trpol_cfg, focops_cfg, cvpo_cfg = (
    _module(k) for k in ("ppol", "cpo", "sacl", "ddpgl", "trpol", "focops", "cvpo"))
focosp_cfg = focops_cfg
