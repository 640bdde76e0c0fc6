"""Train any of the hot-path agents through the REFERENCE'S import names (fsrl / tianshou /
gymnasium / pyrallis), resolved by ``fsrl_b200.compat`` to the device engine -- the flow of the
reference's ``examples/mlp/train_*_agent.py`` (config dataclass <- CLI, ``gym.make`` demo env,
``worker([...])`` vector envs, ``agent.learn(...)``).

  python examples/train_agent.py --algo ppol --task SafetyCarCircle-v0 --epoch 2 --training_num 64
"""
import os
import sys
import types
from dataclasses import asdict

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import fsrl_b200.compat  # noqa: E402

fsrl_b200.compat.install()

import bullet_safety_gym  # noqa: E402,F401  (task registration side effect in the reference)
import gymnasium as gym  # noqa: E402
from tianshou.env import ShmemVectorEnv, SubprocVectorEnv  # noqa: E402,F401

from fsrl.agent import CPOAgent, CVPOAgent, DDPGLagAgent, FOCOPSAgent, PPOLagAgent, SACLagAgent, TRPOLagAgent  # noqa: E402
from fsrl.config import cpo_cfg, cvpo_cfg, ddpgl_cfg, focosp_cfg, ppol_cfg, sacl_cfg, trpol_cfg  # noqa: E402
from fsrl.utils import BaseLogger  # noqa: E402
from fsrl.utils.exp_util import auto_name  # noqa: E402

ALGOS = {
    "ppol": (ppol_cfg, PPOLagAgent, dict(lr="lr", hidden_sizes="hidden_sizes", unbounded="unbounded",
             last_layer_scale="last_layer_scale", target_kl="target_kl", vf_coef="vf_coef",
             max_grad_norm="max_grad_norm", gae_lambda="gae_lambda", eps_clip="eps_clip", dual_clip="dual_clip",
             value_clip="value_clip", advantage_normalization="norm_adv", recompute_advantage="recompute_adv",
             use_lagrangian="use_lagrangian", lagrangian_pid="lagrangian_pid", rescaling="rescaling",
             gamma="gamma", max_batchsize="max_batchsize", reward_normalization="rew_norm")),
    "cpo": (cpo_cfg, CPOAgent, dict(lr="lr", hidden_sizes="hidden_sizes", unbounded="unbounded",
            last_layer_scale="last_layer_scale", target_kl="target_kl", backtrack_coeff="backtrack_coeff",
            damping_coeff="damping_coeff", max_backtracks="max_backtracks", optim_critic_iters="optim_critic_iters",
            l2_reg="l2_reg", gae_lambda="gae_lambda", advantage_normalization="norm_adv", gamma="gamma",
            max_batchsize="max_batchsize", reward_normalization="rew_norm")),
    "sacl": (sacl_cfg, SACLagAgent, dict(actor_lr="actor_lr", critic_lr="critic_lr", hidden_sizes="hidden_sizes",
             auto_alpha="auto_alpha", alpha_lr="alpha_lr", alpha="alpha", tau="tau", n_step="n_step",
             conditioned_sigma="conditioned_sigma", unbounded="unbounded", last_layer_scale="last_layer_scale",
             use_lagrangian="use_lagrangian", lagrangian_pid="lagrangian_pid", rescaling="rescaling", gamma="gamma")),
    "trpol": (trpol_cfg, TRPOLagAgent, dict(lr="lr", hidden_sizes="hidden_sizes", unbounded="unbounded",
              last_layer_scale="last_layer_scale", target_kl="target_kl", backtrack_coeff="backtrack_coeff",
              max_backtracks="max_backtracks", optim_critic_iters="optim_critic_iters", gae_lambda="gae_lambda",
              advantage_normalization="norm_adv", use_lagrangian="use_lagrangian", lagrangian_pid="lagrangian_pid",
              rescaling="rescaling", gamma="gamma", max_batchsize="max_batchsize", reward_normalization="rew_norm")),
    "focops": (focosp_cfg, FOCOPSAgent, dict(actor_lr="actor_lr", critic_lr="critic_lr", hidden_sizes="hidden_sizes",
               unbounded="unbounded", last_layer_scale="last_layer_scale", auto_nu="auto_nu", nu="nu", nu_max="nu_max",
               nu_lr="nu_lr", l2_reg="l2_reg", delta="delta", eta="eta", tem_lambda="tem_lambda",
               gae_lambda="gae_lambda", max_grad_norm="max_grad_norm", advantage_normalization="norm_adv",
               recompute_advantage="recompute_adv", gamma="gamma", max_batchsize="max_batchsize",
               reward_normalization="rew_norm")),
    "ddpgl": (ddpgl_cfg, DDPGLagAgent, dict(actor_lr="actor_lr", critic_lr="critic_lr", hidden_sizes="hidden_sizes",
              tau="tau", exploration_noise="exploration_noise", n_step="n_step", use_lagrangian="use_lagrangian",
              lagrangian_pid="lagrangian_pid", rescaling="rescaling", gamma="gamma")),
    "cvpo": (cvpo_cfg, CVPOAgent, dict(estep_iter_num="estep_iter_num", estep_kl="estep_kl",
             estep_dual_max="estep_dual_max", estep_dual_lr="estep_dual_lr", sample_act_num="sample_act_num",
             mstep_iter_num="mstep_iter_num", mstep_kl_mu="mstep_kl_mu", mstep_kl_std="mstep_kl_std",
             mstep_dual_max="mstep_dual_max", mstep_dual_lr="mstep_dual_lr", actor_lr="actor_lr", critic_lr="critic_lr",
             gamma="gamma", n_step="n_step", tau="tau", hidden_sizes="hidden_sizes", double_critic="double_critic",
             conditioned_sigma="conditioned_sigma", unbounded="unbounded", last_layer_scale="last_layer_scale")),
}


def main(argv=None):
    import argparse
    import ast
    ap = argparse.ArgumentParser()
    ap.add_argument("--algo", default="ppol", choices=sorted(ALGOS))
    ns, rest = ap.parse_known_args(argv)
    cfg_mod, agent_cls, mapping = ALGOS[ns.algo]
    cfg = asdict(cfg_mod.TrainCfg())
    it = iter(rest)
    for tok in it:                                   # `--field value` overrides, like pyrallis
        key = tok.lstrip("-")
        val = next(it)
        try:
            cfg[key] = ast.literal_eval(val)
        except (ValueError, SyntaxError):
            cfg[key] = val
    args = types.SimpleNamespace(**cfg)
    default_cfg = asdict(cfg_mod.TrainCfg())
    if args.name is None:
        args.name = auto_name(default_cfg, cfg, args.prefix, args.suffix)
    logger = BaseLogger(args.logdir if args.save_ckpt else None, log_txt=True, name=args.name)
    logger.save_config(cfg, verbose=False)

    demo_env = gym.make(args.task)
    kw = {k: getattr(args, v) for k, v in mapping.items()}
    agent = agent_cls(env=demo_env, logger=logger, cost_limit=args.cost_limit, device=args.device,
                      thread=args.thread, seed=args.seed, deterministic_eval=args.deterministic_eval,
                      action_scaling=args.action_scaling, action_bound_method=args.action_bound_method, **kw)
    training_num = min(args.training_num, args.episode_per_collect)
    worker = eval(args.worker)
    train_envs = worker([lambda: gym.make(args.task) for _ in range(training_num)])
    test_envs = worker([lambda: gym.make(args.task) for _ in range(args.testing_num)])
    learn_kw = dict(train_envs=train_envs, test_envs=test_envs, epoch=args.epoch,
                    episode_per_collect=args.episode_per_collect, step_per_epoch=args.step_per_epoch,
                    buffer_size=args.buffer_size, testing_num=args.testing_num, batch_size=args.batch_size,
                    reward_threshold=args.reward_threshold, save_interval=args.save_interval, resume=args.resume,
                    save_ckpt=args.save_ckpt, verbose=args.verbose, show_progress=False)
    if hasattr(args, "repeat_per_collect"):
        learn_kw["repeat_per_collect"] = args.repeat_per_collect
    else:
        learn_kw["update_per_step"] = args.update_per_step
    epoch, stats, info = agent.learn(**learn_kw)
    rews, lens, cost = agent.evaluate(test_envs, eval_episodes=args.testing_num)
    print(f"done: epochs {epoch}, train_speed {info['train_speed']:.0f} env-steps/s, "
          f"eval reward {rews:.2f} cost {cost:.2f}")
    return epoch, stats, info


if __name__ == "__main__":
    main()
