"""Train PPO-Lagrangian on SafetyHalfCheetahVelocityGymnasium-v1 with normalized observations, tianshou's
MuJoCo recipe: the training envs are wrapped by ``VectorEnvNormObs`` (their running statistics update on the GPU),
``learn`` normalizes the test envs with the training statistics, frozen, and the checkpoint carries them as
``"obs_rms"``.  The script then reloads the checkpoint into fresh wrapped envs and evaluates it.

  python examples/train_norm_obs.py --epoch 2 --training_num 16
"""
import argparse
import os
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from fsrl_b200 import envs  # noqa: E402
from fsrl_b200.agent import PPOLagAgent  # noqa: E402
from fsrl_b200.envs import DeviceVectorEnv, VectorEnvNormObs  # noqa: E402
from fsrl_b200.utils.logger import BaseLogger  # noqa: E402


def main(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--task", default="SafetyHalfCheetahVelocityGymnasium-v1")
    p.add_argument("--epoch", type=int, default=100)
    p.add_argument("--step_per_epoch", type=int, default=20000)
    p.add_argument("--training_num", type=int, default=20)
    p.add_argument("--testing_num", type=int, default=2)
    p.add_argument("--seed", type=int, default=10)
    p.add_argument("--logdir", default=None)
    args = p.parse_args(argv)

    logdir = args.logdir or tempfile.mkdtemp(prefix="train_norm_obs_")
    logger = BaseLogger(logdir, log_txt=True, name="ppol_norm_obs")
    agent = PPOLagAgent(envs.make(args.task), logger, cost_limit=25, seed=args.seed, hidden_sizes=(64, 64))
    train_envs = VectorEnvNormObs(DeviceVectorEnv(args.task, args.training_num, seed=args.seed))
    test_envs = DeviceVectorEnv(args.task, args.testing_num, seed=args.seed + 1)
    agent.learn(train_envs, test_envs, epoch=args.epoch, episode_per_collect=args.training_num,
                step_per_epoch=args.step_per_epoch, testing_num=args.testing_num, save_interval=1, verbose=False,
                show_progress=False)

    ckpt = torch.load(os.path.join(logger.log_dir, "checkpoint", "model.pt"), weights_only=False)
    eval_envs = VectorEnvNormObs(DeviceVectorEnv(args.task, args.testing_num, seed=args.seed + 1),
                                 update_obs_rms=False)
    eval_envs.get_obs_rms().load_state_dict(ckpt["obs_rms"])
    rew, length, cost = agent.evaluate(eval_envs, ckpt["model"], eval_episodes=args.testing_num)
    print(f"reloaded checkpoint: reward {rew:.3f}, length {length:.1f}, cost {cost:.3f}, "
          f"obs_rms count {eval_envs.get_obs_rms().count}")
    return rew, length, cost


if __name__ == "__main__":
    main()
