"""Train PPO-Lagrangian on a user-written env stepped on the host, through the REFERENCE'S import names
(fsrl / tianshou / gymnasium, resolved by ``fsrl_b200.compat``).  Any gymnasium-style env works the same way:
``DummyVectorEnv`` over env constructors that are not registered device tasks yields a ``HostVectorEnv``; the env
steps in this process, the actor, the action noise and the replay ring stay on the GPU.

  python examples/train_host_env.py --epoch 2 --training_num 8
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import fsrl_b200.compat  # noqa: E402

fsrl_b200.compat.install()

from gymnasium.spaces import Box  # noqa: E402
from tianshou.env import DummyVectorEnv  # noqa: E402

from fsrl.agent import PPOLagAgent  # noqa: E402


class _Spec:
    def __init__(self, id, max_episode_steps):
        self.id, self.max_episode_steps = id, max_episode_steps


class HazardReach:
    """A point on a plane steers to a goal; a hazard disc around the origin costs 1 per step spent inside it.
    Gymnasium's API: reset() -> (obs, info), step(a) -> (obs, reward, terminated, truncated, info with "cost")."""

    def __init__(self, max_episode_steps=200, seed=None):
        self.observation_space = Box(-np.inf, np.inf, (6,), np.float32)
        self.action_space = Box(-1.0, 1.0, (2,), np.float32)
        self.spec = _Spec("HazardReach-v0", max_episode_steps)
        self.rng = np.random.default_rng(seed)

    def _obs(self):
        return np.concatenate([self.pos, self.vel, self.goal - self.pos]).astype(np.float32)

    def reset(self, seed=None, options=None):
        if seed is not None:
            self.rng = np.random.default_rng(seed)
        self.pos = self.rng.uniform(-2.0, -1.0, 2)
        self.vel = np.zeros(2)
        self.goal = self.rng.uniform(1.0, 2.0, 2)
        self.t = 0
        return self._obs(), {}

    def step(self, action):
        self.t += 1
        a = np.clip(np.asarray(action, np.float64), -1.0, 1.0)
        d0 = np.linalg.norm(self.goal - self.pos)
        self.vel = 0.8 * self.vel + 0.1 * a
        self.pos = self.pos + self.vel
        d1 = np.linalg.norm(self.goal - self.pos)
        reward = 10.0 * (d0 - d1)
        cost = float(np.linalg.norm(self.pos) < 0.7)
        terminated = bool(d1 < 0.1)
        truncated = self.t >= self.spec.max_episode_steps
        return self._obs(), reward, terminated, truncated, {"cost": cost}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--epoch", type=int, default=2)
    ap.add_argument("--training_num", type=int, default=8)
    ap.add_argument("--step_per_epoch", type=int, default=8000)
    ap.add_argument("--cost_limit", type=float, default=5.0)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args(argv)
    agent = PPOLagAgent(env=HazardReach(), cost_limit=args.cost_limit, seed=args.seed, hidden_sizes=(64, 64))
    train_envs = DummyVectorEnv([lambda i=i: HazardReach(seed=args.seed + i) for i in range(args.training_num)])
    test_envs = DummyVectorEnv([lambda i=i: HazardReach(seed=1000 + i) for i in range(2)])
    epoch, stats, info = agent.learn(train_envs=train_envs, test_envs=test_envs, epoch=args.epoch,
                                     episode_per_collect=args.training_num, step_per_epoch=args.step_per_epoch,
                                     repeat_per_collect=4, buffer_size=args.training_num * 200, testing_num=2,
                                     batch_size=256, save_ckpt=False, verbose=False, show_progress=False)
    rew, length, cost = agent.evaluate(test_envs, eval_episodes=2)
    print(f"done: epochs {epoch}, eval reward {rew:.2f} length {length:.0f} cost {cost:.2f}")
    return epoch, rew, cost


if __name__ == "__main__":
    main()
