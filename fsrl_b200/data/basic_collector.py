"""``BasicCollector`` with the reference's constructor, ``collect`` contract and result keys
(/root/reference/fsrl/data/basic_collector.py:13-283): one env, ``n_episode`` sequential episodes,
optionally feeding a :class:`TrajectoryBuffer`.

The reference steps a gym env on the host and hands every transition to
``TrajectoryBuffer.store``.  Here the one env is a device env stepped by the fused rollout kernel
(a one-env :class:`FastCollector`), and finished episodes reach the trajectory buffer through the
device harvest; a single env makes the two orders the same (completion order).
"""
from __future__ import annotations

from typing import Any, Dict, Optional

from ..envs import DeviceEnv, DeviceVectorEnv
from .buffer import DeviceVectorReplayBuffer
from .fast_collector import FastCollector
from .traj_buf import TrajectoryBuffer


class BasicCollector:
    """Collect whole episodes from one env.

    :param policy: a policy of :mod:`fsrl_b200.policy`.
    :param env: what ``gym.make(task)`` returns (a :class:`DeviceEnv`, stepped with env seed 0) or a
        :class:`DeviceVectorEnv` holding one env.
    :param buffer: a replay buffer with one sub-buffer (``ReplayBuffer(size)``) that receives every
        transition; with None and a ``traj_buffer`` a private ring of the least size is used.
    :param bool exploration_noise: add the policy's exploration noise to its actions.
    :param TrajectoryBuffer traj_buffer: receives every finished episode.
    """

    def __init__(self, policy, env, buffer: Optional[DeviceVectorReplayBuffer] = None,
                 exploration_noise: Optional[bool] = False, traj_buffer: Optional[TrajectoryBuffer] = None):
        if isinstance(env, DeviceEnv):
            env = DeviceVectorEnv(env.task, 1, device=getattr(policy, "device", "cuda"), seed=0)
        if not isinstance(env, DeviceVectorEnv) or len(env) != 1:
            raise TypeError("BasicCollector steps one device env: pass gym.make(task) or a one-env DeviceVectorEnv")
        self.env = env
        self.policy = policy
        self.exploration_noise = exploration_noise
        self.traj_buffer = traj_buffer
        self._action_space = env.action_space
        self._fast = FastCollector(policy, env, buffer, exploration_noise=bool(exploration_noise),
                                   traj_buffer=traj_buffer)
        self.buffer = self._fast.buffer

    def reset(self, reset_buffer: bool = True, gym_reset_kwargs: Optional[Dict[str, Any]] = None) -> None:
        self._fast.reset(reset_buffer, gym_reset_kwargs)

    def reset_buffer(self, keep_statistics: bool = False) -> None:
        self._fast.reset_buffer(keep_statistics)

    def reset_stat(self) -> None:
        self._fast.reset_stat()

    def reset_env(self, gym_reset_kwargs: Optional[Dict[str, Any]] = None) -> None:
        self._fast.reset_env(gym_reset_kwargs)

    @property
    def collect_step(self) -> int:
        return self._fast.collect_step

    @property
    def collect_episode(self) -> int:
        return self._fast.collect_episode

    @property
    def collect_time(self) -> float:
        return self._fast.collect_time

    def collect(self, n_episode: int = 0, random: bool = False, render: Optional[float] = None, no_grad: bool = True,
                gym_reset_kwargs: Optional[Dict[str, Any]] = None) -> Dict[str, Any]:
        """Run ``n_episode`` episodes one after the other; returns ``n/ep``, ``n/st``, ``rew``, ``len``,
        ``total_cost``, ``cost``, ``truncated``, ``terminated``.  The reference's default ``n_episode=0`` stops
        after one step and divides by zero episodes; here ``n_episode < 1`` is rejected."""
        if n_episode is None or n_episode < 1:
            raise ValueError(f"BasicCollector.collect needs n_episode >= 1, got {n_episode}")
        return self._fast.collect(n_episode=n_episode, random=random, no_grad=no_grad,
                                  gym_reset_kwargs=gym_reset_kwargs)
