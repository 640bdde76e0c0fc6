"""``BasicCollector`` with the reference's constructor, ``collect`` contract and result keys
(/root/reference/fsrl/data/basic_collector.py:13-283): one env, ``n_episode`` sequential episodes,
optionally feeding a :class:`TrajectoryBuffer`.

The reference steps a gym env on the host and hands every transition to
``TrajectoryBuffer.store``.  Here every collect goes through a one-env :class:`FastCollector`: a device env
is stepped by the fused rollout kernel and finished episodes reach the trajectory buffer through the device
harvest; any other gymnasium-style env (a real simulator, a user's own env) becomes a one-env
:class:`HostVectorEnv`, stepped on the host while the device acts, stores and copies its finished episodes
out of the ring.  A single env makes the two orders the same (completion order).
"""
from __future__ import annotations

from typing import Any, Dict, Optional

from ..envs import DeviceEnv, DeviceVectorEnv
from ..host_envs import HostVectorEnv, is_vector_env
from ..obs_norm import VectorEnvNormObs
from .buffer import DeviceVectorReplayBuffer
from .fast_collector import FastCollector
from .traj_buf import TrajectoryBuffer


class BasicCollector:
    """Collect whole episodes from one env.

    :param policy: a policy of :mod:`fsrl_b200.policy`.
    :param env: what ``gym.make(task)`` returns (a :class:`DeviceEnv`, stepped with env seed 0), a
        :class:`DeviceVectorEnv` holding one env, any single gymnasium-style env (``reset`` / ``step``, ``Box``
        spaces, 4- or 5-tuple ``step``, ``cost`` in ``info``), or a :class:`HostVectorEnv` or other vector env
        holding one env.
    :param buffer: a replay buffer with one sub-buffer (``ReplayBuffer(size)``) that receives every
        transition; with None and a ``traj_buffer`` a private ring of the least size is used.
    :param bool exploration_noise: add the policy's exploration noise to its actions.
    :param TrajectoryBuffer traj_buffer: receives every finished episode.
    """

    def __init__(self, policy, env, buffer: Optional[DeviceVectorReplayBuffer] = None,
                 exploration_noise: Optional[bool] = False, traj_buffer: Optional[TrajectoryBuffer] = None):
        device = getattr(policy, "device", "cuda")
        if isinstance(env, DeviceEnv):
            env = DeviceVectorEnv(env.task, 1, device=device, seed=0)
        elif isinstance(env, (DeviceVectorEnv, HostVectorEnv, VectorEnvNormObs)):
            pass
        elif is_vector_env(env):
            if len(env) == 1:
                env = HostVectorEnv.from_vector_env(env, device=device)
        elif callable(getattr(env, "step", None)) and callable(getattr(env, "reset", None)):
            env = HostVectorEnv._from_envs([env], device=device)
        if not isinstance(env, (DeviceVectorEnv, HostVectorEnv)) or len(env) != 1:
            raise TypeError("BasicCollector steps one env: pass gym.make(task), a gymnasium-style env, or a "
                            f"DeviceVectorEnv / HostVectorEnv holding one env (got {type(env).__name__}"
                            f"{f' of {len(env)} envs' if hasattr(env, '__len__') else ''})")
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
