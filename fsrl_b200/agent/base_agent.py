"""Agent shells with the reference's ``learn`` / ``evaluate`` / ``state_dict`` surface
(/root/reference/fsrl/agent/base_agent.py:53-93,108-209,225-324): they wire a device replay
buffer, two FastCollectors and a trainer around a policy.  Host control code."""
from __future__ import annotations

import contextlib
import warnings
from abc import ABC, abstractmethod
from typing import Optional, Tuple

import torch

from ..data import FastCollector, VectorReplayBuffer
from ..envs import DeviceEnv, DeviceVectorEnv, HostVectorEnv
from ..host_envs import is_vector_env
from ..obs_norm import VectorEnvNormObs
from ..trainer import OffpolicyTrainer, OnpolicyTrainer
from ..utils.exp_util import seed_all
from ..utils.logger import BaseLogger, DummyLogger


def _as_vector(envs, device, seed=0):
    """A device env as a one-env DeviceVectorEnv; any other vector-protocol object (a tianshou vector env of
    host envs) as a HostVectorEnv, so that the replay buffer and the collectors see one env object.  A
    VectorEnvNormObs passes through."""
    if isinstance(envs, VectorEnvNormObs):
        return envs
    if isinstance(envs, DeviceEnv):
        return DeviceVectorEnv(envs.task, 1, device=device, seed=seed)
    if not isinstance(envs, (DeviceVectorEnv, HostVectorEnv)) and is_vector_env(envs):
        return HostVectorEnv.from_vector_env(envs, device=device, seed=seed)
    return envs


class BaseAgent(ABC):
    name = "BaseAgent"

    @abstractmethod
    def __init__(self, *args, **kwargs) -> None:
        self.policy = None
        self.task = None
        self.logger = DummyLogger()
        self.cost_limit = 0

    @abstractmethod
    def learn(self, *args, **kwargs) -> None:
        raise NotImplementedError

    def evaluate(self, test_envs, state_dict: Optional[dict] = None, eval_episodes: int = 10,
                 render: bool = False, train_mode: bool = False) -> Tuple[float, float, float]:
        if state_dict is not None:
            self.policy.load_state_dict(state_dict)
        self.policy.train() if train_mode else self.policy.eval()
        test_envs = _as_vector(test_envs, self.policy.device)
        # a normalizing wrapper only normalizes here: evaluation leaves its statistics as they are
        frozen = test_envs.frozen() if isinstance(test_envs, VectorEnvNormObs) else contextlib.nullcontext()
        with frozen:
            eval_collector = FastCollector(self.policy, test_envs)
            result = eval_collector.collect(n_episode=eval_episodes, render=render)
        return result["rew"], result["len"], result["cost"]

    @property
    def state_dict(self):
        return self.policy.state_dict()

    # shared by the presets' constructors
    def _prologue(self, logger, cost_limit, seed: int, thread: int, device: str) -> str:
        """Keep the logger and the cost limit, seed every RNG and set torch's host threads; returns the device
        the networks are built on.  Runs before any network is built, as default initialisation draws from the
        seeded generators."""
        self.logger, self.cost_limit = logger, cost_limit
        seed_all(seed)
        torch.set_num_threads(thread)
        if device == "cpu":
            # the reference's default device; this engine has a GPU path only -- say so instead of remapping silently.
            # stacklevel 3: the preset's caller, not the preset's constructor
            warnings.warn("fsrl_b200 runs on CUDA devices only: device='cpu' is mapped to 'cuda'", RuntimeWarning,
                          stacklevel=3)
            device = "cuda"
        return device

    def _adopt_policy(self, policy, seed: int) -> None:
        """Make ``policy`` the agent's: its networks move into the device arena and its action noise is keyed
        by the seed."""
        self.policy = policy
        policy.arena
        policy.set_action_seed(seed)

    # shared by both learn() flavours
    def _setup(self, train_envs, test_envs, buffer_size, reward_threshold, save_ckpt):
        assert self.policy is not None, "The policy is not initialized"
        self.policy.train()
        dev = self.policy.device
        train_envs = _as_vector(train_envs, dev)
        if test_envs is not None:
            test_envs = _as_vector(test_envs, dev)
            if isinstance(train_envs, VectorEnvNormObs) and not isinstance(test_envs, VectorEnvNormObs):
                # tianshou's MuJoCo recipe: the test envs normalize with the training statistics, frozen
                test_envs = VectorEnvNormObs(test_envs, update_obs_rms=False)
                test_envs.set_obs_rms(train_envs.get_obs_rms())
        buffer = VectorReplayBuffer(buffer_size, len(train_envs), device=dev)
        train_collector = FastCollector(self.policy, train_envs, buffer, exploration_noise=True)
        test_collector = FastCollector(self.policy, test_envs) if test_envs is not None else None

        def stop_fn(reward, cost):
            return reward > reward_threshold and cost < self.cost_limit

        if save_ckpt:
            if isinstance(train_envs, VectorEnvNormObs):
                rms = train_envs.get_obs_rms()
                self.logger.setup_checkpoint_fn(lambda: {"model": self.state_dict, "obs_rms": rms.state_dict()})
            else:
                self.logger.setup_checkpoint_fn(lambda: {"model": self.state_dict})
        return train_collector, test_collector, stop_fn

    def _run(self, trainer, verbose):
        epoch, stat, info = 0, {}, {}
        for epoch, stat, info in trainer:
            self.logger.store(tab="train", cost_limit=self.cost_limit)
            if verbose:
                print(f"Epoch: {epoch}", info)
        return epoch, stat, info


class OffpolicyAgent(BaseAgent):
    name = "OffpolicyAgent"

    def __init__(self) -> None:
        super().__init__()

    def learn(self, train_envs, test_envs=None, epoch: int = 300, episode_per_collect: int = 5,
              step_per_epoch: int = 3000, update_per_step: float = 0.1, buffer_size: int = 100000,
              testing_num: int = 2, batch_size: int = 256, reward_threshold: float = 450,
              save_interval: int = 4, resume: bool = False, save_ckpt: bool = True,
              verbose: bool = True, show_progress: bool = True):
        tc, sc, stop_fn = self._setup(train_envs, test_envs, buffer_size, reward_threshold, save_ckpt)
        trainer = OffpolicyTrainer(policy=self.policy, train_collector=tc, test_collector=sc,
                                   max_epoch=epoch, batch_size=batch_size, cost_limit=self.cost_limit,
                                   step_per_epoch=step_per_epoch, update_per_step=update_per_step,
                                   episode_per_test=testing_num, episode_per_collect=episode_per_collect,
                                   stop_fn=stop_fn, logger=self.logger, resume_from_log=resume,
                                   save_model_interval=save_interval, verbose=verbose,
                                   show_progress=show_progress)
        return self._run(trainer, verbose)


class OnpolicyAgent(BaseAgent):
    name = "OnpolicyAgent"

    def __init__(self) -> None:
        super().__init__()

    def learn(self, train_envs, test_envs=None, epoch: int = 300, episode_per_collect: int = 20,
              step_per_epoch: int = 10000, repeat_per_collect: int = 4, buffer_size: int = 100000,
              testing_num: int = 2, batch_size: int = 512, reward_threshold: float = 450,
              save_interval: int = 4, resume: bool = False, save_ckpt: bool = True,
              verbose: bool = True, show_progress: bool = True):
        tc, sc, stop_fn = self._setup(train_envs, test_envs, buffer_size, reward_threshold, save_ckpt)
        trainer = OnpolicyTrainer(policy=self.policy, train_collector=tc, test_collector=sc,
                                  max_epoch=epoch, batch_size=batch_size, cost_limit=self.cost_limit,
                                  step_per_epoch=step_per_epoch, repeat_per_collect=repeat_per_collect,
                                  episode_per_test=testing_num, episode_per_collect=episode_per_collect,
                                  stop_fn=stop_fn, logger=self.logger, resume_from_log=resume,
                                  save_model_interval=save_interval, verbose=verbose,
                                  show_progress=show_progress)
        return self._run(trainer, verbose)
