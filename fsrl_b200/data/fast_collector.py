"""``FastCollector`` with the reference's constructor, ``collect`` contract and result keys
(/root/reference/fsrl/data/fast_collector.py:47-69,192-408), running every vector step as
one fused CUDA launch (csrc/rollout.cu) against a :class:`DeviceVectorEnv`.

Episode-count semantics are the reference's: the ready set is the first
``min(env_num, n_episode)`` envs (:235-236), finished envs are reset and keep going until the
remaining episode budget is smaller than the ready set, at which point the lowest-index
finished envs are retired first (:357-363); every collect ends with a reset of all envs
(:375-388).  When ``n_episode <= env_num`` each ready env runs exactly one episode and the
bookkeeping is done inline by the step kernel; otherwise a one-CTA resolve kernel applies
the ordered surplus rule after each step.

A policy the rollout kernel cannot run (its own ``forward``, or an actor the parameter arena
rejects) takes the generic path (``collector.fused == False``): per vector step the collector calls
``policy(batch)`` and ``exploration_noise`` in torch, then a step kernel with those actions runs the
same map_action, env step, buffer store and episode bookkeeping as the fused kernel.

A :class:`HostVectorEnv` (or any other object with tianshou's vector-env protocol, wrapped once by
``HostVectorEnv.from_vector_env``) takes the host path: the reference's loop runs on the host around the
envs' own ``step`` / ``reset``, and per vector step one launch (csrc/rollout_host.cu) stores the previous
step's transitions into the same ring and computes this step's actions with the fused path's actor,
sampling and noise stream.  Finished envs are reset, surplus ones retired without a reset, as on the
device path; the statistics are summed on the host in float64, in step order.  A ``traj_buffer`` is fed there
without a ring scan: the loop offers each finished episode with the float64 return and cost the env reported, and
copies the kept ones from the ring (``fsrl_traj_copy_host``) right after the launch that stores their last transition,
so an episode must fit the ring (``cap >= max_episode_steps``, or ``cap >=`` its length when the horizon is unknown).

An env wrapped by :class:`~fsrl_b200.obs_norm.VectorEnvNormObs` collects normalized observations: per vector step
the statistics take the ``obs_next`` of every env that stepped, then the reset observations of the envs that
restarted, and the ring and the actor see the normalized rows.  Device envs then take one
``fsrl_rollout_norm_steps`` per step (six launches) instead of the one-launch collect; host envs normalize inside
their per-step ``fsrl_host_collect_step_norm``.
"""
from __future__ import annotations

import contextlib
import ctypes
import time
import types
from typing import Any, Callable, Dict, Optional

import numpy as np
import torch

from .. import _lib
from ..envs import DeviceVectorEnv
from ..host_envs import HostVectorEnv, is_vector_env
from ..obs_norm import VectorEnvNormObs
from .batch import Batch
from .buffer import DeviceVectorReplayBuffer
from .traj_buf import TrajectoryBuffer, TrajectoryHarvest


def _fused_policy(policy) -> bool:
    """Whether the policy's actor runs inside the fused rollout kernel.  That takes a ``fill_rollout``
    the policy itself defines, or the built-in one of a ``BasePolicy`` that keeps the built-in
    ``forward`` and whose networks the parameter arena can hold.  Any other policy is called per step."""
    from ..policy.base_policy import BasePolicy
    if not hasattr(policy, "fill_rollout"):
        return False
    if not isinstance(policy, BasePolicy):
        return True

    def ours(name):
        owner = next(c for c in type(policy).__mro__ if name in vars(c))
        return owner.__module__.startswith("fsrl_b200.")

    if not ours("fill_rollout"):
        return True
    return ours("forward") and policy._arena_holds_nets()


class FastCollector(object):
    def __init__(self, policy, env: DeviceVectorEnv, buffer: Optional[DeviceVectorReplayBuffer] = None,
                 preprocess_fn: Optional[Callable[..., Batch]] = None,
                 exploration_noise: bool = False, traj_buffer: Optional[TrajectoryBuffer] = None) -> None:
        super().__init__()
        # the observation-normalizing wrapper: self.env is the env it wraps, self.norm the wrapper
        self.norm = env if isinstance(env, VectorEnvNormObs) else None
        if self.norm is not None:
            if traj_buffer is not None:
                raise NotImplementedError("traj_buffer with a VectorEnvNormObs env would store a dataset of normalized "
                                          "observations; harvest from the unwrapped env")
            if getattr(policy, "_dp", None) is not None:
                raise NotImplementedError("VectorEnvNormObs under data parallelism: each rank's statistics would "
                                          "diverge")
            env = self.norm.venv
        if not isinstance(env, (DeviceVectorEnv, HostVectorEnv)):
            if not is_vector_env(env):
                raise TypeError("fsrl_b200.FastCollector steps a DeviceVectorEnv, a HostVectorEnv or an object with "
                                f"the vector-env protocol (len, step(action, id), reset(id)); got {type(env).__name__}")
            env = HostVectorEnv.from_vector_env(env, device=getattr(policy, "device", "cuda"))
        if preprocess_fn is not None:
            raise NotImplementedError("preprocess_fn would need a host round trip per step")
        # host path: the host steps the envs, one launch per vector step acts and stores
        self.host = isinstance(env, HostVectorEnv)
        if self.host and not _fused_policy(policy):
            what = "host envs collecting into a traj_buffer" if traj_buffer is not None else "host envs"
            raise NotImplementedError(f"{what} need a policy whose actor the rollout kernel runs (a built-in "
                                      "actor the parameter arena holds); this policy would take the generic path")
        self.env = env
        self.env_num = len(env)
        self.exploration_noise = exploration_noise
        self._store = buffer is not None
        self.traj_buffer = traj_buffer
        if traj_buffer is not None:
            if not self.host:       # host envs: the collect loop itself knows every finished episode, no scan
                self._harvest = TrajectoryHarvest(self.env_num, env.device)
            if buffer is None:      # the harvest reads finished episodes from a ring: a private one of the least size
                if self.host and env.max_episode_steps is None:
                    raise ValueError("traj_buffer over host envs without a horizon (spec.max_episode_steps is None) "
                                     "needs a buffer: a private ring cannot be sized; pass a VectorReplayBuffer "
                                     "whose sub-buffers hold the longest episode")
                buffer = DeviceVectorReplayBuffer(self.env_num * self.min_ring_capacity(), self.env_num)
        self._assign_buffer(buffer)
        self.policy = policy
        # fused: the actor runs inside the rollout kernel; generic: the policy is called once per vector step
        self.fused = _fused_policy(policy)
        self.preprocess_fn = None
        self._action_space = env.action_space
        self.reset(False)

    def _assign_buffer(self, buffer) -> None:
        if buffer is None:
            # the reference creates VectorReplayBuffer(env_num, env_num) for a buffer-less
            # collector (:72-73) whose content nobody reads (evaluate()); we skip the stores
            self.buffer = None
            return
        assert buffer.buffer_num >= self.env_num                        # :75
        buffer.allocate(self.env.D, self.env.A, self.env.device)
        self.buffer = buffer

    def reset(self, reset_buffer: bool = True, gym_reset_kwargs: Optional[Dict[str, Any]] = None) -> None:
        self.reset_env(gym_reset_kwargs)
        if reset_buffer:
            self.reset_buffer()
        self.reset_stat()

    def reset_stat(self) -> None:
        self.collect_step, self.collect_episode, self.collect_time = 0, 0, 0.0

    def reset_buffer(self, keep_statistics: bool = False) -> None:
        if self.buffer is not None:
            self.buffer.reset(keep_statistics=keep_statistics)

    def reset_env(self, gym_reset_kwargs: Optional[Dict[str, Any]] = None) -> None:
        if self.norm is not None:
            # one update of all E rows
            if self.host:
                self._obs = self.norm.host_reset_all(**(gym_reset_kwargs or {}))
            else:
                self.norm.reset()
            return
        if self.host:
            self._obs = self.env.reset_obs(None, **(gym_reset_kwargs or {}))
            return
        self.env.reset()

    def min_ring_capacity(self, n_episode: Optional[int] = None) -> int:
        """Ring slots per env a ``traj_buffer`` harvest needs: an episode must still be in the ring when the scan
        after its last step runs.  That is once after the collect when every ready env runs one episode
        (``n_episode <= env_num``), else after every chunk of ``min(T, 64)`` steps.  Host envs copy an episode
        right after the launch that stores its last transition: ``T`` slots (None when the horizon is unknown)."""
        T = self.env.max_episode_steps
        if self.host:
            return T
        if n_episode is not None and n_episode <= self.env_num:
            return T
        return T + self._chunk()

    def _chunk(self) -> int:
        return max(1, min(self.env.max_episode_steps, 64))

    # ------------------------------------------------------------------------------------------------
    def _descriptor(self, random: bool) -> "_lib.Rollout":
        r = _lib.Rollout()
        self.env.fill(r)
        if self.buffer is not None:
            self.buffer.fill(r)
        if self.fused:
            self.policy.fill_rollout(r, exploration_noise=self.exploration_noise)
        else:
            # the policy's own map_action settings, the reference's defaults without them
            r.actor.H = 64
            r.action_bound = {"": 0, "clip": 1, "tanh": 2}[getattr(self.policy, "action_bound_method", "clip")]
            r.action_scaling = int(getattr(self.policy, "action_scaling", True))
        if random:
            r.mode = _lib.MODE_RANDOM
        return r

    def _generic_steps(self, r, n_steps: int, stream: int, no_grad: bool) -> None:
        """n vector steps of the generic path: policy(batch) -> exploration_noise on all E rows (retired
        envs included), then one caller-action step kernel + the resolve kernel.  No host sync.  The policy
        sees a copy of the observations (a device tensor), so keeping or editing batch.obs cannot reach
        the env state; exploration_noise receives the policy's action as the device tensor it returned."""
        env, policy = self.env, self.policy
        want = (env.env_num, env.A)
        for _ in range(n_steps):
            with torch.no_grad() if no_grad else contextlib.nullcontext():
                batch = Batch(obs=env.obs_cur.clone(), info=Batch())
                act = policy(batch, None).act
                if self.exploration_noise:
                    act = policy.exploration_noise(act, batch)
            act = torch.as_tensor(act, dtype=torch.float32, device=env.device).contiguous()
            if tuple(act.shape) != want:
                raise ValueError(f"the policy returned actions of shape {tuple(act.shape)}; the collect needs {want}")
            if self.norm is not None:
                desc = self.norm.descriptor()
                _lib.check(_lib.lib.fsrl_rollout_norm_steps(ctypes.byref(r), ctypes.byref(desc), 1, act.data_ptr(),
                                                            stream))
            else:
                _lib.check(_lib.lib.fsrl_rollout_steps_act(ctypes.byref(r), act.data_ptr(), stream))

    def collect(self, n_episode: int = 1, random: bool = False, render: bool = False,
                no_grad: bool = True, gym_reset_kwargs: Optional[Dict[str, Any]] = None) -> Dict[str, Any]:
        if n_episode is not None:
            assert n_episode > 0                                        # :234
        else:
            raise TypeError("Please specify n_episode"
                            "in FastCollector.collect().")
        start_time = time.time()
        r = self._descriptor(random)
        if self.host:
            st = self._host_steps(r, int(n_episode), render, gym_reset_kwargs)
        else:
            st = self._device_steps(r, n_episode, no_grad, random)
        step_count, episode_count = int(st.step_count), int(st.episode_count)
        self.collect_step += step_count
        self.collect_episode += episode_count
        # a collect always ends with fresh resets of every env (:375-388)
        self.reset_env()
        self.collect_time += max(time.time() - start_time, 1e-9)

        if episode_count > 0:
            rew_mean = st.sum_ep_rew / episode_count
            len_mean = st.sum_ep_len / episode_count
        else:
            rew_mean = len_mean = 0
        done_count = st.term_count + st.trunc_count
        return {
            "n/ep": episode_count,
            "n/st": step_count,
            "rew": rew_mean,
            "len": len_mean,
            "total_cost": st.total_cost,
            "cost": st.total_cost / episode_count,
            "truncated": st.trunc_count / done_count,
            "terminated": st.term_count / done_count,
        }

    def _host_steps(self, r, n_episode: int, render: bool, gym_reset_kwargs) -> types.SimpleNamespace:
        """The reference's collect loop (:252-368) over host envs; the device acts and stores once per step.

        With a ``traj_buffer`` the loop also keeps every env's episode: its first ring slot (``b_ptr`` read once,
        then advanced here by one per stored transition) and its float64 cost.  An env that finishes is offered
        to the buffer in ascending env id within the step, the device path's (finish step, env) order, and the
        kept episodes are copied out of the ring right after the next launch, which stores their last transition."""
        env = self.env
        E = self.env_num
        kw = gym_reset_kwargs or {}
        obs = self._obs
        ready = np.arange(min(E, n_episode))
        ep_rew, ep_len = np.zeros(E, np.float64), np.zeros(E, np.int64)
        st = types.SimpleNamespace(step_count=0, episode_count=0, total_cost=0.0, sum_ep_rew=0.0, sum_ep_len=0,
                                   term_count=0, trunc_count=0)
        stored = None                         # the previous step's transitions, stored by the next launch
        norm = self.norm
        fresh = None                          # wrapped: the envs restarted since the last launch, and their obs
        traj = self.traj_buffer
        if traj is not None:
            T, cap = env.max_episode_steps, self.buffer.cap
            if T is not None and cap < T:
                raise ValueError(f"a traj_buffer harvest of host envs needs a ring of at least {T} slots per env "
                                 f"(max_episode_steps); the buffer has {cap}")
            head = self.buffer.ptr[:E].cpu().numpy().astype(np.int64)   # the ring slot each env's next store takes
            ep_start, ep_cost = head.copy(), np.zeros(E, np.float64)
            jobs = []                         # kept episodes whose last transition the next launch stores
            with torch.cuda.device(env.device):
                stream = torch.cuda.current_stream().cuda_stream
        while True:
            act = env.device_step(r, ready, obs[ready], stored, norm, fresh)
            fresh = None
            if traj is not None and jobs:
                traj._copy_host(r, jobs, T or 0, env.D, env.A, env.device, stream)
                jobs = []
            obs_next, rew, term, trunc, cost = env.step_envs(act, ready)
            if traj is not None:
                over = ready[ep_len[ready] >= cap]
                if len(over):
                    e = int(over[0])
                    raise ValueError(f"env {e}'s episode reached {ep_len[e] + 1} steps, longer than the ring's "
                                     f"{cap} slots per env: storing it would overwrite its first transition before "
                                     "the traj_buffer copies it; pass a buffer whose sub-buffers hold the longest "
                                     "episode")
                ep_start[ready] = np.where(ep_len[ready] == 0, head[ready], ep_start[ready])
                head[ready] = (head[ready] + 1) % cap
                ep_cost[ready] += cost
            if render:
                env.render()
            if self.buffer is not None or norm is not None:
                stored = (ready, obs_next, rew, cost, term, trunc)
            st.total_cost += float(np.sum(cost, dtype=np.float64))
            st.step_count += len(ready)
            ep_rew[ready] += rew.astype(np.float64)
            ep_len[ready] += 1
            obs[ready] = obs_next
            done = term | trunc
            if done.any():
                ids = ready[done]
                st.episode_count += len(ids)
                st.sum_ep_rew += float(np.sum(ep_rew[ids]))
                st.sum_ep_len += int(np.sum(ep_len[ids]))
                st.term_count += int(term.sum())
                st.trunc_count += int(trunc.sum())
                if traj is not None:
                    jobs = traj._offer_episodes((int(e), int(ep_start[e]), int(ep_len[e]), float(ep_rew[e]),
                                                 float(ep_cost[e])) for e in ids)
                    ep_cost[ids] = 0.0
                ep_rew[ids], ep_len[ids] = 0.0, 0
                # the surplus rule (:357-363): the lowest finished ids retire, without a reset; the rest restart
                surplus = min(max(len(ready) - (n_episode - st.episode_count), 0), len(ids))
                if surplus < len(ids):
                    restart = ids[surplus:]
                    obs[restart] = env.reset_obs(restart, **kw)
                    if norm is not None:
                        fresh = (restart, obs[restart])
                if surplus:
                    ready = ready[~np.isin(ready, ids[:surplus])]
            if st.episode_count >= n_episode:
                break
        if stored is not None:
            env.device_step(r, ready[:0], obs[:0], stored, norm, fresh)
            if traj is not None and jobs:
                traj._copy_host(r, jobs, T or 0, env.D, env.A, env.device, stream)
        return st

    def _device_steps(self, r, n_episode: int, no_grad: bool, random: bool):
        env = self.env
        r.inline_done = 1 if n_episode <= self.env_num else 0
        T = env.max_episode_steps
        traj = self.traj_buffer
        if traj is not None and self.buffer.cap < self.min_ring_capacity(n_episode):
            raise ValueError(f"a traj_buffer harvest of collect(n_episode={n_episode}) needs a ring of at least "
                             f"{self.min_ring_capacity(n_episode)} slots per env; the buffer has {self.buffer.cap}")
        with torch.cuda.device(env.device):
            stream = torch.cuda.current_stream().cuda_stream
            if (self.fused or random) and self.norm is not None:
                desc = self.norm.descriptor()

                def steps(n):
                    _lib.check(_lib.lib.fsrl_rollout_norm_steps(ctypes.byref(r), ctypes.byref(desc), n, None, stream))
            elif self.fused or random:
                def steps(n):
                    _lib.check(_lib.lib.fsrl_rollout_steps(ctypes.byref(r), n, stream))
            else:
                def steps(n):
                    self._generic_steps(r, n, stream, no_grad)
            _lib.check(_lib.lib.fsrl_collect_begin(ctypes.byref(r), int(n_episode), stream))
            if traj is not None:
                self._harvest.begin(r, stream)
            if r.inline_done:
                # every ready env runs exactly one episode of at most T steps
                steps(T)
                st = env.read_stats()
                if traj is not None:
                    self._harvest_into(traj, r, min(n_episode, self.env_num), T, stream)
            else:
                chunk = self._chunk()
                while True:
                    steps(chunk)
                    st = env.read_stats()
                    if traj is not None:
                        self._harvest_into(traj, r, 0, chunk, stream)
                    if st.finished:
                        break
        if not st.finished:
            raise RuntimeError("rollout did not reach n_episode within the step bound "
                               f"(episodes {st.episode_count}/{n_episode})")
        return st

    def _harvest_into(self, traj: TrajectoryBuffer, r, n_ready: int, window: int, stream: int) -> None:
        rows = self._harvest.scan(r, n_ready, window, stream)
        env = self.env
        traj._commit(r, rows, env.max_episode_steps, env.D, env.A, env.device, stream)
