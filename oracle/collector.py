"""Oracle (test infrastructure): CPU restatement of FastCollector.collect
(/root/reference/fsrl/data/fast_collector.py:192-408) over the CPU env twin, storing into a
VectorReplayBuffer-shaped dict of numpy arrays (env-major sub-buffers, SURVEY.md App. A.25).
Action noise comes from the documented Philox stream (oracle/philox.py) instead of torch's
CPU generator so that device rollouts can be replayed."""
from __future__ import annotations

import numpy as np
import torch

from .envs import OracleVecEnv
from .philox import action_noise, action_uniform

LOG_SQRT_2PI = np.float32(0.9189385332046727)


class OracleBuffer:
    def __init__(self, total_size, n_env, D, A):
        self.cap = int(np.ceil(total_size / n_env))
        self.E = n_env
        n = self.cap * n_env
        self.obs = np.zeros((n, D), np.float32); self.obs_next = np.zeros((n, D), np.float32)
        self.act = np.zeros((n, A), np.float32)
        self.rew = np.zeros(n, np.float32); self.cost = np.zeros(n, np.float32)
        self.logp = np.zeros(n, np.float32)
        self.terminated = np.zeros(n, bool); self.truncated = np.zeros(n, bool)
        self.ptr = np.zeros(n_env, np.int64); self.len = np.zeros(n_env, np.int64)

    def reset(self):
        self.ptr[:] = 0; self.len[:] = 0

    def add(self, ids, obs, act, rew, cost, logp, term, trunc, obs_next):
        p = ids * self.cap + self.ptr[ids]
        self.obs[p], self.act[p], self.rew[p], self.cost[p], self.logp[p] = obs, act, rew, cost, logp
        self.terminated[p], self.truncated[p], self.obs_next[p] = term, trunc, obs_next
        self.ptr[ids] = (self.ptr[ids] + 1) % self.cap
        self.len[ids] = np.minimum(self.len[ids] + 1, self.cap)

    def sample_all(self):
        idx = []
        for e in range(self.E):
            L, cap = self.len[e], self.cap
            start = self.ptr[e] if L == cap else 0
            idx.append(e * cap + (start + np.arange(L)) % cap)
        return np.concatenate(idx) if idx else np.zeros(0, np.int64)

    def unfinished_index(self):
        out = []
        for e in range(self.E):
            if self.len[e] > 0:
                last = e * self.cap + (self.ptr[e] - 1) % self.cap
                if not (self.terminated[last] or self.truncated[last]):
                    out.append(last)
        return np.asarray(out, np.int64)


def collect(env: OracleVecEnv, actor, n_episode, seed_act, act_ctr, buffer=None, mode="train",
            head="gauss_indep", action_bound="clip", action_scaling=True, low=None, high=None,
            expl_sigma=0.0):
    """Returns the reference's stats dict.  ``actor``: torch module mapping obs -> (mu, sigma)
    or mu.  ``act_ctr``: per-env uint32 noise counters (updated in place).  The envs must
    have been reset (env.reset()) beforehand; ends with a reset of all envs (:375-388)."""
    E = env.E
    ready = np.arange(min(E, n_episode))                                     # :235
    obs = env.observe(ready)
    step_count = 0; total_cost = 0.0; term_c = 0; trunc_c = 0; ep_count = 0
    ep_rews, ep_lens = [], []
    run_rew = np.zeros(E, np.float64); run_len = np.zeros(E, np.int64)
    low = np.full(env.A, -1, np.float32) if low is None else np.asarray(low, np.float32)
    high = np.full(env.A, 1, np.float32) if high is None else np.asarray(high, np.float32)
    while True:
        n = len(ready)
        with torch.no_grad():
            if mode == "random":
                # action_space.sample() + map_action_inverse (fast_collector.py:258-264)
                act = action_uniform(seed_act, ready, act_ctr[ready], env.A)
                if action_bound == "tanh":
                    with np.errstate(divide="ignore"):
                        act = (np.float32(0.5) * (np.log1p(act) - np.log1p(-act))).astype(np.float32)
                logp = np.zeros(n, np.float32)
                act_ctr[ready] += np.uint32(1)
            else:
                out = actor(torch.from_numpy(obs))
                if head == "deterministic":
                    mu = out.numpy().astype(np.float32); sigma = None
                else:
                    mu, sigma = (t.numpy().astype(np.float32) for t in out)
                if mode == "train":
                    eps = action_noise(seed_act, ready, act_ctr[ready], env.A)
                    act_ctr[ready] += np.uint32(1)
                else:
                    eps = np.zeros_like(mu)
                if head == "deterministic":
                    act = mu.copy(); logp = np.zeros(n, np.float32)
                    if mode == "train" and expl_sigma > 0:
                        act = (np.float32(expl_sigma) * eps + act).astype(np.float32)
                elif head == "gauss_indep":
                    act = (sigma * eps + mu).astype(np.float32) if mode == "train" else mu.copy()
                    z = (act - mu) / sigma
                    logp = (-0.5 * z * z - np.log(sigma) - LOG_SQRT_2PI).sum(1).astype(np.float32)
                else:  # gauss_cond (SAC, sac_lag.py:147-183)
                    pre = (sigma * eps + mu).astype(np.float32) if mode == "train" else mu.copy()
                    z = eps if mode == "train" else np.zeros_like(mu)
                    sq = np.tanh(pre)
                    logp = ((-0.5 * z * z - np.log(sigma) - LOG_SQRT_2PI)
                            - np.log(1.0 - sq * sq + np.finfo(np.float32).eps)).sum(1).astype(np.float32)
                    act = sq.astype(np.float32)
        # map_action (base_policy.py:244-256)
        a = act
        if action_bound == "clip":
            a = np.clip(a, np.float32(-1), np.float32(1))
        elif action_bound == "tanh":
            a = np.tanh(a)
        if action_scaling:
            a = (low + ((high - low) * (a + np.float32(1))) / np.float32(2)).astype(np.float32)
        obs_next, rew, cost, term, trunc = env.step(a, ready)                    # :286
        trunc = trunc & ~term
        done = term | trunc
        total_cost += float(cost.sum())                                          # :326
        if buffer is not None:
            buffer.add(ready, obs, act, rew, cost, logp, term, trunc, obs_next)   # :333
        step_count += n
        run_rew[ready] += rew.astype(np.float64); run_len[ready] += 1
        if done.any():
            loc = np.where(done)[0]
            glob = ready[loc]
            ep_count += len(loc)
            ep_rews.append(run_rew[glob].copy()); ep_lens.append(run_len[glob].copy())
            run_rew[glob] = 0; run_len[glob] = 0
            term_c += int(term.sum()); trunc_c += int(trunc.sum())
            surplus = max(0, len(ready) - (n_episode - ep_count))                 # :358
            retire = loc[:surplus]                                                # :361
            keep = loc[surplus:]
            # the reference resets every finished env (:351) and then drops the surplus ones;
            # a dropped env is reset again by the end-of-collect reset_env (:388), so skipping
            # its first reset is unobservable except for the env's reset-RNG counter, which
            # is our own design: retired envs are NOT reset here (matches csrc/rollout.cu)
            obs_next = obs_next.copy()
            if len(keep):
                obs_next[keep] = env.reset(ready[keep])
            if surplus > 0:
                mask = np.ones(len(ready), bool)
                mask[retire] = False
                ready = ready[mask]; obs_next = obs_next[mask]
        obs = obs_next                                                             # :365
        if ep_count >= n_episode:
            break
    env.reset()                                                                    # :388
    rews = np.concatenate(ep_rews); lens = np.concatenate(ep_lens)
    done_c = term_c + trunc_c
    return {"n/ep": ep_count, "n/st": step_count, "rew": rews.mean(), "len": lens.mean(),
            "total_cost": total_cost, "cost": total_cost / ep_count,
            "truncated": trunc_c / done_c, "terminated": term_c / done_c}
