"""CPU twin of the HazardDash test env (tests/envs/hazard_dash.h) in numpy float32, op for op, so device
trajectories of its plugin replay bit for bit; the interface of oracle/envs.py's OracleVecEnv (reset / observe /
step over env ids), which oracle/collector.py drives.  Also the paths the plugin tests share."""
import os

import numpy as np

from oracle.philox import KEY_RESET, philox4x32, usym

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENV_DIR = os.path.join(ROOT, "tests", "envs")
# where build() puts the plugins of the headers in ENV_DIR (git-ignored build output)
PLUGIN_DIR = os.path.join(ROOT, "fsrl_b200", "_obj", "env_plugins")

f32 = np.float32
DT, DAMP, ARENA, GOAL_R, HAZ_R, LIDAR, ECOST = (f32(v) for v in (0.1, 0.9, 2.0, 0.25, 0.3, 2.0, 0.005))
NHAZ = 12


def header(name):
    return os.path.join(ENV_DIR, name + ".h")


class HazardDashTwin:
    D, A, S, T = 19, 3, 32, 200

    def __init__(self, n_env, seed):
        self.E = n_env
        self.seed = np.uint32(seed)
        self.st = np.zeros((self.S, n_env), dtype=f32)
        self.ep_idx = np.zeros(n_env, dtype=np.uint32)
        self.t = np.zeros(n_env, dtype=np.int32)

    def _ids(self, ids):
        return np.arange(self.E) if ids is None else np.asarray(ids)

    def reset(self, ids=None):
        ids = self._ids(ids)
        env, ep = ids.astype(np.uint32), self.ep_idx[ids]
        st = np.zeros((self.S, len(ids)), dtype=f32)
        r = philox4x32(env, ep, 0, 0, self.seed, KEY_RESET)
        st[0] = usym(r[0]) * f32(0.5)
        st[1] = usym(r[1]) * f32(0.5)
        st[4] = usym(r[2]) * f32(1.5)
        st[5] = usym(r[3]) * f32(1.5)
        r = philox4x32(env, ep, 1, 0, self.seed, KEY_RESET)
        st[6] = f32(1.0) + usym(r[0]) * f32(0.5)
        for c in range(NHAZ // 2):
            r = philox4x32(env, ep, 2 + c, 0, self.seed, KEY_RESET)
            for j in range(4):
                st[8 + 4 * c + j] = usym(r[j]) * ARENA
        self.st[:, ids] = st
        self.ep_idx[ids] += np.uint32(1)
        self.t[ids] = 0
        return self.observe(ids)

    def observe(self, ids=None):
        ids = self._ids(ids)
        st = self.st[:, ids]
        x, y = st[0], st[1]
        o = np.zeros((len(ids), self.D), dtype=f32)
        o[:, 0], o[:, 1] = x / ARENA, y / ARENA
        o[:, 2], o[:, 3] = st[2], st[3]
        o[:, 4], o[:, 5] = (st[4] - x) / ARENA, (st[5] - y) / ARENA
        o[:, 6] = st[6]
        for h in range(NHAZ):
            dx, dy = st[8 + 2 * h] - x, st[9 + 2 * h] - y
            o[:, 7 + h] = np.minimum(np.sqrt(dx * dx + dy * dy), LIDAR) / LIDAR
        return o

    def step(self, act, ids=None):
        """act[n][A] env-range actions; returns obs_next, rew, cost, term, trunc (trunc: horizon reached)."""
        ids = self._ids(ids)
        a = np.asarray(act, dtype=f32)
        st = self.st[:, ids].copy()
        x, y, vx, vy, gx, gy = st[0], st[1], st[2], st[3], st[4], st[5]
        d0 = np.sqrt((gx - x) * (gx - x) + (gy - y) * (gy - y))
        k = f32(1.0) + f32(0.5) * a[:, 2]
        vx = vx * DAMP + (a[:, 0] * k) * DT
        vy = vy * DAMP + (a[:, 1] * k) * DT
        x = x + vx * DT
        y = y + vy * DT
        e = st[6] - (np.abs(a[:, 0]) + np.abs(a[:, 1])) * (np.abs(k) * ECOST)
        d = np.sqrt((gx - x) * (gx - x) + (gy - y) * (gy - y))
        cost = np.zeros(len(ids), dtype=f32)
        for h in range(NHAZ):
            dx, dy = st[8 + 2 * h] - x, st[9 + 2 * h] - y
            cost[dx * dx + dy * dy < HAZ_R * HAZ_R] = f32(1.0)
        goal = d < GOAL_R
        rew = (d0 - d) * f32(10.0)
        rew = np.where(goal, rew + f32(1.0), rew).astype(f32)
        term = goal | (e <= f32(0.0)) | (np.abs(x) > ARENA) | (np.abs(y) > ARENA)
        st[0], st[1], st[2], st[3], st[6] = x, y, vx, vy, e
        st[7] = st[7] + cost
        self.st[:, ids] = st
        self.t[ids] += 1
        trunc = self.t[ids] >= self.T
        return self.observe(ids), rew, cost, term, trunc
