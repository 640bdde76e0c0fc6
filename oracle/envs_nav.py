"""Oracle (test infrastructure): CPU twin of the Safety-Gymnasium navigation kinds 16-22 in
fsrl_b200/csrc/envs.cuh (the Point and Car robots on Circle 1 / 2 and Goal 1 / 2), vectorised over envs
in numpy float32.

Like oracle/envs.py these are our documented models, not Safety-Gymnasium's MuJoCo dynamics (SURVEY.md
F5).  Every op is IEEE-exact (+ - * / sqrt, polynomial sin/cos), written in the same order as the CUDA
code, so device trajectories match this twin bit for bit given identical actions.  ``OracleVecEnvNav``
extends ``OracleVecEnvExt``: kinds 0-8 run the unchanged twins of oracle/envs.py and
oracle/envs_flight.py, so every caller of the oracle (oracle/collector.py included) takes every kind.
"""
from __future__ import annotations

import numpy as np

from . import envs_flight as _flight
from .envs import LIDAR_EDGE_C, LIDAR_EDGE_S, _car_advance, _heading_from_box
from .envs_flight import OracleVecEnvExt
from .philox import KEY_GOAL, KEY_RESET, philox4x32, usym

f32 = np.float32
POINT_CIRCLE1, POINT_CIRCLE2, CAR_CIRCLE1, CAR_CIRCLE2, POINT_GOAL2, CAR_GOAL1, CAR_GOAL2 = range(16, 23)
# kind -> (Car body, Circle task, level)
NAV = {POINT_CIRCLE1: (False, True, 1), POINT_CIRCLE2: (False, True, 2), CAR_CIRCLE1: (True, True, 1),
       CAR_CIRCLE2: (True, True, 2), POINT_GOAL2: (False, False, 2), CAR_GOAL1: (True, False, 1),
       CAR_GOAL2: (True, False, 2)}
KINDS = dict(_flight.KINDS, point_circle1=POINT_CIRCLE1, point_circle2=POINT_CIRCLE2, car_circle1=CAR_CIRCLE1,
             car_circle2=CAR_CIRCLE2, point_goal2=POINT_GOAL2, car_goal1=CAR_GOAL1, car_goal2=CAR_GOAL2)
DIMS = dict(_flight.DIMS)
DIMS.update({k: (28, 2, 7, 500) for k in (POINT_CIRCLE1, POINT_CIRCLE2, CAR_CIRCLE1, CAR_CIRCLE2)})
DIMS.update({POINT_GOAL2: (60, 2, 10, 1000), CAR_GOAL1: (60, 2, 28, 1000), CAR_GOAL2: (60, 2, 10, 1000)})

# constants mirrored from csrc/envs.cuh (namespaces pgoal, nav)
P = {k: f32(v) for k, v in dict(DT=0.05, VMAX=1.0, WMAX=3.0, AV=0.2, AW=0.3, ARENA=2.0, GOAL_R=0.3, HAZ_R=0.2,
                                 CAR_VW=1.0, CAR_AL=0.2, TRACK=0.5, CIRC_R=1.5, WALL=1.125, START=0.8,
                                 VASE_R=0.25).items()}


def _advance(car, st, act):
    """Both bodies hold x, y, c, s, v, w.  The Car's wheel speeds lag their commands (a0, a1), which is the same
    lag on v towards (a0 + a1) / 2 * CAR_VW and on w towards (a1 - a0) / TRACK * CAR_VW."""
    if not car:
        _car_advance(st, act[:, 0], act[:, 1], 1.0, 3.0, 0.2, 0.3, 0.05)
        return
    a0, a1 = act[:, 0], act[:, 1]
    _car_advance(st, (a0 + a1) * f32(0.5), (a1 - a0) * f32(0.5), P["CAR_VW"], (f32(2) * P["CAR_VW"]) / P["TRACK"],
                 P["CAR_AL"], P["CAR_AL"], P["DT"])


def _sensors(o, v, w, v_prev, c, s):
    o[:, 0] = (v - v_prev) / P["DT"]; o[:, 1] = v * w; o[:, 2] = f32(9.81)
    o[:, 3] = v; o[:, 8] = w; o[:, 9] = c; o[:, 10] = f32(0.0) - s


def _lidar(o, col0, ox, oy, x, y, c, s):
    dx = ox - x; dy = oy - y
    rx = c * dx + s * dy
    ry = c * dy - s * dx
    d = np.sqrt(rx * rx + ry * ry)
    val = np.maximum(f32(0), f32(1) - d / f32(3.0))
    n = o.shape[0]
    b = np.zeros(n, dtype=np.int64)
    for kk in range(16):
        k1 = (kk + 1) & 15
        c0 = LIDAR_EDGE_C[kk] * ry - LIDAR_EDGE_S[kk] * rx
        c1 = LIDAR_EDGE_C[k1] * ry - LIDAR_EDGE_S[k1] * rx
        b = np.where((c0 >= 0) & (c1 < 0), kk, b)
    idx = np.arange(n)
    o[idx, col0 + b] = np.maximum(o[idx, col0 + b], val)


class OracleVecEnvNav(OracleVecEnvExt):
    """OracleVecEnvExt over every device kind, the navigation kinds 16-22 included."""

    def __init__(self, kind, n_env, seed):
        k = KINDS[kind] if isinstance(kind, str) else int(kind)
        if k not in NAV:
            super().__init__(k, n_env, seed)
            return
        self.kind = k
        self.car, self.circle, self.level = NAV[k]
        self.D, self.A, self.S, self.T = DIMS[k]
        self.E = n_env
        self.seed = np.uint32(seed)
        self.st = np.zeros((self.S, n_env), dtype=f32)
        self.ep_idx = np.zeros(n_env, dtype=np.uint32)
        self.t = np.zeros(n_env, dtype=np.int32)

    def layout(self, ids=None, st=None):
        """[(vase, x, y)] of the current episode's hazards, then vases, for the envs ``ids`` (Goal tasks).
        Level 1 reads the state; level 2 regenerates the draws 1-10 of the reset's Philox stream."""
        ids = np.arange(self.E) if ids is None else np.asarray(ids)
        st = self.st[:, ids] if st is None else st
        if self.level == 1:
            return [(False, st[9 + 2 * h], st[10 + 2 * h]) for h in range(8)] + [(True, st[25], st[26])]
        env = ids.astype(np.uint32)
        ep = (self.ep_idx[ids] - np.uint32(1)).astype(np.uint32)
        out = []
        for h in range(10):
            q = philox4x32(env, ep, 1 + h, 0, self.seed, KEY_RESET)
            out.append((h >= 5, usym(q[0]) * P["ARENA"], usym(q[1]) * P["ARENA"]))
            out.append((h >= 5, usym(q[2]) * P["ARENA"], usym(q[3]) * P["ARENA"]))
        return out

    def reset(self, ids=None):
        if self.kind not in NAV:
            return super().reset(ids)
        ids = np.arange(self.E) if ids is None else np.asarray(ids)
        env = ids.astype(np.uint32)
        ep = self.ep_idx[ids]
        r = philox4x32(env, ep, 0, 0, self.seed, KEY_RESET)
        st = np.zeros((self.S, len(ids)), dtype=f32)
        if self.circle:
            st[0] = usym(r[0]) * P["START"]; st[1] = usym(r[1]) * P["START"]
            st[2], st[3] = _heading_from_box(usym(r[2]), usym(r[3]))
        else:
            st[0] = usym(r[0]) * f32(0.5); st[1] = usym(r[1]) * f32(0.5)
            st[2], st[3] = _heading_from_box(usym(r[2]), usym(r[3]))
            g = philox4x32(env, ep, 0, 0, self.seed, KEY_GOAL)
            st[6] = usym(g[0]) * P["ARENA"]; st[7] = usym(g[1]) * P["ARENA"]
            if self.level == 1:
                for h in range(5):
                    q = philox4x32(env, ep, 1 + h, 0, self.seed, KEY_RESET)
                    if h < 4:
                        for j in range(4):
                            st[9 + 4 * h + j] = usym(q[j]) * P["ARENA"]
                    else:
                        st[25] = usym(q[0]) * P["ARENA"]; st[26] = usym(q[1]) * P["ARENA"]
        self.st[:, ids] = st
        self.ep_idx[ids] += np.uint32(1)
        self.t[ids] = 0
        return self.observe(ids)

    def observe(self, ids=None):
        if self.kind not in NAV:
            return super().observe(ids)
        ids = np.arange(self.E) if ids is None else np.asarray(ids)
        st = self.st[:, ids]
        o = np.zeros((len(ids), self.D), dtype=f32)
        x, y, c, s = st[0], st[1], st[2], st[3]
        _sensors(o, st[4], st[5], st[self.S - 1], c, s)
        if self.circle:
            _lidar(o, 12, f32(0), f32(0), x, y, c, s)
        else:
            _lidar(o, 12, st[6], st[7], x, y, c, s)
            for vase, ox, oy in self.layout(ids, st):
                _lidar(o, 44 if vase else 28, ox, oy, x, y, c, s)
        return o

    def step(self, act, ids=None):
        if self.kind not in NAV:
            return super().step(act, ids)
        ids = np.arange(self.E) if ids is None else np.asarray(ids)
        act = np.asarray(act, dtype=f32)
        st = [self.st[i, ids].copy() for i in range(self.S)]
        n = len(ids)
        car = self.car
        if self.circle:
            st[6] = st[4].copy()
            _advance(car, st, act)
            v = st[4]
            x, y = st[0], st[1]
            vx, vy = v * st[2], v * st[3]
            r = np.sqrt(x * x + y * y)
            rew = ((x * vy - y * vx) / (np.maximum(r, f32(1e-6)) * (f32(1) + np.abs(r - P["CIRC_R"])))) * f32(0.1)
            out = np.abs(x) > P["WALL"]
            if self.level == 2:
                out = out | (np.abs(y) > P["WALL"])
            cost = out.astype(f32)
        else:
            vp = self.S - 1
            dxo = st[6] - st[0]; dyo = st[7] - st[1]
            dist_old = np.sqrt(dxo * dxo + dyo * dyo)
            st[vp] = st[4].copy()
            _advance(car, st, act)
            st[0] = np.minimum(P["ARENA"], np.maximum(-P["ARENA"], st[0]))
            st[1] = np.minimum(P["ARENA"], np.maximum(-P["ARENA"], st[1]))
            dxn = st[6] - st[0]; dyn = st[7] - st[1]
            dist = np.sqrt(dxn * dxn + dyn * dyn)
            rew = dist_old - dist
            hit = dist <= P["GOAL_R"]
            rew = np.where(hit, rew + f32(1), rew).astype(f32)
            st[8] = np.where(hit, st[8] + f32(1), st[8]).astype(f32)
            if hit.any():
                env = ids.astype(np.uint32)
                ep = (self.ep_idx[ids] - np.uint32(1)).astype(np.uint32)
                g = philox4x32(env, ep, (np.uint32(16) + st[8].astype(np.uint32)), 0, self.seed, KEY_GOAL)
                st[6] = np.where(hit, usym(g[0]) * P["ARENA"], st[6]).astype(f32)
                st[7] = np.where(hit, usym(g[1]) * P["ARENA"], st[7]).astype(f32)
            cost = np.zeros(n, f32)
            for vase, ox, oy in self.layout(ids, np.stack(st)):
                if vase and self.level == 1:
                    continue
                dx = ox - st[0]; dy = oy - st[1]
                lim = P["VASE_R"] * P["VASE_R"] if vase else P["HAZ_R"] * P["HAZ_R"]
                cost = np.where(dx * dx + dy * dy <= lim, f32(1), cost).astype(f32)
        for i in range(self.S):
            self.st[i, ids] = st[i]
        self.t[ids] += 1
        trunc = self.t[ids] >= self.T
        return self.observe(ids), rew.astype(f32), cost, np.zeros(n, dtype=bool), trunc
