"""Oracle (test infrastructure): CPU twin of the device environments of kinds 6-8 in
fsrl_b200/csrc/envs.cuh (Ant-Run, Drone-Circle, Drone-Run), vectorised over envs in numpy float32.

Like oracle/envs.py these are our documented models, not Bullet-Safety-Gym's pybullet dynamics
(SURVEY.md F5).  Every op is IEEE-exact (+ - * / sqrt, polynomial sin/cos), written in the same order
as the CUDA code, so device trajectories match this twin bit for bit given identical actions.
``OracleVecEnvExt`` extends ``OracleVecEnv``: kinds 0-5 run the unchanged twin of oracle/envs.py,
so every caller of the oracle (oracle/collector.py included) takes all nine kinds.
"""
from __future__ import annotations

import numpy as np

from . import envs as _base
from .envs import OracleVecEnv, _car_advance, _heading_from_box, _rotate
from .philox import KEY_RESET, philox4x32, usym

f32 = np.float32
ANT_RUN, DRONE_CIRCLE, DRONE_RUN = 6, 7, 8
KINDS = dict(_base.KINDS, ant_run=ANT_RUN, drone_circle=DRONE_CIRCLE, drone_run=DRONE_RUN)
DIMS = dict(_base.DIMS)
DIMS.update({ANT_RUN: (34, 8, 31, 300), DRONE_CIRCLE: (18, 4, 17, 300), DRONE_RUN: (19, 4, 18, 200)})

# constants mirrored from csrc/envs.cuh (namespaces antr, drone)
ANTR = dict(DT=0.05, VMAX=2.0, WMAX=2.0, AV=0.1, AW=0.15, YLIM=1.0, VLIM=0.8, RSCALE=1.0)
DR = dict(DT=0.05, G=9.8, TM=4.9, KM=0.3, KT=20.0, KP=25.0, KD=6.0, KY=4.0, KDY=2.0, DRAG=0.5,
          Z0=1.0, FLIP=0.8, R=1.5, XLIM=1.125, YLIM=0.6, VLIM=1.0, RSCALE=1.0)
DR = {k: f32(v) for k, v in DR.items()}
ANTR = {k: f32(v) for k, v in ANTR.items()}


def _sincos(d):
    """Polynomial sin / cos of a small angle (the series of rotate_heading)."""
    d2 = d * d
    sn = d * (f32(1) - (d2 / f32(6)) * (f32(1) - d2 / f32(20)))
    cs = f32(1) - (d2 / f32(2)) * (f32(1) - (d2 / f32(12)) * (f32(1) - d2 / f32(30)))
    return sn, cs


def _ant_joints(st, act):
    """Ant-Circle's 8 damped joint oscillators; returns (thrust, turn, ctrl)."""
    n = act.shape[0]
    thrust = np.zeros(n, f32); turn = np.zeros(n, f32); ctrl = np.zeros(n, f32)
    for j in range(8):
        q, qd, a = st[6 + j], st[14 + j], act[:, j]
        qd = qd + (((f32(20.0) * a) - (f32(10.0) * q)) - (f32(4.0) * qd)) * f32(0.05)
        q = q + qd * f32(0.05)
        st[6 + j], st[14 + j], st[22 + j] = q, qd, a
        if j < 4:
            thrust = thrust + q
        else:
            turn = turn + q
        ctrl = ctrl + a * a
    return thrust, turn, ctrl


def _drone_advance(st, act):
    """Quadrotor step; returns the terminated flags."""
    P = DR
    m = []
    for j in range(4):
        mj = st[13 + j] + (((act[:, j] + f32(1)) * f32(0.5)) - st[13 + j]) * P["KM"]
        st[13 + j] = mj
        m.append(mj)
    thr = P["TM"] * ((m[0] + m[1]) + (m[2] + m[3]))
    tr = (m[0] + m[3]) - (m[1] + m[2])
    tp = (m[0] + m[1]) - (m[2] + m[3])
    ty = (m[0] + m[2]) - (m[1] + m[3])
    x, y, z, c, s, vx, vy, vz, phi, th, p, q, r = (st[i] for i in range(13))
    p = p + (((P["KT"] * tr) - (P["KP"] * phi)) - (P["KD"] * p)) * P["DT"]
    phi = phi + p * P["DT"]
    q = q + (((P["KT"] * tp) - (P["KP"] * th)) - (P["KD"] * q)) * P["DT"]
    th = th + q * P["DT"]
    r = r + ((P["KY"] * ty) - (P["KDY"] * r)) * P["DT"]
    c, s = _rotate(c, s, r * P["DT"])
    sp, cp = _sincos(phi)
    sth, cth = _sincos(th)
    axb = thr * sth
    ayb = thr * sp
    ax = c * axb - s * ayb
    ay = s * axb + c * ayb
    az = (thr * cp) * cth - P["G"]
    vx = vx + (ax - P["DRAG"] * vx) * P["DT"]
    vy = vy + (ay - P["DRAG"] * vy) * P["DT"]
    vz = vz + (az - P["DRAG"] * vz) * P["DT"]
    x = x + vx * P["DT"]
    y = y + vy * P["DT"]
    z = z + vz * P["DT"]
    for i, val in enumerate((x, y, z, c, s, vx, vy, vz, phi, th, p, q, r)):
        st[i] = val
    return (z <= f32(0)) | (np.abs(phi) > P["FLIP"]) | (np.abs(th) > P["FLIP"])


def _drone_body_obs(st, o, col0):
    """The 15 body channels shared by both Drone tasks, written to o[:, col0:col0 + 15]."""
    o[:, col0] = st[2] - DR["Z0"]
    o[:, col0 + 1] = st[5]; o[:, col0 + 2] = st[6]; o[:, col0 + 3] = st[7]
    o[:, col0 + 4] = st[3]; o[:, col0 + 5] = st[4]
    o[:, col0 + 6] = st[8]; o[:, col0 + 7] = st[9]
    o[:, col0 + 8] = st[10]; o[:, col0 + 9] = st[11]; o[:, col0 + 10] = st[12]
    for j in range(4):
        o[:, col0 + 11 + j] = (st[13 + j] - f32(0.5)) * f32(2.0)


class OracleVecEnvExt(OracleVecEnv):
    """OracleVecEnv over all nine device kinds."""

    def __init__(self, kind, n_env, seed):
        k = KINDS[kind] if isinstance(kind, str) else int(kind)
        if k < ANT_RUN:
            super().__init__(k, n_env, seed)
            return
        self.kind = k
        self.D, self.A, self.S, self.T = DIMS[k]
        self.E = n_env
        self.seed = np.uint32(seed)
        self.st = np.zeros((self.S, n_env), dtype=f32)
        self.ep_idx = np.zeros(n_env, dtype=np.uint32)
        self.t = np.zeros(n_env, dtype=np.int32)

    def reset(self, ids=None):
        if self.kind < ANT_RUN:
            return super().reset(ids)
        ids = np.arange(self.E) if ids is None else np.asarray(ids)
        env = ids.astype(np.uint32)
        ep = self.ep_idx[ids]
        n = len(ids)
        r = philox4x32(env, ep, 0, 0, self.seed, KEY_RESET)
        st = np.zeros((self.S, n), dtype=f32)
        if self.kind == ANT_RUN:
            st[1] = usym(r[0]) * f32(0.2)
            st[2], st[3] = _heading_from_box(np.ones(n, f32), usym(r[1]) * f32(0.3))
            q = philox4x32(env, ep, 1, 0, self.seed, KEY_RESET)
            q2 = philox4x32(env, ep, 2, 0, self.seed, KEY_RESET)
            for j in range(4):
                st[6 + j] = usym(q[j]) * f32(0.1)
                st[10 + j] = usym(q2[j]) * f32(0.1)
        else:
            if self.kind == DRONE_CIRCLE:
                st[0] = usym(r[0]) * f32(0.3)
            st[1] = usym(r[1]) * f32(0.3)
            st[2] = DR["Z0"]
            st[3], st[4] = _heading_from_box(usym(r[2]), usym(r[3]))
            q = philox4x32(env, ep, 1, 0, self.seed, KEY_RESET)
            st[8] = usym(q[0]) * f32(0.1)
            st[9] = usym(q[1]) * f32(0.1)
            for j in range(4):
                st[13 + j] = f32(0.5)
        self.st[:, ids] = st
        self.ep_idx[ids] += np.uint32(1)
        self.t[ids] = 0
        return self.observe(ids)

    def observe(self, ids=None):
        if self.kind < ANT_RUN:
            return super().observe(ids)
        st = self.st if ids is None else self.st[:, ids]
        n = st.shape[1]
        o = np.zeros((n, self.D), dtype=f32)
        if self.kind == ANT_RUN:
            P = ANTR
            y, c, s, v, w = st[1], st[2], st[3], st[4], st[5]
            o[:, 0] = y; o[:, 1] = v * c; o[:, 2] = v * s; o[:, 3] = c; o[:, 4] = s
            o[:, 5] = w / P["WMAX"]; o[:, 6] = v / P["VLIM"]; o[:, 7] = st[0] / f32(10.0)
            aq = np.zeros(n, f32)
            for j in range(8):
                o[:, 8 + j] = st[6 + j]
                o[:, 16 + j] = st[14 + j] * f32(0.1)
                o[:, 24 + j] = st[22 + j]
                aq = aq + np.abs(st[6 + j])
            o[:, 32] = np.abs(y) - P["YLIM"]
            o[:, 33] = f32(0.5) + aq * f32(0.0125)
        elif self.kind == DRONE_CIRCLE:
            x, y = st[0], st[1]
            rr = np.sqrt(x * x + y * y)
            o[:, 0] = x / DR["R"]; o[:, 1] = y / DR["R"]
            _drone_body_obs(st, o, 2)
            o[:, 17] = (rr - DR["R"]) / DR["R"]
        else:
            vx, vy = st[5], st[6]
            sp = np.sqrt(vx * vx + vy * vy)
            o[:, 0] = st[1]
            _drone_body_obs(st, o, 1)
            o[:, 16] = sp - DR["VLIM"]
            o[:, 17] = np.abs(st[1]) - DR["YLIM"]
            o[:, 18] = st[0] / f32(10.0)
        return o

    def step(self, act, ids=None):
        if self.kind < ANT_RUN:
            return super().step(act, ids)
        ids = np.arange(self.E) if ids is None else np.asarray(ids)
        act = np.asarray(act, dtype=f32)
        st = [self.st[i, ids].copy() for i in range(self.S)]
        if self.kind == ANT_RUN:
            P = ANTR
            x_old = st[0].copy()
            thrust, turn, ctrl = _ant_joints(st, act)
            f = np.minimum(f32(1), np.maximum(f32(-1), thrust * f32(0.25)))
            g = np.minimum(f32(1), np.maximum(f32(-1), turn * f32(0.25)))
            _car_advance(st, f, g, P["VMAX"], P["WMAX"], P["AV"], P["AW"], P["DT"])
            rew = ((st[0] - x_old) / P["DT"]) * P["RSCALE"] - f32(0.005) * ctrl
            cost = ((np.abs(st[1]) > P["YLIM"]) | (st[4] > P["VLIM"])).astype(f32)
            st[30] = st[30] + cost
            term = np.zeros(len(ids), dtype=bool)
        else:
            P = DR
            x_old = st[0].copy()
            term = _drone_advance(st, act)
            x, y, vx, vy = st[0], st[1], st[5], st[6]
            if self.kind == DRONE_CIRCLE:
                rr = np.sqrt(x * x + y * y)
                rew = (x * vy - y * vx) / (P["R"] * (f32(1) + np.abs(rr - P["R"])))
                cost = (np.abs(x) > P["XLIM"]).astype(f32)
            else:
                sp = np.sqrt(vx * vx + vy * vy)
                rew = ((x - x_old) / P["DT"]) * P["RSCALE"]
                cost = ((np.abs(y) > P["YLIM"]) | (sp > P["VLIM"])).astype(f32)
                st[17] = st[17] + cost
        for i in range(self.S):
            self.st[i, ids] = st[i]
        self.t[ids] += 1
        trunc = self.t[ids] >= self.T
        return self.observe(ids), rew.astype(f32), cost.astype(f32), term, trunc
