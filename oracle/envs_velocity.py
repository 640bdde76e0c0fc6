"""Oracle (test infrastructure): CPU twin of the Safety-Gymnasium velocity kinds 33-37 in
fsrl_b200/csrc/envs.cuh (namespace vel: HalfCheetah, Hopper, Swimmer, Walker2d and Ant), vectorised over envs
in numpy float32.

Like oracle/envs_nav.py these are our documented models, not gymnasium's MuJoCo dynamics (SURVEY.md F5).
Every op is IEEE-exact (+ - * / sqrt, polynomial sin/cos), written in the same order as the CUDA code, so
device trajectories match this twin bit for bit given identical actions.  ``OracleVecEnvVel`` extends
``OracleVecEnvBP``: every other kind runs the unchanged twins, so one class takes every device kind.
"""
from __future__ import annotations

import numpy as np

from . import envs_button_push as _bp
from .envs import _rotate
from .envs_button_push import OracleVecEnvBP
from .envs_flight import _sincos
from .philox import KEY_RESET, philox4x32, usym

f32 = np.float32
HALF_CHEETAH, HOPPER, SWIMMER, WALKER2D, ANT = range(33, 38)
KINDS = dict(_bp.KINDS, half_cheetah=HALF_CHEETAH, hopper=HOPPER, swimmer=SWIMMER, walker2d=WALKER2D, ant=ANT)
DIMS = dict(_bp.DIMS)
DIMS.update({HALF_CHEETAH: (17, 6, 17, 1000), HOPPER: (11, 3, 11, 1000), SWIMMER: (8, 2, 9, 1000),
             WALKER2D: (17, 6, 17, 1000), ANT: (27, 8, 26, 1000)})
PLANAR = (HALF_CHEETAH, HOPPER, WALKER2D)

# constants mirrored from csrc/envs.cuh (namespace vel)
V = {k: f32(v) for k, v in dict(DT=0.05, KA=20.0, KQ=10.0, KD=4.0, RDT=0.1, ZK=40.0, ZD=10.0, ZQ=0.05, FALL=1.5,
                                 SW_KW=0.5, SW_YD=2.0, ANT_KW=0.02, ANT_YD=2.0, ANT_AT=0.5, ANT_AS=20.0,
                                 ANT_AD=6.0, ANT_ZA=0.1).items()}
# per robot: the speed of a saturated gait, the gait gain, the cost threshold, the control weight, the healthy
# reward, the standing height, and the pitch stiffness (> 0: unstable), thigh coupling and damping
R = {HALF_CHEETAH: dict(VMAX=4.0, GK=0.05, VCOST=2.8, WCTRL=0.1, HEALTHY=0.0, Z0=0.6, PU=-20.0, PT=0.5, PD=2.0),
     HOPPER: dict(VMAX=0.5, GK=0.2, VCOST=0.35, WCTRL=1e-3, HEALTHY=1.0, Z0=1.25, PU=2.0, PT=2.0, PD=1.0),
     SWIMMER: dict(VMAX=0.07, GK=0.2, VCOST=0.05, WCTRL=1e-4, HEALTHY=0.0, Z0=0.0, PU=0.0, PT=0.0, PD=0.0),
     WALKER2D: dict(VMAX=2.5, GK=0.1, VCOST=1.7, WCTRL=1e-3, HEALTHY=1.0, Z0=1.25, PU=2.0, PT=2.0, PD=1.0),
     ANT: dict(VMAX=3.5, GK=0.05, VCOST=2.5, WCTRL=0.5, HEALTHY=1.0, Z0=0.6, PU=0.0, PT=0.0, PD=0.0)}
R = {k: {n: f32(v) for n, v in p.items()} for k, p in R.items()}
NJ = {HALF_CHEETAH: 6, HOPPER: 3, SWIMMER: 2, WALKER2D: 6, ANT: 8}
# the joint pairs whose swept area drives the robot: (i, k) adds q_i * qd_k - q_k * qd_i
PAIRS = {HALF_CHEETAH: [(0, 1), (1, 2), (3, 4), (4, 5)], HOPPER: [(0, 1), (1, 2)], SWIMMER: [(0, 1)],
         WALKER2D: [(0, 1), (1, 2), (3, 4), (4, 5)], ANT: [(0, 4), (1, 5), (2, 6), (3, 7)]}


def _clamp1(v):
    return np.minimum(f32(1), np.maximum(f32(-1), v)).astype(f32)


def _joints(st, q0, n, act):
    """The n damped, driven joints q = st[q0:q0 + n], qd = st[q0 + n:q0 + 2n], integrated in place; returns
    sum a_j^2."""
    ctrl = np.zeros(act.shape[0], f32)
    for j in range(n):
        a, q, qd = act[:, j], st[q0 + j], st[q0 + n + j]
        qd = qd + (((V["KA"] * a) - (V["KQ"] * q)) - (V["KD"] * qd)) * V["DT"]
        st[q0 + j], st[q0 + n + j] = q + qd * V["DT"], qd
        ctrl = ctrl + a * a
    return ctrl


def _area(q, qd, i, k):
    return q[i] * qd[k] - q[k] * qd[i]


def _gait(kind, q, qd):
    """The saturated gait force in [-1, 1]: the pairs' summed swept area times the gait gain."""
    g = np.zeros(q[0].shape, f32)
    for i, k in PAIRS[kind]:
        g = g + _area(q, qd, i, k)
    return _clamp1(g * R[kind]["GK"])


class OracleVecEnvVel(OracleVecEnvBP):
    """OracleVecEnvBP over every device kind, the velocity kinds 33-37 included."""

    def __init__(self, kind, n_env, seed):
        k = KINDS[kind] if isinstance(kind, str) else int(kind)
        if k not in NJ:
            super().__init__(k, n_env, seed)
            return
        self.kind = k
        self.D, self.A, self.S, self.T = DIMS[k]
        self.N = NJ[k]
        self.q0 = {SWIMMER: 5, ANT: 10}.get(k, 5)
        self.E = n_env
        self.seed = np.uint32(seed)
        self.st = np.zeros((self.S, n_env), dtype=f32)
        self.ep_idx = np.zeros(n_env, dtype=np.uint32)
        self.t = np.zeros(n_env, dtype=np.int32)

    # ---- gym protocol -------------------------------------------------------------------------------------
    def reset(self, ids=None):
        if self.kind not in NJ:
            return super().reset(ids)
        ids = np.arange(self.E) if ids is None else np.asarray(ids)
        env = ids.astype(np.uint32)
        ep = self.ep_idx[ids]
        k = self.kind
        r = philox4x32(env, ep, 0, 0, self.seed, KEY_RESET)
        st = np.zeros((self.S, len(ids)), dtype=f32)
        if k in PLANAR:
            st[0] = R[k]["Z0"] + usym(r[0]) * f32(0.005)
            st[2] = usym(r[1]) * f32(0.02)
            st[3] = usym(r[2]) * f32(0.02)
        elif k == SWIMMER:
            st[0] = usym(r[0]) * f32(0.05)
            st[2], st[1] = _sincos(st[0])
        else:
            st[0] = R[k]["Z0"] + usym(r[0]) * f32(0.005)
            st[2], st[3] = _unit(usym(r[1]) * f32(0.05))
            st[6] = usym(r[2]) * f32(0.02)
            st[8] = usym(r[3]) * f32(0.02)
        for h in range((self.N + 3) // 4):
            q = philox4x32(env, ep, 1 + h, 0, self.seed, KEY_RESET)
            for j in range(min(4, self.N - 4 * h)):
                st[self.q0 + 4 * h + j] = usym(q[j]) * f32(0.05)
        self.st[:, ids] = st
        self.ep_idx[ids] += np.uint32(1)
        self.t[ids] = 0
        return self.observe(ids)

    def observe(self, ids=None):
        if self.kind not in NJ:
            return super().observe(ids)
        st = self.st if ids is None else self.st[:, np.asarray(ids)]
        o = np.zeros((st.shape[1], self.D), dtype=f32)
        N, q0, k = self.N, self.q0, self.kind
        if k in PLANAR:
            o[:, 0] = st[0]; o[:, 1] = st[2]
            for j in range(N):
                o[:, 2 + j] = st[5 + j]
            o[:, 2 + N] = st[4]; o[:, 3 + N] = st[1]; o[:, 4 + N] = st[3]
            for j in range(N):
                o[:, 5 + N + j] = st[5 + N + j]
        elif k == SWIMMER:
            o[:, 0] = st[0]; o[:, 1] = st[5]; o[:, 2] = st[6]
            o[:, 3] = st[3] * st[1]; o[:, 4] = st[3] * st[2]; o[:, 5] = st[4]
            o[:, 6] = st[7]; o[:, 7] = st[8]
        else:
            c, s = st[2], st[3]
            ch = np.sqrt(np.maximum(f32(0), (f32(1) + c) * f32(0.5)))
            sh = np.sqrt(np.maximum(f32(0), (f32(1) - c) * f32(0.5)))
            sh = np.where(s < 0, -sh, sh).astype(f32)
            sr, cr = _sincos(st[6] * f32(0.5))
            sp, cp = _sincos(st[8] * f32(0.5))
            o[:, 0] = st[0]
            o[:, 1] = (ch * cp) * cr + (sh * sp) * sr
            o[:, 2] = (ch * cp) * sr - (sh * sp) * cr
            o[:, 3] = (ch * sp) * cr + (sh * cp) * sr
            o[:, 4] = (sh * cp) * cr - (ch * sp) * sr
            for j in range(8):
                o[:, 5 + j] = st[q0 + j]
                o[:, 19 + j] = st[q0 + 8 + j]
            o[:, 13] = st[4] * c; o[:, 14] = st[4] * s; o[:, 15] = st[1]
            o[:, 16] = st[7]; o[:, 17] = st[9]; o[:, 18] = st[5]
        return o

    def step(self, act, ids=None):
        if self.kind not in NJ:
            return super().step(act, ids)
        ids = np.arange(self.E) if ids is None else np.asarray(ids)
        act = np.asarray(act, dtype=f32)
        st = [self.st[i, ids].copy() for i in range(self.S)]
        k, N, q0 = self.kind, self.N, self.q0
        p = R[k]
        ctrl = _joints(st, q0, N, act)
        q, qd = st[q0:q0 + N], st[q0 + N:q0 + 2 * N]
        F = _gait(k, q, qd)
        if k in PLANAR:
            st[4] = st[4] + (p["VMAX"] * F - st[4]) * V["RDT"]
            if k == HOPPER:
                tq, kn = q[0], q[1] * q[1]
            elif k == WALKER2D:
                tq, kn = (q[0] + q[3]) * f32(0.5), q[1] * q[1] + q[4] * q[4]
            else:
                tq, kn = q[0] - q[3], q[1] * q[1] + q[4] * q[4]
            st[3] = st[3] + (((p["PU"] * st[2]) - (p["PT"] * tq)) - (p["PD"] * st[3])) * V["DT"]
            st[2] = st[2] + st[3] * V["DT"]
            fall = np.abs(st[2]) > V["FALL"]
            st[2] = np.where(fall, np.where(st[2] > 0, V["FALL"], -V["FALL"]), st[2]).astype(f32)
            st[3] = np.where(fall, f32(0), st[3]).astype(f32)
            _, cth = _sincos(st[2])
            zt = (p["Z0"] - V["ZQ"] * kn) * cth
            st[1] = st[1] + (V["ZK"] * (zt - st[0]) - V["ZD"] * st[1]) * V["DT"]
            st[0] = st[0] + st[1] * V["DT"]
            vx = st[4]
            z, th = st[0], st[2]
            if k == HOPPER:
                term = (z <= f32(0.7)) | (np.abs(th) >= f32(0.2))
            elif k == WALKER2D:
                term = (z <= f32(0.8)) | (z >= f32(2.0)) | (np.abs(th) >= f32(1.0))
            else:
                term = np.zeros(len(ids), bool)
            speed = vx
        elif k == SWIMMER:
            st[3] = st[3] + (p["VMAX"] * F - st[3]) * V["RDT"]
            st[4] = st[4] + (V["SW_KW"] * (q[0] + q[1]) - V["SW_YD"] * st[4]) * V["DT"]
            d = st[4] * V["DT"]
            st[0] = st[0] + d
            st[1], st[2] = _rotate(st[1], st[2], d)
            vx = st[3] * st[1]
            speed = vx
            term = np.zeros(len(ids), bool)
        else:
            st[4] = st[4] + (p["VMAX"] * F - st[4]) * V["RDT"]
            lft = _area(q, qd, 0, 4) + _area(q, qd, 1, 5)
            rgt = _area(q, qd, 2, 6) + _area(q, qd, 3, 7)
            st[5] = st[5] + (V["ANT_KW"] * (lft - rgt) - V["ANT_YD"] * st[5]) * V["DT"]
            st[2], st[3] = _rotate(st[2], st[3], st[5] * V["DT"])
            st[7] = st[7] + (((V["ANT_AT"] * ((q[0] + q[1]) - (q[2] + q[3]))) - (V["ANT_AS"] * st[6]))
                             - (V["ANT_AD"] * st[7])) * V["DT"]
            st[6] = st[6] + st[7] * V["DT"]
            st[9] = st[9] + (((V["ANT_AT"] * ((q[0] + q[3]) - (q[1] + q[2]))) - (V["ANT_AS"] * st[8]))
                             - (V["ANT_AD"] * st[9])) * V["DT"]
            st[8] = st[8] + st[9] * V["DT"]
            zt = p["Z0"] + V["ANT_ZA"] * ((q[4] + q[5]) + (q[6] + q[7]))
            st[1] = st[1] + (V["ZK"] * (zt - st[0]) - V["ZD"] * st[1]) * V["DT"]
            st[0] = st[0] + st[1] * V["DT"]
            vx = st[4] * st[2]
            vy = st[4] * st[3]
            speed = np.sqrt(vx * vx + vy * vy)
            term = (st[0] < f32(0.2)) | (st[0] > f32(1.0))
        rew = (vx + p["HEALTHY"]) - p["WCTRL"] * ctrl
        cost = (speed > p["VCOST"]).astype(f32)
        for i in range(self.S):
            self.st[i, ids] = st[i]
        self.t[ids] += 1
        trunc = self.t[ids] >= self.T
        return self.observe(ids), rew.astype(f32), cost, term, trunc


def _unit(d):
    """The unit heading (cos d, sin d) of a small angle: the polynomial sin / cos, renormalised."""
    sn, cs = _sincos(d)
    n = np.sqrt(cs * cs + sn * sn)
    return cs / n, sn / n
