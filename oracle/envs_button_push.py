"""Oracle (test infrastructure): CPU twin of the Safety-Gymnasium Button and Push kinds 24-31 in
fsrl_b200/csrc/envs.cuh (NavButton / NavPush on the Point and Car bodies), vectorised over envs in numpy
float32.

Like oracle/envs_nav.py these are our documented models, not Safety-Gymnasium's MuJoCo dynamics (SURVEY.md
F5).  Every op is IEEE-exact and written in the same order as the CUDA code, so device trajectories match
this twin bit for bit given identical actions.  ``OracleVecEnvBP`` extends ``OracleVecEnvNav``: every other
kind runs the unchanged twins, so one class takes every device kind.
"""
from __future__ import annotations

import numpy as np

from . import envs_nav as _nav
from .envs import _heading_from_box, _rotate
from .envs_nav import P, OracleVecEnvNav, _advance, _lidar, _sensors
from .philox import KEY_GOAL, KEY_RESET, philox4x32, usym

f32 = np.float32
(POINT_BUTTON1, POINT_BUTTON2, CAR_BUTTON1, CAR_BUTTON2,
 POINT_PUSH1, POINT_PUSH2, CAR_PUSH1, CAR_PUSH2) = range(24, 32)
# kind -> (Car body, Button task, level)
BP = {POINT_BUTTON1: (False, True, 1), POINT_BUTTON2: (False, True, 2), CAR_BUTTON1: (True, True, 1),
      CAR_BUTTON2: (True, True, 2), POINT_PUSH1: (False, False, 1), POINT_PUSH2: (False, False, 2),
      CAR_PUSH1: (True, False, 1), CAR_PUSH2: (True, False, 2)}
KINDS = dict(_nav.KINDS, point_button1=POINT_BUTTON1, point_button2=POINT_BUTTON2, car_button1=CAR_BUTTON1,
             car_button2=CAR_BUTTON2, point_push1=POINT_PUSH1, point_push2=POINT_PUSH2, car_push1=CAR_PUSH1,
             car_push2=CAR_PUSH2)
DIMS = dict(_nav.DIMS)
DIMS.update({k: (76, 2, 12, 1000) for k in (POINT_BUTTON1, POINT_BUTTON2, CAR_BUTTON1, CAR_BUTTON2)})
DIMS.update({POINT_PUSH1: (76, 2, 18, 1000), CAR_PUSH1: (76, 2, 18, 1000),
             POINT_PUSH2: (76, 2, 28, 1000), CAR_PUSH2: (76, 2, 28, 1000)})

# constants mirrored from csrc/envs.cuh (namespaces button, push)
B = {k: f32(v) for k, v in dict(BUTTON_R=0.2, GREM_R=0.2, GREM_W=1.0, GREM_TRAVEL=0.35, PUSH_D=0.3,
                                 PUSH_HAZ_R=0.3, PILLAR_R=0.4, BOX_START=1.0).items()}
DELAY = 10


def _clamp(v):
    return np.minimum(P["ARENA"], np.maximum(-P["ARENA"], v))


def _dist2(ox, oy, x, y):
    dx = ox - x
    dy = oy - y
    return dx * dx + dy * dy


class OracleVecEnvBP(OracleVecEnvNav):
    """OracleVecEnvNav over every device kind, the Button and Push kinds 24-31 included."""

    def __init__(self, kind, n_env, seed):
        k = KINDS[kind] if isinstance(kind, str) else int(kind)
        if k not in BP:
            super().__init__(k, n_env, seed)
            return
        self.kind = k
        self.car, self.button, self.level = BP[k]
        self.D, self.A, self.S, self.T = DIMS[k]
        self.E = n_env
        self.seed = np.uint32(seed)
        self.st = np.zeros((self.S, n_env), dtype=f32)
        self.ep_idx = np.zeros(n_env, dtype=np.uint32)
        self.t = np.zeros(n_env, dtype=np.int32)
        self.nhaz = (4 if self.level == 1 else 8) if self.button else (2 if self.level == 1 else 4)
        self.nmov = (4 if self.level == 1 else 6) if self.button else (1 if self.level == 1 else 4)

    def _keys(self, ids):
        return ids.astype(np.uint32), (self.ep_idx[ids] - np.uint32(1)).astype(np.uint32)

    # ---- Button layout: regenerated from the reset's Philox stream ----------------------------------------
    def buttons(self, ids=None):
        """[(x, y)] of the 4 buttons of the current episodes (draws 1-2)."""
        ids = np.arange(self.E) if ids is None else np.asarray(ids)
        env, ep = self._keys(ids)
        out = []
        for h in range(2):
            q = philox4x32(env, ep, 1 + h, 0, self.seed, KEY_RESET)
            out += [(usym(q[0]) * P["ARENA"], usym(q[1]) * P["ARENA"]), (usym(q[2]) * P["ARENA"], usym(q[3]) * P["ARENA"])]
        return out

    def centres(self, ids=None):
        """[(gremlin, x, y)] of the hazards, then the gremlins' orbit centres (draws 3, 4, ...)."""
        ids = np.arange(self.E) if ids is None else np.asarray(ids)
        env, ep = self._keys(ids)
        out = []
        for h in range((self.nhaz + self.nmov) // 2):
            q = philox4x32(env, ep, 3 + h, 0, self.seed, KEY_RESET)
            for j in range(2):
                k = 2 * h + j
                out.append((k >= self.nhaz, usym(q[2 * j]) * P["ARENA"], usym(q[2 * j + 1]) * P["ARENA"]))
        return out

    def hazards_gremlins(self, ids=None, st=None):
        """[(gremlin, x, y)] of the hazards, then the gremlins at the phase held in the state."""
        ids = np.arange(self.E) if ids is None else np.asarray(ids)
        st = self.st[:, ids] if st is None else st
        pc, ps = st[10], st[11]
        out = []
        g = 0
        for grem, ox, oy in self.centres(ids):
            if not grem:
                out.append((False, ox, oy))
                continue
            qs = -ps if g >= 4 else ps
            ux, uy = [(pc, qs), (-qs, pc), (-pc, -qs), (qs, -pc)][g & 3]
            out.append((True, ox + B["GREM_TRAVEL"] * ux, oy + B["GREM_TRAVEL"] * uy))
            g += 1
        return out

    # ---- gym protocol -------------------------------------------------------------------------------------
    def reset(self, ids=None):
        if self.kind not in BP:
            return super().reset(ids)
        ids = np.arange(self.E) if ids is None else np.asarray(ids)
        env = ids.astype(np.uint32)
        ep = self.ep_idx[ids]
        r = philox4x32(env, ep, 0, 0, self.seed, KEY_RESET)
        st = np.zeros((self.S, len(ids)), dtype=f32)
        st[0] = usym(r[0]) * f32(0.5); st[1] = usym(r[1]) * f32(0.5)
        st[2], st[3] = _heading_from_box(usym(r[2]), usym(r[3]))
        g = philox4x32(env, ep, 0, 0, self.seed, KEY_GOAL)
        if self.button:
            st[7] = (g[0] % np.uint32(4)).astype(f32)
            st[10], st[11] = _heading_from_box(usym(g[1]), usym(g[2]))
        else:
            st[6] = usym(g[0]) * P["ARENA"]; st[7] = usym(g[1]) * P["ARENA"]
            nobj = 1 + self.nhaz + self.nmov
            for h in range((nobj + 1) // 2):
                q = philox4x32(env, ep, 1 + h, 0, self.seed, KEY_RESET)
                for j in range(2):
                    k = 2 * h + j
                    if k < nobj:
                        sc = B["BOX_START"] if k == 0 else P["ARENA"]
                        st[9 + 2 * k] = usym(q[2 * j]) * sc
                        st[10 + 2 * k] = usym(q[2 * j + 1]) * sc
        self.st[:, ids] = st
        self.ep_idx[ids] += np.uint32(1)
        self.t[ids] = 0
        return self.observe(ids)

    def observe(self, ids=None):
        if self.kind not in BP:
            return super().observe(ids)
        ids = np.arange(self.E) if ids is None else np.asarray(ids)
        st = self.st[:, ids]
        o = np.zeros((len(ids), self.D), dtype=f32)
        x, y, c, s = st[0], st[1], st[2], st[3]
        _sensors(o, st[4], st[5], st[6 if self.button else self.S - 1], c, s)
        if self.button:
            goal = st[7].astype(np.int64)
            live = st[9] == 0
            for b, (bx, by) in enumerate(self.buttons(ids)):
                # an object outside the lidar's reach (closeness 0) leaves its sector unchanged: park the
                # envs that do not see this button far away
                far = f32(1e6)
                _lidar(o, 12, np.where(goal == b, bx, far), np.where(goal == b, by, far), x, y, c, s)
                _lidar(o, 28, np.where(live, bx, far), np.where(live, by, far), x, y, c, s)
            for grem, ox, oy in self.hazards_gremlins(ids, st):
                _lidar(o, 44 if grem else 60, ox, oy, x, y, c, s)
        else:
            _lidar(o, 12, st[6], st[7], x, y, c, s)
            _lidar(o, 28, st[9], st[10], x, y, c, s)
            for k in range(self.nhaz):
                _lidar(o, 44, st[11 + 2 * k], st[12 + 2 * k], x, y, c, s)
            for k in range(self.nmov):
                _lidar(o, 60, st[11 + 2 * self.nhaz + 2 * k], st[12 + 2 * self.nhaz + 2 * k], x, y, c, s)
        return o

    def step(self, act, ids=None):
        if self.kind not in BP:
            return super().step(act, ids)
        ids = np.arange(self.E) if ids is None else np.asarray(ids)
        act = np.asarray(act, dtype=f32)
        st = [self.st[i, ids].copy() for i in range(self.S)]
        rew, cost = self._step_button(st, act, ids) if self.button else self._step_push(st, act, ids)
        for i in range(self.S):
            self.st[i, ids] = st[i]
        self.t[ids] += 1
        trunc = self.t[ids] >= self.T
        return self.observe(ids), rew.astype(f32), cost, np.zeros(len(ids), dtype=bool), trunc

    def _step_button(self, st, act, ids):
        n = len(ids)
        but = self.buttons(ids)
        goal = st[7].astype(np.int64)
        gx, gy = but[0]
        for b in range(1, 4):
            gx = np.where(goal == b, but[b][0], gx).astype(f32)
            gy = np.where(goal == b, but[b][1], gy).astype(f32)
        dist_old = np.sqrt(_dist2(gx, gy, st[0], st[1]))
        st[6] = st[4].copy()
        _advance(self.car, st, act)
        st[0] = _clamp(st[0]); st[1] = _clamp(st[1])
        dist = np.sqrt(_dist2(gx, gy, st[0], st[1]))
        rew = dist_old - dist
        live = st[9] == 0
        press = live & (dist <= B["BUTTON_R"])
        st[9] = np.where(live, st[9], st[9] - f32(1)).astype(f32)
        rew = np.where(press, rew + f32(1), rew).astype(f32)
        st[8] = np.where(press, st[8] + f32(1), st[8]).astype(f32)
        st[9] = np.where(press, f32(DELAY), st[9]).astype(f32)
        if press.any():
            env, ep = self._keys(ids)
            r = philox4x32(env, ep, np.uint32(16) + st[8].astype(np.uint32), 0, self.seed, KEY_GOAL)
            new = (goal + 1 + (r[0] % np.uint32(3)).astype(np.int64)) & 3
            st[7] = np.where(press, new.astype(f32), st[7]).astype(f32)
        st[10], st[11] = _rotate(st[10], st[11], B["GREM_W"] * P["DT"])
        cost = np.zeros(n, f32)
        for b, (bx, by) in enumerate(but):
            hit = live & (goal != b) & (_dist2(bx, by, st[0], st[1]) <= B["BUTTON_R"] * B["BUTTON_R"])
            cost = np.where(hit, f32(1), cost).astype(f32)
        for grem, ox, oy in self.hazards_gremlins(ids, np.stack(st)):
            lim = B["GREM_R"] * B["GREM_R"] if grem else P["HAZ_R"] * P["HAZ_R"]
            cost = np.where(_dist2(ox, oy, st[0], st[1]) <= lim, f32(1), cost).astype(f32)
        return rew, cost

    def _step_push(self, st, act, ids):
        n = len(ids)
        vp = self.S - 1
        rb_old = np.sqrt(_dist2(st[9], st[10], st[0], st[1]))
        bg_old = np.sqrt(_dist2(st[6], st[7], st[9], st[10]))
        st[vp] = st[4].copy()
        _advance(self.car, st, act)
        x = _clamp(st[0]); y = _clamp(st[1])
        st[0], st[1] = x, y
        dx = st[9] - x; dy = st[10] - y
        d = np.sqrt(dx * dx + dy * dy)
        touch = d < B["PUSH_D"]
        zero = d == 0
        dn = np.where(zero, f32(1), d)
        ux = np.where(zero, st[2], dx / dn).astype(f32)
        uy = np.where(zero, st[3], dy / dn).astype(f32)
        st[9] = np.where(touch, _clamp(x + B["PUSH_D"] * ux), st[9]).astype(f32)
        st[10] = np.where(touch, _clamp(y + B["PUSH_D"] * uy), st[10]).astype(f32)
        rb = np.sqrt(_dist2(st[9], st[10], x, y))
        bg = np.sqrt(_dist2(st[6], st[7], st[9], st[10]))
        rew = (rb_old - rb) + (bg_old - bg)
        hit = bg <= P["GOAL_R"]
        rew = np.where(hit, rew + f32(1), rew).astype(f32)
        st[8] = np.where(hit, st[8] + f32(1), st[8]).astype(f32)
        if hit.any():
            env, ep = self._keys(ids)
            g = philox4x32(env, ep, np.uint32(16) + st[8].astype(np.uint32), 0, self.seed, KEY_GOAL)
            st[6] = np.where(hit, usym(g[0]) * P["ARENA"], st[6]).astype(f32)
            st[7] = np.where(hit, usym(g[1]) * P["ARENA"], st[7]).astype(f32)
        cost = np.zeros(n, f32)
        for k in range(self.nhaz):
            inside = _dist2(st[11 + 2 * k], st[12 + 2 * k], x, y) <= B["PUSH_HAZ_R"] * B["PUSH_HAZ_R"]
            cost = np.where(inside, f32(1), cost).astype(f32)
        if self.level == 2:
            p0 = 11 + 2 * self.nhaz
            for k in range(self.nmov):
                inside = _dist2(st[p0 + 2 * k], st[p0 + 1 + 2 * k], x, y) <= B["PILLAR_R"] * B["PILLAR_R"]
                cost = np.where(inside, f32(1), cost).astype(f32)
        return rew, cost
