"""Float32 numpy restatement of csrc/render.cu: the scene decode of every env family and the pixel loop, in the CUDA
code's operation order, so frames match ``fsrl_env_render`` bit for bit.  The layouts the device regenerates from the
reset's Philox stream (Goal2's hazards and vases, Button's buttons, hazards and gremlins) come from the oracle env
classes, which regenerate them for step parity."""
from __future__ import annotations

import numpy as np

from oracle.envs_flight import _sincos
from oracle.envs_velocity import DIMS, OracleVecEnvVel

f32 = np.float32
MAX_PRIM = 32
BOX, DISC, SEG = 0, 1, 2
(C_BG, C_FLOOR, C_WALL, C_CIRCLE, C_ROBOT, C_HEADING, C_COST, C_HAZARD, C_VASE, C_GOAL, C_BUTTON, C_GREMLIN, C_BOX,
 C_PILLAR, C_GROUND, C_LIMB, C_GAUGE_BG, C_GAUGE, C_MARK, C_TICK) = range(20)
PALETTE = np.array([
    (24, 24, 32), (54, 58, 70), (120, 40, 40), (70, 160, 90), (70, 130, 230), (250, 250, 250), (240, 60, 40),
    (150, 60, 170), (90, 200, 220), (60, 210, 80), (230, 190, 50), (240, 120, 30), (200, 150, 90), (140, 140, 150),
    (90, 80, 60), (180, 200, 240), (60, 60, 60), (80, 200, 120), (250, 250, 250), (80, 84, 100)], np.uint8)

CIRCLE = {0: (1.5, 1.125), 2: (1.5, 1.125), 4: (3.0, 2.25), 7: (1.5, 1.125)}   # kind -> (R, XLIM)
RUN = {1: (0.6, 1.2), 3: (0.6, 1.5), 6: (1.0, 0.8), 8: (0.6, 1.0)}                # kind -> (YLIM, VLIM)
VCOST = {33: 2.8, 34: 0.35, 35: 0.05, 36: 1.7, 37: 2.5}
Q0 = {33: 5, 34: 5, 35: 5, 36: 5, 37: 10}
ARENA, GOAL_R, HAZ_R, PUSH_HAZ_R, CIRC_R, WALL, Z0 = 2.0, 0.3, 0.2, 0.3, 1.5, 1.125, 1.0


def _wide_sincos(a):
    s, c = _sincos(a * f32(0.25))
    for _ in range(2):
        s, c = (s * c) * f32(2), c * c - s * s
    return s, c


def _turn(c, s, ck, sk):
    return c * ck - s * sk, s * ck + c * sk


class Scene:
    def __init__(self):
        self.p = []
        self.x0 = self.x1 = self.y0 = self.y1 = f32(0)

    def put(self, *prim):
        if len(self.p) < MAX_PRIM:
            self.p.append(tuple(prim[:2]) + tuple(f32(v) for v in prim[2:]))

    def box(self, x0, y0, x1, y1, col):
        self.put(BOX, col, x0, y0, x1, y1, 0, 0)

    def disc(self, cx, cy, r, col):
        r = f32(r)
        self.put(DISC, col, cx, cy, 0, r * r, 0, 0)

    def ring(self, cx, cy, r0, r1, col):
        self.put(DISC, col, cx, cy, r0 * r0, r1 * r1, 0, 0)

    def seg(self, ax, ay, bx, by, hw, col):
        ax, ay, hw = f32(ax), f32(ay), f32(hw)
        dx, dy = f32(bx) - ax, f32(by) - ay
        self.put(SEG, col, ax, ay, dx, dy, dx * dx + dy * dy, hw * hw)

    def window(self, cx, cy, hx, hy):
        cx, cy, hx, hy = f32(cx), f32(cy), f32(hx), f32(hy)
        self.x0, self.x1, self.y0, self.y1 = cx - hx, cx + hx, cy - hy, cy + hy

    def robot(self, x, y, c, s, r, hl, hw, cost):
        self.disc(x, y, r, C_COST if cost else C_ROBOT)
        self.seg(x, y, x + f32(hl) * c, y + f32(hl) * s, hw, C_HEADING)

    def gauge(self, v, lim, vertical):
        v, lim = f32(v), f32(lim)
        L, H = self.x1 - self.x0, self.y1 - self.y0
        frac = min(f32(1), max(f32(0), v / (f32(2) * lim)))
        col = C_COST if not vertical and v > lim else C_GAUGE
        if not vertical:
            g0, g1 = self.x0 + L * f32(0.05), self.x1 - L * f32(0.05)
            h0, h1 = self.y0 + H * f32(0.03), self.y0 + H * f32(0.07)
            gl = g1 - g0
            m, mw = g0 + f32(0.5) * gl, L * f32(0.004)
            self.box(g0, h0, g1, h1, C_GAUGE_BG)
            self.box(g0, h0, g0 + frac * gl, h1, col)
            self.box(m - mw, h0 - H * f32(0.01), m + mw, h1 + H * f32(0.01), C_MARK)
        else:
            g0, g1 = self.y0 + H * f32(0.05), self.y1 - H * f32(0.05)
            h0, h1 = self.x0 + L * f32(0.03), self.x0 + L * f32(0.07)
            gl = g1 - g0
            m, mw = g0 + f32(0.5) * gl, H * f32(0.004)
            self.box(h0, g0, h1, g1, C_GAUGE_BG)
            self.box(h0, g0, h1, g0 + frac * gl, col)
            self.box(h0 - L * f32(0.01), m - mw, h1 + L * f32(0.01), m + mw, C_MARK)

    def progress(self, t, T):
        L, H = self.x1 - self.x0, self.y1 - self.y0
        frac = min(f32(1), f32(t) / f32(T))
        self.box(self.x0, self.y1 - H * f32(0.015), self.x0 + frac * L, self.y1, C_MARK)

    def limbs(self, x, y, c, s, q, lens, hw):
        for k in range(len(q)):
            sn, cs = _wide_sincos(f32(q[k]))
            c, s = _turn(c, s, cs, sn)
            x2, y2 = x + f32(lens[k]) * c, y + f32(lens[k]) * s
            self.seg(x, y, x2, y2, hw, C_LIMB)
            x, y = x2, y2


def _bullet(sc, kind, st, cost):
    ant, ball, drone = kind in (4, 6), kind in (2, 3), kind in (7, 8)
    RR = f32(0.2 if ant else 0.1)
    x, y = st[0], st[1]
    if ball:   # the ball has no heading: its velocity, 0.25 s ahead
        c, s, hl = st[2], st[3], f32(0.25)
    else:
        c, s = (st[3], st[4]) if drone else (st[2], st[3])
        hl = f32(2) * RR
    if kind in CIRCLE:
        R, XLIM = (f32(v) for v in CIRCLE[kind])
        sc.window(0, 0, f32(1.3) * R, f32(1.3) * R)
        sc.box(sc.x0, sc.y0, -XLIM, sc.y1, C_WALL)
        sc.box(XLIM, sc.y0, sc.x1, sc.y1, C_WALL)
        sc.ring(0, 0, f32(0.98) * R, f32(1.02) * R, C_CIRCLE)
        sc.robot(x, y, c, s, RR, hl, f32(0.35) * RR, cost)
        if drone:
            sc.gauge(st[2], Z0, True)
    else:
        YLIM, VLIM = (f32(v) for v in RUN[kind])
        sc.window(x, 0, f32(2) * YLIM, f32(2) * YLIM)
        sc.box(sc.x0, YLIM, sc.x1, sc.y1, C_WALL)
        sc.box(sc.x0, sc.y0, sc.x1, -YLIM, C_WALL)
        tw = f32(0.01) * YLIM
        k = np.ceil(sc.x0)
        while k <= sc.x1:
            sc.box(k - tw, -YLIM, k + tw, YLIM, C_TICK)
            k = k + f32(1)
        sc.robot(x, y, c, s, RR, hl, f32(0.35) * RR, cost)
        if ball:
            v = np.sqrt(st[2] * st[2] + st[3] * st[3])
        elif drone:
            v = np.sqrt(st[5] * st[5] + st[6] * st[6])
        else:
            v = st[4]
        sc.gauge(v, VLIM, False)


def _nav(sc, kind, st, env, e, cost):
    RR = f32(0.15)
    if 16 <= kind <= 19:
        sc.window(0, 0, f32(1.3) * f32(CIRC_R), f32(1.3) * f32(CIRC_R))
        W = f32(WALL)
        sc.box(sc.x0, sc.y0, -W, sc.y1, C_WALL)
        sc.box(W, sc.y0, sc.x1, sc.y1, C_WALL)
        if kind in (17, 19):
            sc.box(sc.x0, W, sc.x1, sc.y1, C_WALL)
            sc.box(sc.x0, sc.y0, sc.x1, -W, C_WALL)
        sc.ring(0, 0, f32(0.98) * f32(CIRC_R), f32(1.02) * f32(CIRC_R), C_CIRCLE)
    else:
        A = f32(ARENA)
        sc.window(0, 0, f32(1.1) * A, f32(1.1) * A)
        sc.box(-A, -A, A, A, C_FLOOR)
        ids = np.array([e])
        if kind in (5, 20, 21, 22):
            sc.disc(st[6], st[7], GOAL_R, C_GOAL)
            if kind in (5, 21):
                objs = [(False, st[9 + 2 * h], st[10 + 2 * h]) for h in range(8)] + [(True, st[25], st[26])]
            else:
                objs = [(v, ox[0], oy[0]) for v, ox, oy in env.layout(ids, st[:, None])]
            for vase, ox, oy in objs:
                if vase:
                    sc.box(ox - f32(0.1), oy - f32(0.1), ox + f32(0.1), oy + f32(0.1), C_VASE)
                else:
                    sc.disc(ox, oy, HAZ_R, C_HAZARD)
        elif 24 <= kind <= 27:
            if st[9] == 0:
                goal = int(st[7])
                for k, (bx, by) in enumerate(env.buttons(ids)):
                    sc.disc(bx[0], by[0], 0.1, C_GOAL if k == goal else C_BUTTON)
            for grem, ox, oy in env.hazards_gremlins(ids, st[:, None]):
                ox, oy = ox[0], oy[0]
                if grem:
                    sc.box(ox - f32(0.1), oy - f32(0.1), ox + f32(0.1), oy + f32(0.1), C_GREMLIN)
                else:
                    sc.disc(ox, oy, HAZ_R, C_HAZARD)
        else:
            nhaz, npil = (2, 1) if kind in (28, 30) else (4, 4)
            sc.disc(st[6], st[7], GOAL_R, C_GOAL)
            for h in range(nhaz):
                sc.disc(st[11 + 2 * h], st[12 + 2 * h], PUSH_HAZ_R, C_HAZARD)
            p0 = 11 + 2 * nhaz
            for p in range(npil):
                sc.disc(st[p0 + 2 * p], st[p0 + 2 * p + 1], 0.25, C_PILLAR)
            sc.box(st[9] - f32(0.15), st[10] - f32(0.15), st[9] + f32(0.15), st[10] + f32(0.15), C_BOX)
    sc.robot(st[0], st[1], st[2], st[3], RR, f32(2) * RR, f32(0.35) * RR, cost)


def _velocity(sc, kind, st, cost):
    q0 = Q0[kind]
    col = C_COST if cost else C_ROBOT
    zero = f32(0)
    if kind == 35:
        sc.window(0, 0, 1.0, 1.0)
        c, s = st[1], st[2]
        sc.seg(0, 0, f32(0.35) * c, f32(0.35) * s, 0.06, col)
        sc.limbs(zero, zero, -c, -s, st[q0:q0 + 2], (0.35, 0.35), 0.05)
        sc.gauge(st[3] * c, VCOST[kind], False)
    elif kind == 37:
        sc.window(0, 0, 1.2, 1.2)
        c, s = st[2], st[3]
        H = f32(0.70710678)
        for k, (dc, ds) in enumerate(((H, H), (-H, H), (-H, -H), (H, -H))):
            lc, ls = _turn(c, s, dc, ds)
            sc.limbs(zero, zero, lc, ls, [st[q0 + k], st[q0 + 4 + k]], (0.35, 0.35), 0.05)
        sc.robot(zero, zero, c, s, 0.2, 0.4, 0.06, cost)
        vx, vy = st[4] * c, st[4] * s
        sc.gauge(np.sqrt(vx * vx + vy * vy), VCOST[kind], False)
    else:
        cheetah = kind == 33
        z = st[0]
        sn, cs = _wide_sincos(st[2])
        sc.window(0, 0.7 if cheetah else 1.0, 1.5 if cheetah else 1.3, 1.0 if cheetah else 1.3)
        sc.box(sc.x0, sc.y0, sc.x1, 0, C_GROUND)
        if cheetah:
            hx, hy = f32(0.5) * cs, f32(0.5) * sn
            bx, by, fx, fy = zero - hx, z - hy, hx, z + hy
            sc.limbs(bx, by, sn, zero - cs, st[q0:q0 + 3], (0.3, 0.3, 0.2), 0.04)
            sc.limbs(fx, fy, sn, zero - cs, st[q0 + 3:q0 + 6], (0.3, 0.3, 0.2), 0.04)
            sc.seg(bx, by, fx, fy, 0.06, col)
        else:
            hx, hy = f32(0.2) * sn, f32(0.2) * cs
            px, py = hx, z - hy
            sc.limbs(px, py, sn, zero - cs, st[q0:q0 + 3], (0.45, 0.5, 0.2), 0.04)
            if kind == 36:
                sc.limbs(px, py, sn, zero - cs, st[q0 + 3:q0 + 6], (0.45, 0.5, 0.2), 0.04)
            sc.seg(px, py, zero - hx, z + hy, 0.06, col)
        sc.gauge(st[4], VCOST[kind], False)


def scene(kind, st, env_t, e, env, cost=False):
    """The primitives and window of env e: st is its state column (S,), env an oracle env holding the episode keys."""
    sc = Scene()
    st = np.asarray(st, f32)
    if kind <= 8 and kind != 5:
        _bullet(sc, kind, st, cost)
    elif kind < 33:
        _nav(sc, kind, st, env, e, cost)
    else:
        _velocity(sc, kind, st, cost)
    sc.progress(int(env_t), DIMS[kind][3])
    return sc


def _covers(p, X, Y):
    t, _, a, b, c, d, e, f = p
    if t == BOX:
        return (X >= a) & (X <= c) & (Y >= b) & (Y <= d)
    ux, uy = X - a, Y - b
    if t == DISC:
        d2 = ux * ux + uy * uy
        return (d2 >= c) & (d2 <= d)
    if e > 0:
        tt = np.minimum(f32(1), np.maximum(f32(0), (ux * c + uy * d) / e))
    else:
        tt = f32(0)
    ex, ey = ux - tt * c, uy - tt * d
    return ex * ex + ey * ey <= f


def draw(sc, height, width):
    """The (height, width, 3) frame of a scene."""
    sx = (sc.x1 - sc.x0) / f32(width)
    sy = (sc.y1 - sc.y0) / f32(height)
    X = (sc.x0 + (np.arange(width, dtype=f32) + f32(0.5)) * sx)[None, :]
    Y = (sc.y1 - (np.arange(height, dtype=f32) + f32(0.5)) * sy)[:, None]
    X, Y = np.broadcast_to(X, (height, width)), np.broadcast_to(Y, (height, width))
    col = np.full((height, width), C_BG, np.int64)
    for p in sc.p:
        col[_covers(p, X, Y)] = p[1]
    return PALETTE[col]


def render(kind, st, env_t, ep_idx, seed, height, width, ids=None, last_cost=None):
    """Frames (n, height, width, 3) u8 of the envs ``ids`` (all by default) from the state ``st`` (S, E), the step
    counters ``env_t`` and episode counters ``ep_idx`` (E,) and the vector env's seed, as fsrl_env_render draws them."""
    st = np.asarray(st, f32)
    E = st.shape[1]
    env = OracleVecEnvVel(kind, E, seed)
    env.st = st
    env.ep_idx = np.asarray(ep_idx).astype(np.uint32)
    ids = np.arange(E) if ids is None else np.asarray(ids)
    out = np.empty((len(ids), height, width, 3), np.uint8)
    for k, e in enumerate(ids):
        cost = last_cost is not None and last_cost[e] > 0
        out[k] = draw(scene(kind, st[:, e], env_t[e], int(e), env, cost), height, width)
    return out
