"""Float32 twins of the scenes the drawn test env plugins (tests/envs_render/*.h) describe, restated on
tests/render_twin.py's Scene and drawn by its pixel loop, with what csrc/render.cuh adds around a struct's draw: the
default window [-1, 1] x [-1, 1], the cap of MAX_PRIM - 1 primitives and the progress bar t / T."""
from __future__ import annotations

import os

import numpy as np

import render_twin as rt
from env_plugin_twin import ARENA, GOAL_R, HAZ_R, NHAZ, ROOT

f32 = np.float32
RENDER_ENV_DIR = os.path.join(ROOT, "tests", "envs_render")
DRAW_MAX = rt.MAX_PRIM - 1          # primitives a draw may add; the progress bar takes the last one
CROWDED_N, CROWDED_R = 40, 0.024


def header(name):
    return os.path.join(RENDER_ENV_DIR, name + ".h")


def hazard_dash_draw(sc, st, cost):
    """tests/envs_render/hazard_dash_drawn.h: floor, goal, 12 hazards, the robot heading along its velocity, the
    energy gauge (19 primitives)."""
    sc.window(0, 0, f32(1.1) * ARENA, f32(1.1) * ARENA)
    sc.box(-ARENA, -ARENA, ARENA, ARENA, rt.C_FLOOR)
    sc.disc(st[4], st[5], GOAL_R, rt.C_GOAL)
    for h in range(NHAZ):
        sc.disc(st[8 + 2 * h], st[9 + 2 * h], HAZ_R, rt.C_HAZARD)
    sc.robot(st[0], st[1], st[2], st[3], f32(0.1), f32(0.5), f32(0.035), cost)
    sc.gauge(st[6], f32(1.0), True)


def crowded_x(k):
    """The centre abscissa of disc k of tests/envs_render/crowded.h."""
    return f32(-0.975) + f32(0.05) * f32(k)


def crowded_draw(sc, st, cost):
    """tests/envs_render/crowded.h: no window, 40 discs in a row at height st[0]."""
    for k in range(CROWDED_N):
        col = rt.C_COST if k == 0 and cost else rt.C_GOAL if k % 2 else rt.C_HAZARD
        sc.disc(crowded_x(k), st[0], CROWDED_R, col)


def scene(draw, st, t, T, cost=False):
    """The scene fsrl_env_render builds around a plugin's draw for one env: st its state column (S,), t its step."""
    sc = rt.Scene()
    sc.window(0, 0, 1, 1)
    draw(sc, np.asarray(st, f32), cost)
    del sc.p[DRAW_MAX:]
    sc.progress(int(t), T)
    return sc


def render(draw, T, st, env_t, height, width, ids=None, last_cost=None):
    """Frames (n, height, width, 3) u8 of the envs ``ids`` (all by default) from the state ``st`` (S, E) and the step
    counters ``env_t`` (E,), as fsrl_env_render draws a plugin whose struct's draw is ``draw``."""
    st = np.asarray(st, f32)
    ids = np.arange(st.shape[1]) if ids is None else np.asarray(ids)
    out = np.empty((len(ids), height, width, 3), np.uint8)
    for k, e in enumerate(ids):
        cost = last_cost is not None and last_cost[e] > 0
        out[k] = rt.draw(scene(draw, st[:, e], env_t[e], T, cost), height, width)
    return out


def pixel(sc, x, y, height, width):
    """The (row, column) whose centre is nearest the world point (x, y) in a frame of sc."""
    sx, sy = (sc.x1 - sc.x0) / f32(width), (sc.y1 - sc.y0) / f32(height)
    return int(np.floor((sc.y1 - f32(y)) / sy)), int(np.floor((f32(x) - sc.x0) / sx))
