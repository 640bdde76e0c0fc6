"""CPU-side checks of the env renderer: fsrl_env_render refuses bad arguments before any device work (the descriptor's
state pointers are never dereferenced), DeviceVectorEnv validates render_mode / render_size, and the float32 twin of
tests/render_twin.py draws what each scene promises on hand-made states."""
import ctypes

import numpy as np
import pytest

import render_twin as rt
from oracle.envs_velocity import OracleVecEnvVel

FAKE = 1 << 20


def _descriptor(E=8, kind=0):
    from fsrl_b200 import _lib
    r = _lib.Rollout()
    r.kind, r.E, r.max_steps = kind, E, 300
    for f in ("env_state", "obs_cur", "env_t", "ep_idx", "act_ctr", "active", "done_now", "ep_rew", "ep_len", "stats"):
        setattr(r, f, FAKE)
    return r


def _render(r, ids, n, h=64, w=64, out=FAKE):
    from fsrl_b200 import _lib
    p = None if ids is None else np.asarray(ids, np.int32)
    rc = _lib.lib.fsrl_env_render(None if r is None else ctypes.byref(r), None if p is None else p.ctypes.data, n, h, w,
                                  None, out, None)
    return rc, _lib.last_error()


def test_render_rejects_bad_arguments_before_device_work():
    from fsrl_b200 import _lib
    cases = [
        (_descriptor(kind=9), None, 8, {}, "unknown env kind 9"),
        (_descriptor(), None, 0, {}, "n = 0 must be at least 1"),
        (_descriptor(), [0, 1], 0, {}, "n = 0 must be at least 1"),
        (_descriptor(), None, 4, {}, "without ids, n must be E = 8"),
        (_descriptor(), [1, 8], 2, {}, "ids[1] = 8 outside [0, E = 8)"),
        (_descriptor(), [-1], 1, {}, "ids[0] = -1 outside [0, E = 8)"),
        (_descriptor(), None, 8, dict(h=15), "frame size 15 x 64 outside [16, 1024]"),
        (_descriptor(), None, 8, dict(h=1025), "frame size 1025 x 64 outside [16, 1024]"),
        (_descriptor(), None, 8, dict(w=15), "frame size 64 x 15 outside [16, 1024]"),
        (_descriptor(), None, 8, dict(w=2048), "frame size 64 x 2048 outside [16, 1024]"),
        (None, None, 8, {}, "null descriptor"),
        (_descriptor(), None, 8, dict(out=None), "null output"),
    ]
    for r, ids, n, kw, msg in cases:
        rc, err = _render(r, ids, n, **kw)
        assert rc == _lib.FSRL_EINVAL and msg in err, (msg, rc, err)
    for field in ("env_state", "env_t", "ep_idx"):
        r = _descriptor()
        setattr(r, field, None)
        rc, err = _render(r, None, 8)
        assert rc == _lib.FSRL_EINVAL and "null state pointer" in err, (field, err)


def test_render_mode_and_size_are_validated():
    from fsrl_b200.envs import DeviceVectorEnv
    for mode in ("human", "rgb", ""):
        with pytest.raises(ValueError, match="render_mode"):
            DeviceVectorEnv("SafetyCarCircle-v0", 2, device="cpu", render_mode=mode)
    for size in ((15, 64), (64, 1025), (0, 0), (2048, 16)):
        with pytest.raises(ValueError, match="render_size"):
            DeviceVectorEnv("SafetyCarCircle-v0", 2, device="cpu", render_mode="rgb_array", render_size=size)
    venv = DeviceVectorEnv("SafetyCarCircle-v0", 2, device="cpu")
    assert venv.render() is None and venv.last_cost is None
    venv = DeviceVectorEnv("SafetyCarCircle-v0", 3, device="cpu", render_mode="rgb_array", render_size=(16, 1024))
    assert venv.render_size == (16, 1024) and tuple(venv.last_cost.shape) == (3,)
    with pytest.raises(RuntimeError, match="CUDA devices only"):   # well-formed, but drawing needs the GPU
        venv.render()


def _pixel(sc, x, y, height, width):
    """The (row, column) whose centre is nearest the world point (x, y)."""
    j = int((x - sc.x0) / (sc.x1 - sc.x0) * width)
    i = int((sc.y1 - y) / (sc.y1 - sc.y0) * height)
    return i, j


def _colour(c):
    return tuple(int(v) for v in rt.PALETTE[c])


def _goal1(robot=(0.5, 0.3), heading=(1.0, 0.0), hazard=(-1.0, 1.0)):
    """A PointGoal1 state with one hazard at `hazard`, the other hazards, the vase and the goal off screen."""
    st = np.zeros(28, np.float32)
    st[0], st[1] = robot
    st[2], st[3] = heading
    st[6:8] = 10.0
    st[9:27] = 10.0
    st[9], st[10] = hazard
    return st


def _draw(kind, st, cost=False, t=0, h=256, w=256):
    env = OracleVecEnvVel(kind, 1, 0)
    env.ep_idx[:] = 1
    sc = rt.scene(kind, st, t, 0, env, cost)
    return sc, rt.draw(sc, h, w)


def test_robot_colour_at_its_pixel_and_over_a_hazard():
    # a pixel just behind the robot's centre (the heading segment starts at the centre)
    for kind, st in [(5, _goal1()), (0, np.array([0.5, 0.3, 1.0, 0.0, 0.0, 0.0], np.float32))]:
        sc, fr = _draw(kind, st)
        assert tuple(fr[_pixel(sc, st[0] - 0.07, st[1], 256, 256)]) == _colour(rt.C_ROBOT), kind
        assert tuple(fr[_pixel(sc, st[0] + 0.15, st[1], 256, 256)]) == _colour(rt.C_HEADING), kind
    # a robot standing in a hazard is drawn over it; the hazard shows around it
    st = _goal1(robot=(-1.0, 1.0))
    sc, fr = _draw(5, st)
    assert tuple(fr[_pixel(sc, -1.07, 1.0, 256, 256)]) == _colour(rt.C_ROBOT)
    assert tuple(fr[_pixel(sc, -1.0, 0.83, 256, 256)]) == _colour(rt.C_HAZARD)


def test_cost_colour_only_when_the_last_cost_is_positive():
    st = _goal1()
    for cost, want in [(False, rt.C_ROBOT), (True, rt.C_COST)]:
        sc, fr = _draw(5, st, cost=cost)
        assert tuple(fr[_pixel(sc, st[0] - 0.07, st[1], 256, 256)]) == _colour(want)
    # through render(): last_cost 0 draws the robot colour, > 0 the cost colour
    S = st.reshape(-1, 1).repeat(3, 1)
    fr = rt.render(5, S, np.zeros(3, np.int32), np.ones(3, np.uint32), 0, 64, 64, last_cost=np.array([0.0, 1.0, -1.0]))
    assert (fr[0] == fr[2]).all() and not (fr[0] == fr[1]).all()
    assert (fr[1] == _colour(rt.C_COST)).all(-1).sum() > 0 and (fr[0] == _colour(rt.C_COST)).all(-1).sum() == 0


def test_hazard_disc_area():
    st = _goal1(robot=(1.5, -1.5))
    for h, w in [(256, 256), (300, 200)]:
        sc, fr = _draw(5, st, h=h, w=w)
        sx, sy = (sc.x1 - sc.x0) / w, (sc.y1 - sc.y0) / h
        n = (fr == _colour(rt.C_HAZARD)).all(-1).sum()
        want = np.pi * 0.2 ** 2 / (sx * sy)
        assert abs(n - want) <= 0.05 * want, (n, want)


def test_buttons_hidden_during_the_delay():
    env = OracleVecEnvVel(25, 1, 4)
    env.reset()
    st = env.st[:, 0].copy()
    counts = []
    for timer in (0.0, 5.0, 1.0, 0.0):
        st[9] = timer
        sc = rt.scene(25, st, 3, 0, env)
        fr = rt.draw(sc, 128, 128)
        counts.append(sum((fr == _colour(c)).all(-1).sum() for c in (rt.C_BUTTON, rt.C_GOAL)))
    assert counts[0] > 0 and counts[1] == 0 and counts[2] == 0 and counts[3] == counts[0]


def test_run_window_follows_the_robot():
    frames = []
    for x in (0.0, 3.37, -7.2):
        st = np.array([x, 0.1, 1.0, 0.0, 0.5, 0.0, 0.0], np.float32)
        sc, fr = _draw(1, st, h=128, w=128)
        assert sc.x0 < x < sc.x1 and abs((sc.x0 + sc.x1) / 2 - x) < 1e-6
        robot = (fr == _colour(rt.C_ROBOT)).all(-1)
        cols = np.nonzero(robot.any(0))[0]
        assert robot.sum() > 0 and abs((cols.min() + cols.max()) / 2 - 63.5) <= 3, cols
        frames.append(fr)
    # the robot sits in the same place, the corridor's ticks move under it
    assert not (frames[0] == frames[1]).all() and not (frames[1] == frames[2]).all()
