"""The Safety-Gymnasium navigation tasks (Point / Car on Circle 1-2 and Goal 1-2) on the CPU: the registry
and the C ABI agree with the env twin (oracle/envs_nav.py) on the dimensions, every config's default
task resolves, and the twin's models behave as csrc/envs.cuh documents them."""
import ctypes
import dataclasses

import numpy as np
import pytest

from oracle.envs_nav import DIMS, NAV, P, OracleVecEnvNav
from oracle.philox import action_uniform

NEW = {"SafetyPointCircle1Gymnasium-v0": 16, "SafetyPointCircle2Gymnasium-v0": 17,
       "SafetyCarCircle1Gymnasium-v0": 18, "SafetyCarCircle2Gymnasium-v0": 19,
       "SafetyPointGoal2Gymnasium-v0": 20, "SafetyCarGoal1Gymnasium-v0": 21, "SafetyCarGoal2Gymnasium-v0": 22}
CIRCLES = [t for t, k in NEW.items() if NAV[k][1]]
GOALS = [t for t, k in NEW.items() if not NAV[k][1]] + ["SafetyPointGoal1Gymnasium-v0"]
f32 = np.float32


def _scale(u):
    # map_action with scaling onto [-1, 1] (rollout.cu), as the device applies it
    return (f32(-1) + (f32(2) * (u + f32(1))) / f32(2)).astype(f32)


def _kind(task):
    from fsrl_b200 import envs
    return envs.KINDS[task]


@pytest.mark.parametrize("task", sorted(NEW))
def test_dims_agree_with_the_twin(task):
    from fsrl_b200 import envs
    kind = NEW[task]
    assert envs.KINDS[task] == kind
    assert envs.env_dims(kind) == DIMS[kind]
    D, A, S, T = DIMS[kind]
    e = envs.make(task)
    assert e.observation_space.shape == (D,) and e.action_space.shape == (A,)
    assert e.spec.max_episode_steps == T and e.state_dim == S
    assert S <= 32 and A <= 8 and D <= 64
    assert (D <= 40) == (task in CIRCLES)        # Circle fits the persistent PPO launch's obs-width gate


@pytest.mark.parametrize("kind", list(range(-1, 64)) + [128])   # to FSRL_ENV_PLUGIN_FIRST, and FSRL_ENV_PLUGIN_END
def test_unassigned_kinds_are_rejected(kind):
    """Every id below the plugin kinds: an assigned one reports its twin's widths and horizon, any other is an unknown
    kind to the widths query, the rollout and the renderer."""
    from fsrl_b200 import _lib, envs
    from oracle.envs_velocity import DIMS as ALL_DIMS
    if kind in ALL_DIMS:
        assert envs.env_dims(kind) == ALL_DIMS[kind]
        return
    with pytest.raises(Exception, match="unknown env kind"):
        envs.env_dims(kind)
    r = _lib.Rollout(kind=kind, E=8)
    assert _lib.lib.fsrl_env_reset_all(ctypes.byref(r), None) == _lib.FSRL_EINVAL
    assert f"unknown env kind {kind}" in _lib.last_error()
    assert _lib.lib.fsrl_env_render(ctypes.byref(r), None, 8, 64, 64, None, None, None) == _lib.FSRL_EINVAL
    assert f"unknown env kind {kind}" in _lib.last_error()


def test_every_config_default_task_resolves():
    from fsrl_b200 import config, envs
    seen = set()
    for mod in ("ppol_cfg", "cpo_cfg", "sacl_cfg", "ddpgl_cfg", "trpol_cfg", "focops_cfg", "cvpo_cfg"):
        m = getattr(config, mod)
        for name in dir(m):
            cls = getattr(m, name)
            if isinstance(cls, type) and dataclasses.is_dataclass(cls):
                task = cls().task
                assert envs.make(task).spec.id == task, (mod, name)
                seen.add(task)
    assert "SafetyPointCircle1Gymnasium-v0" in seen


def _steer(env, tx, ty, fwd, gain, car):
    """Actions that turn the robot towards the world direction (tx, ty) and drive at `fwd`."""
    st = env.st
    c, s = st[2], st[3]
    n = np.sqrt(tx * tx + ty * ty) + 1e-9
    cross = (c * ty - s * tx) / n
    dot = (c * tx + s * ty) / n
    turn = np.where(dot < 0, np.sign(cross + 1e-12), np.clip(gain * cross, -1, 1))
    f = np.where(dot > 0.5, fwd, 0.0)
    if car:
        a = np.stack([f - turn * 0.5, f + turn * 0.5], 1)
    else:
        a = np.stack([f, turn], 1)
    return np.clip(a, -1, 1).astype(f32)


def test_car_wheels():
    env = OracleVecEnvNav(NEW["SafetyCarCircle1Gymnasium-v0"], 8, 3)
    env.reset()
    c0, s0 = env.st[2].copy(), env.st[3].copy()
    for _ in range(50):
        env.step(np.full((8, 2), 0.7, f32))
    # equal wheel commands: no turn, and the robot moved along its heading
    assert np.allclose(env.st[2], c0, atol=1e-6) and np.allclose(env.st[3], s0, atol=1e-6)
    assert np.all(env.st[4] > 0.6)
    x0, y0 = env.st[0].copy(), env.st[1].copy()
    env.st[4:6] = 0
    for _ in range(20):
        env.step(np.tile(np.array([[0.5, -0.5]], f32), (8, 1)))
    # opposite commands: the car turns in place (clockwise for a faster left wheel)
    assert np.array_equal(env.st[0], x0) and np.array_equal(env.st[1], y0)
    assert np.all(np.abs(env.st[2] - c0) + np.abs(env.st[3] - s0) > 0.5)


@pytest.mark.parametrize("task", CIRCLES)
def test_tangential_controller_earns_positive_reward(task):
    E = 64
    env = OracleVecEnvNav(NEW[task], E, 5)
    env.reset()
    total = np.zeros(E)
    for _ in range(env.T):
        x, y = env.st[0], env.st[1]
        r = np.sqrt(x * x + y * y) + 1e-6
        k = 2.0 * (1.5 - r)
        a = _steer(env, -y / r + k * x / r, x / r + k * y / r, 0.8, 3.0, env.car)
        _, rew, _, _, _ = env.step(a)
        total += rew
    assert total.mean() > 0.0 and (total > 0).mean() > 0.9, total


@pytest.mark.parametrize("task", CIRCLES)
def test_driving_along_y_costs_only_at_level_2(task):
    env = OracleVecEnvNav(NEW[task], 1, 0)
    env.reset()
    env.st[:, 0] = 0
    env.st[3, 0] = 1                          # at the origin, heading +y
    a = np.array([[1, 1]] if env.car else [[1, 0]], f32)
    costs = [env.step(a)[2][0] for _ in range(100)]
    assert env.st[1, 0] > 2 and env.st[0, 0] == 0
    assert (max(costs) == 1) == (env.level == 2)


@pytest.mark.parametrize("task", GOALS)
def test_go_to_goal_controller_collects_goals(task):
    E = 32
    env = OracleVecEnvNav(_kind(task), E, 9)
    env.reset()
    for _ in range(env.T):
        a = _steer(env, env.st[6] - env.st[0], env.st[7] - env.st[1], 1.0, 4.0, "Car" in task)
        env.step(a)
    assert (env.st[8] >= 1).mean() > 0.75, env.st[8]


@pytest.mark.parametrize("task", ["SafetyPointGoal2Gymnasium-v0", "SafetyCarGoal2Gymnasium-v0"])
def test_touching_a_level_2_vase_costs(task):
    E = 16
    env = OracleVecEnvNav(NEW[task], E, 4)
    env.reset()
    lay = env.layout()
    assert sum(v for v, _, _ in lay) == 10 and len(lay) == 20
    probed = 0
    for i, (vase, vx, vy) in enumerate(lay):
        if not vase:
            continue
        # no other hazard or vase within reach of the probes below
        clear = np.all([(vx - ox) ** 2 + (vy - oy) ** 2 > 0.7 ** 2 for j, (_, ox, oy) in enumerate(lay) if j != i], 0)
        for off, want in ((0.0, 1), (0.2, 1), (0.35, 0)):
            env.st[0], env.st[1] = vx + f32(off), vy
            env.st[2], env.st[3], env.st[4], env.st[5] = 1, 0, 0, 0
            inside = np.abs(env.st[0]) < P["ARENA"]
            _, _, cost, _, _ = env.step(np.zeros((E, 2), f32))
            m = clear & inside
            assert np.all(cost[m] == want), (off, cost[m])
            probed += int(m.sum())
    assert probed > 0


@pytest.mark.parametrize("task", sorted(NEW))
def test_random_play_has_nonzero_cost_rate(task):
    E = 256
    env = OracleVecEnvNav(NEW[task], E, 7)
    env.reset()
    ids = np.arange(E)
    ctr = np.zeros(E, np.uint32)
    cost = 0.0
    steps = min(env.T, 400)
    for _ in range(steps):
        a = _scale(action_uniform(np.uint32(3), ids, ctr, env.A))
        ctr += np.uint32(1)
        _, _, c, term, trunc = env.step(a)
        assert not term.any()
        cost += float(c.sum())
    assert cost / (E * steps) > 0.0
    assert not trunc.any() or steps == env.T


def test_existing_kinds_run_the_unchanged_twins():
    from oracle.envs_flight import OracleVecEnvExt
    for kind in range(9):
        a, b = OracleVecEnvExt(kind, 9, 5), OracleVecEnvNav(kind, 9, 5)
        assert np.array_equal(a.reset(), b.reset())
        for t in range(30):
            act = _scale(action_uniform(np.uint32(1), np.arange(9), np.full(9, t, np.uint32), a.A))
            for x, y in zip(a.step(act), b.step(act)):
                assert np.array_equal(x, y)
        assert np.array_equal(a.st, b.st)
