"""The Safety-Gymnasium Button and Push tasks (Point / Car, levels 1-2) on the CPU: the registry, the C ABI and
the env twin (oracle/envs_button_push.py) agree on the dimensions, and the twin's models behave as
csrc/envs.cuh documents them.  The model checks catch a twin and kernel that agree with each other but are
both wrong."""
import numpy as np
import pytest

from oracle.envs_button_push import BP, DELAY, DIMS, B, OracleVecEnvBP
from oracle.envs_nav import P
from oracle.philox import action_uniform
from test_nav_envs_host import _scale, _steer

NEW = {"SafetyPointButton1Gymnasium-v0": 24, "SafetyPointButton2Gymnasium-v0": 25,
       "SafetyCarButton1Gymnasium-v0": 26, "SafetyCarButton2Gymnasium-v0": 27,
       "SafetyPointPush1Gymnasium-v0": 28, "SafetyPointPush2Gymnasium-v0": 29,
       "SafetyCarPush1Gymnasium-v0": 30, "SafetyCarPush2Gymnasium-v0": 31}
BUTTONS = [t for t, k in NEW.items() if BP[k][1]]
PUSHES = [t for t, k in NEW.items() if not BP[k][1]]
f32 = np.float32


def _goal_button(env):
    but = env.buttons()
    g = env.st[7].astype(np.int64)
    return np.choose(g, [b[0] for b in but]), np.choose(g, [b[1] for b in but])


def _push(env):
    """Drive to a point behind the box on the goal's far side, then push it along the box -> goal line."""
    st = env.st
    x, y, bx, by, gx, gy = st[0], st[1], st[9], st[10], st[6], st[7]
    ux, uy = gx - bx, gy - by
    n = np.sqrt(ux * ux + uy * uy) + 1e-9
    ux, uy = ux / n, uy / n
    rx, ry = bx - x, by - y
    aligned = (rx * ux + ry * uy) / (np.sqrt(rx * rx + ry * ry) + 1e-9) > 0.9
    tx = np.where(aligned, gx - x, bx - 0.5 * ux - x)
    ty = np.where(aligned, gy - y, by - 0.5 * uy - y)
    return _steer(env, tx, ty, np.where(aligned, 0.6, 1.0), 4.0, env.car)


def _random_actions(env, ctr):
    a = _scale(action_uniform(np.uint32(3), np.arange(env.E), ctr, env.A))
    ctr += np.uint32(1)
    return a


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
    assert D == 76 and A == 2 and S <= 32 and T == 1000
    env = OracleVecEnvBP(kind, 3, 1)
    assert env.reset().shape == (3, D) and env.st.shape == (S, 3)


@pytest.mark.parametrize("kind", list(range(9, 16)) + [23, 32])
def test_unassigned_kinds_are_rejected(kind):
    from fsrl_b200 import envs
    with pytest.raises(Exception, match="unknown env kind"):
        envs.env_dims(kind)


def test_the_engine_takes_the_widest_critic_input():
    """obs + act of these tasks is 78 wide: the engine's input-gradient stride (exported by the library) covers it."""
    from fsrl_b200.engine import DX_LD
    assert DX_LD >= 76 + 2


@pytest.mark.parametrize("task", BUTTONS)
def test_pressing_the_goal_button_moves_the_goal(task):
    E = 32
    env = OracleVecEnvBP(NEW[task], E, 9)
    env.reset()
    presses = 0
    for _ in range(400):
        gx, gy = _goal_button(env)
        goal, count = env.st[7].copy(), env.st[8].copy()
        _, rew, _, _, _ = env.step(_steer(env, gx - env.st[0], gy - env.st[1], 1.0, 4.0, env.car))
        pressed = env.st[8] > count
        # a press: +1 over the distance progress (< 0.1 per step), and the goal moves to another button
        assert np.all(rew[pressed] > 0.9) and np.all(rew[~pressed] < 0.1)
        assert np.all(env.st[7][pressed] != goal[pressed]) and np.all(env.st[7][~pressed] == goal[~pressed])
        assert np.all(env.st[9][pressed] == DELAY)
        presses += int(pressed.sum())
    assert (env.st[8] >= 1).mean() > 0.75 and presses > 2 * E, env.st[8]


@pytest.mark.parametrize("task", ["SafetyPointButton1Gymnasium-v0", "SafetyCarButton2Gymnasium-v0"])
def test_buttons_lidar_is_zero_for_exactly_the_delay_after_a_press(task):
    E = 32
    env = OracleVecEnvBP(NEW[task], E, 9)
    env.reset()
    hidden = np.zeros(E, np.int64)        # observations since the last press with an all-zero buttons lidar
    runs = []
    for _ in range(400):
        gx, gy = _goal_button(env)
        count = env.st[8].copy()
        obs, _, _, _, _ = env.step(_steer(env, gx - env.st[0], gy - env.st[1], 1.0, 4.0, env.car))
        pressed = env.st[8] > count
        zero = ~obs[:, 28:44].any(1)
        # a live lidar reads a button within 2.9 (< LIDAR_MAX = 3), which one nearly always is in the 4 x 4 arena
        near = np.min([(bx - env.st[0]) ** 2 + (by - env.st[1]) ** 2 for bx, by in env.buttons()], 0) < 2.9 ** 2
        assert np.all(zero[pressed])
        assert np.all(zero[near] == (env.st[9][near] > 0))
        ended = ~zero & near & (hidden > 0)
        runs += hidden[ended].tolist()
        hidden = np.where(pressed | (zero & (hidden > 0)), hidden + 1, np.where(near, 0, hidden))
    assert len(runs) > E and set(runs) == {DELAY}, runs


@pytest.mark.parametrize("task", BUTTONS)
def test_touching_a_wrong_button_costs_only_while_the_buttons_are_live(task):
    E = 32
    env = OracleVecEnvBP(NEW[task], E, 4)
    env.reset()
    but = env.buttons()
    goal = env.st[7].astype(np.int64)
    probed = 0
    for b, (bx, by) in enumerate(but):
        others = [(ox, oy) for j, (ox, oy) in enumerate(but) if j != b] + \
                 [(ox, oy) for _, ox, oy in env.hazards_gremlins()]
        clear = np.all([(bx - ox) ** 2 + (by - oy) ** 2 > 0.7 ** 2 for ox, oy in others], 0) & (goal != b)
        for timer, want in ((0, 1), (5, 0), (1, 0)):
            env.st[0], env.st[1] = bx, by
            env.st[2], env.st[3], env.st[4], env.st[5] = 1, 0, 0, 0
            env.st[7], env.st[8], env.st[9] = goal, 0, timer
            _, _, cost, _, _ = env.step(np.zeros((E, 2), f32))
            assert np.all(cost[clear] == want), (timer, cost[clear])
            assert np.all(env.st[8][clear] == 0)        # standing on a wrong button presses nothing
        probed += int(clear.sum())
    assert probed > 0


@pytest.mark.parametrize("task", ["SafetyPointButton1Gymnasium-v0", "SafetyCarButton2Gymnasium-v0"])
def test_gremlins_orbit_their_centres(task):
    E = 8
    env = OracleVecEnvBP(NEW[task], E, 2)
    env.reset()
    centres = [(ox, oy) for grem, ox, oy in env.centres() if grem]
    assert len(centres) == env.nmov == (4 if env.level == 1 else 6)
    prev = None
    for _ in range(60):
        env.step(np.zeros((E, 2), f32))
        grem = [(ox, oy) for g, ox, oy in env.hazards_gremlins() if g]
        off = [(gx - cx, gy - cy) for (gx, gy), (cx, cy) in zip(grem, centres)]
        for dx, dy in off:
            assert np.allclose(np.sqrt(dx.astype(np.float64) ** 2 + dy ** 2), 0.35, rtol=0, atol=2e-6)
        if prev is not None:
            for k, ((dx, dy), (px, py)) in enumerate(zip(off, prev)):
                turn = px * dy - py * dx       # > 0: counter-clockwise
                assert np.all(np.abs(dx - px) + np.abs(dy - py) > 0.01), k
                assert np.all(turn > 0) if k < 4 else np.all(turn < 0), k
        prev = off


@pytest.mark.parametrize("task", ["SafetyPointPush1Gymnasium-v0", "SafetyCarPush2Gymnasium-v0"])
def test_box_moves_only_on_contact_and_ends_at_push_distance(task):
    E = 64
    env = OracleVecEnvBP(NEW[task], E, 6)
    env.reset()
    ctr = np.zeros(E, np.uint32)
    moved_total = 0
    for t in range(300):
        box = env.st[9:11].copy()
        # half the steps drive at the box, so that contacts are frequent
        a = _push(env) if t % 2 else _random_actions(env, ctr)
        env.step(a)
        x, y = env.st[0], env.st[1]
        d_before = np.sqrt((box[0] - x) ** 2 + (box[1] - y) ** 2)     # the moved robot against the old box
        moved = np.any(env.st[9:11] != box, 0)
        # a box against the wall may be pushed into it and stay where it is
        free = np.all(np.abs(box) < P["ARENA"], 0)
        assert np.all(d_before[moved] < B["PUSH_D"]) and np.all(d_before[~moved & free] >= B["PUSH_D"])
        inside = np.all(np.abs(env.st[9:11]) < P["ARENA"], 0)
        d_after = np.sqrt((env.st[9] - x).astype(np.float64) ** 2 + (env.st[10] - y) ** 2)
        assert np.allclose(d_after[moved & inside], 0.3, rtol=0, atol=1e-6)
        moved_total += int(moved.sum())
    assert moved_total > E


@pytest.mark.parametrize("task", PUSHES)
def test_pushing_the_box_to_the_goal_scores(task):
    E = 32
    env = OracleVecEnvBP(NEW[task], E, 9)
    env.reset()
    for _ in range(1000):
        count = env.st[8].copy()
        _, rew, _, _, _ = env.step(_push(env))
        scored = env.st[8] > count
        assert np.all(rew[scored] > 0.9)
    assert (env.st[8] >= 1).mean() > 0.75, env.st[8]


@pytest.mark.parametrize("task", PUSHES)
def test_pillars_cost_only_at_level_2(task):
    E = 32
    env = OracleVecEnvBP(NEW[task], E, 4)
    env.reset()
    p0 = 11 + 2 * env.nhaz
    pillars = [(env.st[p0 + 2 * k].copy(), env.st[p0 + 1 + 2 * k].copy()) for k in range(env.nmov)]
    hazards = [(env.st[11 + 2 * k].copy(), env.st[12 + 2 * k].copy()) for k in range(env.nhaz)]
    probed = 0
    for i, (px, py) in enumerate(pillars):
        others = hazards + [p for j, p in enumerate(pillars) if j != i]
        clear = np.all([(px - ox) ** 2 + (py - oy) ** 2 > 0.9 ** 2 for ox, oy in others], 0)
        for off, want in ((0.0, 1), (0.35, 1), (0.45, 0)):
            env.st[0], env.st[1] = px + f32(off), py
            env.st[2], env.st[3], env.st[4], env.st[5] = 1, 0, 0, 0
            env.st[9], env.st[10] = 5, 5            # the box out of the way
            _, _, cost, _, _ = env.step(np.zeros((E, 2), f32))
            m = clear & (np.abs(env.st[0]) < P["ARENA"])
            assert np.all(cost[m] == (want if env.level == 2 else 0)), (off, cost[m])
            probed += int(m.sum())
    assert probed > 0


@pytest.mark.parametrize("task", sorted(NEW))
def test_random_play_has_nonzero_cost_rate(task):
    E = 64
    env = OracleVecEnvBP(NEW[task], E, 7)
    env.reset()
    ctr = np.zeros(E, np.uint32)
    cost = 0.0
    for _ in range(200):
        _, _, c, term, _ = env.step(_random_actions(env, ctr))
        assert not term.any()
        cost += float(c.sum())
    assert cost / (E * 200) > 0.0


def test_other_kinds_run_the_unchanged_twins():
    from oracle.envs_nav import OracleVecEnvNav
    for kind in list(range(9)) + list(range(16, 23)):
        a, b = OracleVecEnvNav(kind, 9, 5), OracleVecEnvBP(kind, 9, 5)
        assert np.array_equal(a.reset(), b.reset())
        for t in range(20):
            act = _scale(action_uniform(np.uint32(1), np.arange(9), np.full(9, t, np.uint32), a.A))
            for x, y in zip(a.step(act), b.step(act)):
                assert np.array_equal(x, y)
        assert np.array_equal(a.st, b.st)
