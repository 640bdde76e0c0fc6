"""The Safety-Gymnasium velocity tasks (HalfCheetah, Hopper, Swimmer, Walker2d, Ant) on the CPU: the registry, the C
ABI and the env twin (oracle/envs_velocity.py) agree on the dimensions, and the twin's models behave as
csrc/envs.cuh documents them.  The model checks catch a twin and kernel that agree with each other but are both
wrong: no speed without a gait, a gait that is fast enough to cost and one slow enough not to, a balance that
random play loses and joint feedback keeps."""
import numpy as np
import pytest

from oracle.envs_button_push import OracleVecEnvBP
from oracle.envs_velocity import (ANT, DIMS, HALF_CHEETAH, HOPPER, NJ, SWIMMER, WALKER2D, R, OracleVecEnvVel)
from oracle.philox import action_uniform
from test_nav_envs_host import _scale

NEW = {"SafetyHalfCheetahVelocityGymnasium-v1": HALF_CHEETAH, "SafetyHopperVelocityGymnasium-v1": HOPPER,
       "SafetySwimmerVelocityGymnasium-v1": SWIMMER, "SafetyWalker2dVelocityGymnasium-v1": WALKER2D,
       "SafetyAntVelocityGymnasium-v1": ANT}
BALANCE = (HOPPER, WALKER2D)
f32 = np.float32
E = 64
W = 3.0                    # gait frequency, rad/s: near the joints' resonance


def _velocity(kind, obs):
    """(vx, the speed the cost compares) from an observation."""
    N = NJ[kind]
    if kind == SWIMMER:
        return obs[:, 3], obs[:, 3]
    if kind == ANT:
        vx, vy = obs[:, 13], obs[:, 14]
        return vx, np.sqrt(vx * vx + vy * vy)
    return obs[:, 2 + N], obs[:, 2 + N]


def _balance(env):
    """Pitch feedback on the thighs (joint 0, and 3 on Walker2d): a = 0.8 th + 0.7 th'."""
    return np.clip(f32(0.8) * env.st[2] + f32(0.7) * env.st[3], -1, 1).astype(f32)


def _gait(env, t, amp):
    """The open-loop gait: sinusoids of amplitude `amp` at W rad/s, each joint of a pair a quarter period behind
    the one before it, so that every pair sweeps the same positive area.
      HalfCheetah  legs (0, 1, 2) and (3, 4, 5), the back leg half a period behind the front one
      Hopper       joints 1, 2; the thigh (0) balances
      Walker2d     joints 1, 2 and 4, 5 half a period apart; the thighs (0, 3) balance
      Swimmer      joints 0, 1
      Ant          hip j at phase j quarter-turns, ankle j + 4 a quarter period behind it: the ankle angles sum
                   to 0, so the height holds"""
    kind, n = env.kind, env.E
    ph = W * 0.05 * t
    s = lambda off: np.full(n, amp * np.sin(ph - off), f32)
    q = np.pi / 2
    if kind == HALF_CHEETAH:
        return np.stack([s(0), s(q), s(2 * q), s(2 * q), s(3 * q), s(4 * q)], 1).astype(f32)
    if kind == HOPPER:
        return np.stack([_balance(env), s(0), s(q)], 1).astype(f32)
    if kind == WALKER2D:
        b = _balance(env)
        return np.stack([b, s(0), s(q), b, s(2 * q), s(3 * q)], 1).astype(f32)
    if kind == SWIMMER:
        return np.stack([s(0), s(q)], 1).astype(f32)
    return np.stack([s(j * q) for j in range(4)] + [s(j * q + q) for j in range(4)], 1).astype(f32)


def _run(kind, policy, steps=1000, seed=3):
    """Step E envs of `kind` without resets; returns per-step arrays (E, steps) of reward, cost, terminated, vx."""
    env = OracleVecEnvVel(kind, E, seed)
    env.reset()
    out = {k: np.zeros((E, steps), f32) for k in ("rew", "cost", "term", "vx")}
    for t in range(steps):
        obs, rew, cost, term, _ = env.step(policy(env, t))
        out["rew"][:, t], out["cost"][:, t], out["term"][:, t] = rew, cost, term
        out["vx"][:, t] = _velocity(kind, obs)[0]
    return out


def _random(seed=3):
    ctr = np.zeros(E, np.uint32)

    def policy(env, t):
        a = _scale(action_uniform(np.uint32(seed), np.arange(env.E), ctr, env.A))
        ctr[:] += np.uint32(1)
        return a
    return policy


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
    assert D <= 40 and A <= 8 and S <= 32 and T == 1000      # inside the persistent PPO launch's gate
    env = OracleVecEnvVel(kind, 3, 1)
    assert env.reset().shape == (3, D) and env.st.shape == (S, 3)


def test_the_next_kind_is_rejected():
    from fsrl_b200 import envs
    with pytest.raises(Exception, match="unknown env kind"):
        envs.env_dims(38)


def test_humanoid_stays_unknown():
    from fsrl_b200 import envs
    with pytest.raises(KeyError, match="unknown task"):
        envs.make("SafetyHumanoidVelocityGymnasium-v1")


@pytest.mark.parametrize("task", sorted(NEW))
def test_reward_and_cost_follow_the_velocity(task):
    """reward = vx + healthy - w_ctrl |a|^2 and cost = [speed > threshold], recomputed from the step's observation
    and actions, over random play and over the fast gait (where the cost fires)."""
    kind = NEW[task]
    p = R[kind]
    for policy in (_random(), lambda env, t: _gait(env, t, 1.0)):
        env = OracleVecEnvVel(kind, E, 5)
        env.reset()
        seen_cost = 0.0
        for t in range(300):
            a = policy(env, t)
            obs, rew, cost, _, _ = env.step(a)
            vx, speed = _velocity(kind, obs)
            ctrl = np.zeros(E, f32)
            for j in range(env.A):
                ctrl = ctrl + a[:, j] * a[:, j]
            assert np.array_equal(rew, (vx + p["HEALTHY"]) - p["WCTRL"] * ctrl), t
            assert np.array_equal(cost, (speed > p["VCOST"]).astype(f32)), t
            seen_cost += cost.sum()
    assert seen_cost > 0


@pytest.mark.parametrize("task", sorted(NEW))
@pytest.mark.parametrize("const", [0.0, 0.6, -1.0, "mixed"])
def test_constant_actions_make_no_speed(task, const):
    kind = NEW[task]
    A = DIMS[kind][1]
    a = (np.full((E, A), const, f32) if const != "mixed" else
         np.random.default_rng(2).uniform(-1, 1, (E, A)).astype(f32))
    out = _run(kind, lambda env, t: a)
    assert np.abs(out["vx"][:, 500:]).mean() < 1e-3 * R[kind]["VMAX"]


@pytest.mark.parametrize("task", sorted(NEW))
def test_fast_gait_costs_and_slow_gait_does_not(task):
    kind = NEW[task]
    p = R[kind]
    fast = _run(kind, lambda env, t: _gait(env, t, 1.0))
    slow = _run(kind, lambda env, t: _gait(env, t, 0.5))
    for out in (fast, slow):
        assert not out["term"].any()                    # the gait (and on Hopper / Walker2d its balance) holds up
    assert fast["cost"][:, 200:].mean() > 0.5
    assert not slow["cost"].any()
    assert slow["rew"][:, 200:].mean() > p["HEALTHY"] + 0.2 * p["VCOST"]     # standing still earns HEALTHY
    assert fast["vx"][:, 200:].mean() > p["VCOST"] > slow["vx"][:, 200:].mean() > 0


@pytest.mark.parametrize("task", [t for t, k in NEW.items() if k in BALANCE])
def test_balance_keeps_every_reset_alive(task):
    kind = NEW[task]
    A = DIMS[kind][1]

    def policy(env, t):
        a = np.zeros((env.E, A), f32)
        a[:, 0] = _balance(env)
        if kind == WALKER2D:
            a[:, 3] = a[:, 0]
        return a
    for seed in (3, 4):
        out = _run(kind, policy, seed=seed)
        assert not out["term"].any()


@pytest.mark.parametrize("task", [t for t, k in NEW.items() if k in BALANCE])
def test_random_play_topples_most_episodes(task):
    kind = NEW[task]
    out = _run(kind, _random(), steps=DIMS[kind][3])
    ended = out["term"].any(1)
    assert ended.mean() > 0.5, ended.mean()
    # without feedback the robot falls too: holding the joints still is not a balance
    still = _run(kind, lambda env, t: np.zeros((env.E, env.A), f32))
    assert still["term"].any(1).all()


def test_ant_jumps_out_of_bounds():
    """Pushing every ankle to +1 lifts the torso past z = 1 and terminates; pulling them to -1 drops it below 0.2."""
    for sign in (1.0, -1.0):
        a = np.zeros((E, 8), f32)
        a[:, 4:] = sign
        out = _run(ANT, lambda env, t: a, steps=60)
        first = out["term"].argmax(1)
        assert out["term"].any(1).all() and first.max() < 40, sign


@pytest.mark.parametrize("task", ["SafetyHalfCheetahVelocityGymnasium-v1", "SafetySwimmerVelocityGymnasium-v1"])
def test_random_play_never_terminates(task):
    out = _run(NEW[task], _random())
    assert not out["term"].any()


def test_ant_quaternion_is_a_unit_rotation():
    env = OracleVecEnvVel(ANT, E, 8)
    env.reset()
    pol = _random()
    for t in range(200):
        obs, _, _, _, _ = env.step(pol(env, t))
        n = (obs[:, 1:5].astype(np.float64) ** 2).sum(1)
        assert np.abs(n - 1).max() < 1e-5, t


@pytest.mark.parametrize("kind", list(range(0, 9)) + list(range(16, 23)) + list(range(24, 32)))
def test_other_kinds_run_the_unchanged_twin(kind):
    n = 9
    a, b = OracleVecEnvBP(kind, n, 5), OracleVecEnvVel(kind, n, 5)
    assert np.array_equal(a.reset(), b.reset())
    ctr = np.zeros(n, np.uint32)
    for t in range(30):
        act = _scale(action_uniform(np.uint32(1), np.arange(n), ctr, a.A))
        ctr += np.uint32(1)
        ids = np.arange(0, n, 2) if t % 2 else None
        for x, y in zip(a.step(act if ids is None else act[ids], ids), b.step(act if ids is None else act[ids], ids)):
            assert np.array_equal(x, y), (kind, t)
        if t == 10:
            assert np.array_equal(a.reset([1, 4]), b.reset([1, 4]))
    assert np.array_equal(a.st, b.st) and np.array_equal(a.observe(), b.observe())
