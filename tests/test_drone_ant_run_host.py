"""SafetyAntRun-v0, SafetyDroneCircle-v0 and SafetyDroneRun-v0 on the CPU: the registry and the C ABI
agree with the env twin (oracle/envs_flight.py) on the dimensions, and the twin's models have the
three properties their constants were chosen for (csrc/envs.cuh):
  1. holding the hover command (a = 0 on every rotor) keeps every Drone reset alive for T steps;
  2. uniform random actions end a clear majority of Drone episodes by termination before T;
  3. a uniform random policy sees a nonzero cost rate on every new task."""
import numpy as np
import pytest

from oracle.envs_flight import DIMS, OracleVecEnvExt
from oracle.philox import action_uniform

NEW = {"SafetyAntRun-v0": 6, "SafetyDroneCircle-v0": 7, "SafetyDroneRun-v0": 8}
DRONES = ("SafetyDroneCircle-v0", "SafetyDroneRun-v0")
E = 512


def _scale(u):
    # map_action with scaling onto [-1, 1] (rollout.cu), as the device applies it
    return (np.float32(-1) + (np.float32(2) * (u + np.float32(1))) / np.float32(2)).astype(np.float32)


def _random_play(kind, seed=7, act_seed=3):
    """One episode per env under uniform random actions; returns (terminated flag, episode length,
    summed cost, steps) per env."""
    env = OracleVecEnvExt(kind, E, seed)
    env.reset()
    A, T = env.A, env.T
    ids = np.arange(E)
    ctr = np.zeros(E, np.uint32)
    live = np.ones(E, bool)
    termed = np.zeros(E, bool)
    length = np.zeros(E, np.int64)
    cost = np.zeros(E)
    for t in range(T):
        a = _scale(action_uniform(np.uint32(act_seed), ids, ctr, A))
        ctr += np.uint32(1)
        _, _, c, term, trunc = env.step(a)
        cost[live] += c[live]
        length[live] += 1
        termed |= term & live
        live &= ~(term | trunc)
    return termed, length, cost


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
    # inside the persistent PPO launch's obs-width gate, the MLP input limit and the env limits
    assert D <= 40 and S <= 32 and A <= 8


def test_unknown_kind_is_rejected():
    from fsrl_b200 import envs
    with pytest.raises(Exception, match="unknown env kind"):   # raised by the library's kind check
        envs.env_dims(9)


@pytest.mark.parametrize("task", DRONES)
def test_hover_survives_the_horizon(task):
    env = OracleVecEnvExt(NEW[task], E, 11)
    obs = env.reset()
    motors = slice(13, 17) if task == "SafetyDroneCircle-v0" else slice(12, 16)
    assert np.all(obs[:, motors] == 0)          # motors start at hover thrust
    for _ in range(env.T):
        _, _, _, term, trunc = env.step(np.zeros((E, env.A), np.float32))
        assert not term.any()
    assert trunc.all()
    assert np.all(env.st[2] > 0.5)              # altitude stays well above the ground


@pytest.mark.parametrize("task", DRONES)
def test_random_play_terminates_most_episodes(task):
    termed, length, _ = _random_play(NEW[task])
    assert termed.mean() > 0.6, termed.mean()
    assert np.median(length[termed]) < DIMS[NEW[task]][3] // 2


@pytest.mark.parametrize("task", sorted(NEW))
def test_random_play_has_nonzero_cost_rate(task):
    termed, length, cost = _random_play(NEW[task])
    assert cost.sum() / length.sum() > 0.0
    if task == "SafetyAntRun-v0":
        assert not termed.any()                 # Ant-Run is truncation only


def test_existing_kinds_run_the_unchanged_twin():
    from oracle.envs import OracleVecEnv
    for kind in range(6):
        a, b = OracleVecEnv(kind, 9, 5), OracleVecEnvExt(kind, 9, 5)
        assert np.array_equal(a.reset(), b.reset())
        act = _scale(action_uniform(np.uint32(1), np.arange(9), np.zeros(9, np.uint32), a.A))
        for x, y in zip(a.step(act), b.step(act)):
            assert np.array_equal(x, y)
