"""VectorEnvNormObs on the GPU against its float64 CPU restatement (tests/obs_norm_twin.py) over the bit-exact env
twins: random and train-mode collects on the inline and the resolve path, the generic path, the host path against
the device path, determinism, the successor identity of the ring, frozen statistics, the gym protocol, the agent's
checkpoint round trip and the launches of an unwrapped collect.

Bounds: raw dynamics (actions, rewards, costs, flags, env state) bit-exact; statistics within 1e-9 relative
(1e-12 absolute), count exact; every normalized observation within 1 float32 ulp of the float64 restatement."""
import os

import numpy as np
import pytest
import torch

from helpers import buffer_to_numpy, build_ppo
from obs_norm_twin import OracleNormObs
from oracle.envs_velocity import OracleVecEnvVel

pytestmark = pytest.mark.gpu

CHEETAH, HOPPER = "SafetyHalfCheetahVelocityGymnasium-v1", "SafetyHopperVelocityGymnasium-v1"
BUTTON = "SafetyPointButton1Gymnasium-v0"        # D = 76
TASKS = [CHEETAH, HOPPER, BUTTON]
RAW = ("act", "rew", "cost", "terminated", "truncated", "ptr", "len")


def _h(t):
    return t.detach().cpu().numpy()


def _twin(venv):
    return OracleVecEnvVel(venv.kind, venv.env_num, venv.seed_value)


def _ulps(a, b):
    """Max distance in float32 ulps between two float32 arrays of the same shape."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return int(np.abs(ia - ib).max()) if a.size else 0


def _assert_stats(rms, orms):
    assert rms.count == orms.count
    for got, want in ((rms.mean, orms.mean), (rms.var, orms.var)):
        np.testing.assert_allclose(got, want, rtol=1e-9, atol=1e-12)


def _wrapped(task, E, buffer_size, generic=False, update=True, hidden=(64, 64)):
    from fsrl_b200 import envs
    from fsrl_b200.data import FastCollector, VectorReplayBuffer
    from fsrl_b200.envs import VectorEnvNormObs
    if generic:         # a 3-hidden-layer torch actor: the generic path
        from test_env_step_gpu import _deep_policy
        torch.manual_seed(0)
        policy = _deep_policy(envs.make(task))
        venv = envs.DeviceVectorEnv(task, E, seed=12)
        buf = VectorReplayBuffer(buffer_size, E)
    else:
        policy, venv, buf, _ = build_ppo(task, hidden=hidden, n_env=E, buffer_size=buffer_size)
    norm = VectorEnvNormObs(venv, update_obs_rms=update)
    col = FastCollector(policy, norm, buf, exploration_noise=True)
    onorm = OracleNormObs(_twin(venv), update=update)
    if not generic:     # build_ppo's collector reset the env once unwrapped, the wrapped collector once more
        onorm.inner.reset()
    onorm.reset()
    return policy, venv, norm, buf, col, onorm


def _assert_successors(b, cap, E):
    """obs[t + 1] == obs_next[t] bit for bit wherever env e continued (ring not wrapped)."""
    D = b["obs"].shape[1]
    obs, nxt = (b[k].reshape(E, cap, D).view(np.int32) for k in ("obs", "obs_next"))
    ended = (b["terminated"] | b["truncated"]).reshape(E, cap)
    cont = (np.arange(cap - 1)[None, :] < b["len"].astype(np.int64)[:, None] - 1) & ~ended[:, :-1]
    bad = np.argwhere(cont & (obs[:, 1:] != nxt[:, :-1]).any(axis=2))
    assert len(bad) == 0, bad[:4].tolist()


@pytest.mark.parametrize("task", TASKS)
@pytest.mark.parametrize("E,n_episode", [(16, 16), (6, 14)])
def test_random_collect_matches_oracle(task, E, n_episode):
    _check_random_collect(task, E, n_episode)


def _check_random_collect(task, E, n_episode, hidden=(64, 64), twin=None, T=1000):
    """A random-mode collect of the wrapped device env against the twin wrapper (ring of T slots per env and
    round); ``twin`` may replace the twin's inner env (a recording proxy).  Returns the twin wrapper."""
    from oracle import collector as ocol
    rounds = n_episode // E + 2
    policy, venv, norm, buf, col, onorm = _wrapped(task, E, E * T * rounds, hidden=hidden)
    if twin is not None:
        onorm.inner = twin(onorm.inner)
    _assert_stats(norm.get_obs_rms(), onorm.rms)
    stats = col.collect(n_episode=n_episode, random=True)
    obuf = ocol.OracleBuffer(E * T * rounds, E, venv.D, venv.A)
    ctr = np.zeros(E, np.uint32)
    ostats = ocol.collect(onorm, None, n_episode, policy._act_seed, ctr, obuf, mode="random",
                          action_bound=policy.action_bound_method or "none")
    for k in ("n/ep", "n/st", "terminated", "truncated", "total_cost", "len"):
        assert stats[k] == ostats[k], k
    b = buffer_to_numpy(buf)
    for k in RAW:
        want = getattr(obuf, k) if hasattr(obuf, k) else None
        assert np.array_equal(b[k], want), k
    for k in ("obs", "obs_next"):
        assert _ulps(b[k], getattr(obuf, k)) <= 1, k
    _assert_stats(norm.get_obs_rms(), onorm.rms)
    assert _ulps(_h(venv.obs_cur), onorm.observe()) <= 1
    assert np.array_equal(_h(venv.env_state), onorm.inner.st)
    assert np.array_equal(_h(venv.act_ctr).astype(np.uint32), ctr)
    _assert_successors(b, buf.cap, E)
    if task == HOPPER:
        assert b["terminated"].any()
    return onorm


def _replay_inline(policy, norm_env, b, cap, E, onorm):
    """Replay an inline collect (every env one episode from slot 0) through the twin wrapper vector step by vector
    step with the ring's actions: at step t the envs whose episode is longer than t step, in ascending id."""
    L = b["len"].astype(int)
    for t in range(int(L.max())):
        ids = np.nonzero(L > t)[0]
        p = ids * cap + t
        assert _ulps(b["obs"][p], onorm.observe(ids)) <= 1, t
        a = np.asarray(policy.map_action(b["act"][p]), np.float32)
        obs, rew, cost, term, trunc = onorm.step(a, ids)
        assert _ulps(b["obs_next"][p], obs) <= 1, t
        assert np.array_equal(b["rew"][p], rew) and np.array_equal(b["cost"][p], cost), t
        assert np.array_equal(b["terminated"][p], term), t
    onorm.reset()


@pytest.mark.parametrize("task", TASKS)
@pytest.mark.parametrize("generic", [False, True], ids=["fused", "generic"])
def test_train_collect_replays_through_twin(task, generic):
    E, T = 8, 1000
    policy, venv, norm, buf, col, onorm = _wrapped(task, E, E * T * 2, generic=generic)
    assert col.fused is not generic
    policy.train()
    stats = col.collect(n_episode=E)
    assert stats["n/ep"] == E
    b = buffer_to_numpy(buf)
    _replay_inline(policy, norm, b, buf.cap, E, onorm)
    _assert_stats(norm.get_obs_rms(), onorm.rms)
    assert np.array_equal(_h(venv.env_state), onorm.inner.st)
    _assert_successors(b, buf.cap, E)


def _host_vs_device(task, E, n_episode, mode, hidden=(64, 64)):
    from fsrl_b200.data import FastCollector, VectorReplayBuffer
    from fsrl_b200.envs import DeviceVectorEnv, VectorEnvNormObs
    from host_twin import host_twin
    policy, _, _, _ = build_ppo(task, hidden=hidden, n_env=E)
    getattr(policy, mode)()
    out = []
    for venv in (DeviceVectorEnv(task, E, seed=7), host_twin(task, E, 7)):
        norm = VectorEnvNormObs(venv)
        buf = VectorReplayBuffer(E * 1000 * (n_episode // E + 2), E)
        col = FastCollector(policy, norm, buf, exploration_noise=True)
        st = col.collect(n_episode=n_episode)
        st2 = col.collect(n_episode=n_episode)
        rms = norm.get_obs_rms()
        out.append((buffer_to_numpy(buf), rms.mean, rms.var, rms.count, _h(venv.act_ctr), st, st2, buf.cap))
    return out


@pytest.mark.parametrize("task", [HOPPER, BUTTON])
@pytest.mark.parametrize("E,n_episode", [(8, 8), (5, 13)])
def test_host_path_matches_device_path_bitwise(task, E, n_episode):
    _check_host_vs_device(task, E, n_episode)


def _check_host_vs_device(task, E, n_episode, hidden=(64, 64)):
    (bd, md, vd, cd, ad, sd, sd2, cap), (bh, mh, vh, ch, ah, sh, sh2, _) = _host_vs_device(task, E, n_episode, "train",
                                                                                          hidden)
    for k in bd:
        assert np.array_equal(bd[k], bh[k]), k
    assert md.tobytes() == mh.tobytes() and vd.tobytes() == vh.tobytes() and cd == ch
    assert np.array_equal(ad, ah)
    for k in ("n/ep", "n/st", "total_cost", "terminated", "truncated"):
        assert sd[k] == sh[k] and sd2[k] == sh2[k], k
    _assert_successors(bd, cap, E) if n_episode <= E else None


def test_two_runs_are_bit_identical():
    a = _host_vs_device(HOPPER, 5, 13, "train")[0]
    b = _host_vs_device(HOPPER, 5, 13, "train")[0]
    for k in a[0]:
        assert np.array_equal(a[0][k], b[0][k]), k
    assert a[1].tobytes() == b[1].tobytes() and a[2].tobytes() == b[2].tobytes() and a[3] == b[3]


def test_resolve_path_successor_identity():
    """On the resolve path restarted envs continue in the ring: their first obs is the reset row normalized after
    the second update, every other successor repeats obs_next bit for bit."""
    E, n_episode = 6, 14
    policy, venv, norm, buf, col, onorm = _wrapped(HOPPER, E, E * 1000 * 4)
    policy.train()
    col.collect(n_episode=n_episode)
    _assert_successors(buffer_to_numpy(buf), buf.cap, E)


def test_frozen_statistics_stay_bit_unchanged():
    from fsrl_b200.data import FastCollector
    from fsrl_b200.envs import DeviceVectorEnv, VectorEnvNormObs
    policy, venv, norm, buf, col, _ = _wrapped(CHEETAH, 8, 8 * 1000 * 2)
    col.collect(n_episode=8, random=True)
    rms = norm.get_obs_rms()
    before = (rms.mean.tobytes(), rms.var.tobytes(), rms.count)
    test = VectorEnvNormObs(DeviceVectorEnv(CHEETAH, 4, seed=3), update_obs_rms=False)
    test.set_obs_rms(rms)
    FastCollector(policy, test).collect(n_episode=6)
    test.reset([1, 2])
    test.step(torch.zeros((2, venv.A), device="cuda"), [2, 0])
    assert (rms.mean.tobytes(), rms.var.tobytes(), rms.count) == before
    # a normalizing wrapper passed to evaluate only normalizes, even with update_obs_rms=True
    from fsrl_b200.agent import PPOLagAgent
    from fsrl_b200 import envs
    agent = PPOLagAgent(envs.make(CHEETAH), hidden_sizes=(64, 64))
    live = VectorEnvNormObs(DeviceVectorEnv(CHEETAH, 2, seed=4))
    live.reset()
    snap = live.get_obs_rms().state_dict()
    agent.evaluate(live, eval_episodes=2)
    after = live.get_obs_rms().state_dict()
    assert snap["mean"].tobytes() == after["mean"].tobytes() and snap["count"] == after["count"]
    assert live.update_obs_rms


@pytest.mark.parametrize("task", [HOPPER, BUTTON])
@pytest.mark.parametrize("host", [False, True], ids=["device", "host"])
def test_gym_protocol_matches_oracle(task, host):
    from fsrl_b200.envs import DeviceVectorEnv, VectorEnvNormObs
    from host_twin import host_twin
    from oracle.philox import action_uniform
    E = 7
    venv = host_twin(task, E, 5) if host else DeviceVectorEnv(task, E, seed=5)
    norm = VectorEnvNormObs(venv)
    onorm = OracleNormObs(OracleVecEnvVel(DeviceVectorEnv(task, 1).kind, E, 5))
    to_np = (lambda x: np.asarray(x)) if host else _h
    assert _ulps(to_np(norm.reset()[0]), onorm.reset()) <= 1
    for i, ids in enumerate(([0, 1, 2, 3, 4, 5, 6], [5, 2, 0], [6], [3, 1, 4, 0, 2])):
        ids = np.asarray(ids)
        a = action_uniform(11, ids, np.full(len(ids), i, np.uint32), venv.A)
        obs, rew, term, trunc, info = norm.step(torch.as_tensor(a, device="cuda") if not host else a, ids)
        oo, orew, ocost, oterm, otrunc = onorm.step(a, ids)
        assert _ulps(to_np(obs), oo) <= 1, i
        assert np.array_equal(to_np(rew).astype(np.float32), orew.astype(np.float32)), i
        if i == 1:
            r = norm.reset([4, 1])[0]
            assert _ulps(to_np(r), onorm.reset([4, 1])) <= 1
    _assert_stats(norm.get_obs_rms(), onorm.rms)


def test_unwrapped_collect_launches_unchanged():
    """An unwrapped inline collect is still one begin, one step and one resolve launch and one reset."""
    from fsrl_b200 import _lib
    policy, venv, buf, col = build_ppo(CHEETAH, n_env=16, buffer_size=16 * 1000)
    l0 = int(_lib.lib.fsrl_launch_count())
    col.collect(n_episode=16)
    assert int(_lib.lib.fsrl_launch_count()) - l0 == 4


def test_agent_checkpoint_round_trip(tmp_path):
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples"))
    import train_norm_obs
    from fsrl_b200.agent import PPOLagAgent
    from fsrl_b200 import envs
    from fsrl_b200.envs import DeviceVectorEnv, VectorEnvNormObs
    from fsrl_b200.utils.logger import BaseLogger
    task = CHEETAH
    logger = BaseLogger(str(tmp_path), log_txt=False, name="rt")
    agent = PPOLagAgent(envs.make(task), logger, hidden_sizes=(64, 64), seed=3)
    train = VectorEnvNormObs(DeviceVectorEnv(task, 8, seed=1))
    agent.learn(train, DeviceVectorEnv(task, 2, seed=2), epoch=2, episode_per_collect=8, step_per_epoch=16000,
                testing_num=2, save_interval=1, verbose=False, show_progress=False)
    ckpt = torch.load(os.path.join(logger.log_dir, "checkpoint", "model.pt"), weights_only=False)
    assert ckpt["obs_rms"]["count"] == train.get_obs_rms().count > 0
    assert ckpt["obs_rms"]["mean"].tobytes() == train.get_obs_rms().mean.tobytes()

    def ev(rms_state, model):
        e = VectorEnvNormObs(DeviceVectorEnv(task, 2, seed=9), update_obs_rms=False)
        e.get_obs_rms().load_state_dict(rms_state)
        return agent.evaluate(e, model, eval_episodes=2)

    in_memory = ev(train.get_obs_rms().state_dict(), None)
    fresh = PPOLagAgent(envs.make(task), hidden_sizes=(64, 64), seed=5)
    e = VectorEnvNormObs(DeviceVectorEnv(task, 2, seed=9), update_obs_rms=False)
    e.get_obs_rms().load_state_dict(ckpt["obs_rms"])
    assert fresh.evaluate(e, ckpt["model"], eval_episodes=2) == in_memory
    rew, length, cost = train_norm_obs.main(["--epoch", "1", "--step_per_epoch", "4000", "--training_num", "4",
                                             "--logdir", str(tmp_path / "ex")])
    assert np.isfinite(rew)


def test_collector_refusals_on_gpu():
    from fsrl_b200.data import FastCollector, TrajectoryBuffer
    from fsrl_b200.envs import VectorEnvNormObs
    policy, venv, buf, _ = build_ppo(CHEETAH, n_env=4, buffer_size=4 * 1000)
    with pytest.raises(NotImplementedError, match="normalized"):
        FastCollector(policy, VectorEnvNormObs(venv), buf, traj_buffer=TrajectoryBuffer(1000))
    policy._dp = object()
    with pytest.raises(NotImplementedError, match="data parallelism"):
        FastCollector(policy, VectorEnvNormObs(venv), buf)
