"""Offline datasets from host-stepped envs (FastCollector's host path with ``traj_buffer=``, BasicCollector over a
gymnasium-style env, ``fsrl_traj_copy_host``).

The CPU twins are bit-exact models of the device envs, so a harvest over a HostVectorEnv of twins must keep the same
trajectories, in the same arena slots, with the same bits as the device harvest over the DeviceVectorEnv of the same
task and seed.  Independently of the device path, the harvested trajectories must be what the envs saw: a recorder
around every env logs each transition, and the episodes the oracle TrajectoryBuffer keeps from that stream are the
dataset.  User envs cover what no twin does: an unknown horizon, a ring shorter than an episode and float64 rewards
that float32 cannot hold."""
import os
import random

import numpy as np
import pytest
import torch

from helpers import build_ppo
from host_twin import TwinEnv, twin, twin_fns
from oracle.trajbuf import OracleTrajBuf

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ("observations", "next_observations", "actions", "rewards", "costs", "terminals", "timeouts")
CAR_CIRCLE, DRONE_RUN, HOPPER = "SafetyCarCircle-v0", "SafetyDroneRun-v0", "SafetyHopperVelocityGymnasium-v1"
POINT_GOAL1 = "SafetyPointGoal1Gymnasium-v0"


def _T(task):
    from fsrl_b200 import envs
    return envs.make(task).spec.max_episode_steps


def _assert_stats_equal(sd, sh):
    for a, b in zip(sd, sh):
        for k in ("n/ep", "n/st", "terminated", "truncated"):
            assert a[k] == b[k], k
        for k in ("rew", "len", "cost", "total_cost"):
            assert b[k] == pytest.approx(a[k], rel=1e-12, abs=1e-12), k


def _assert_same_buffer(tb_d, tb_h):
    assert [m.tolist() for m in tb_h.metrics] == [m.tolist() for m in tb_d.metrics]
    assert tb_h._index.slots == tb_d._index.slots and tb_h._index.lens == tb_d._index.lens
    assert len(tb_h) == len(tb_d)
    if len(tb_d.buffer):
        assert tb_h._arena.stride == tb_d._arena.stride
        gd, gh = tb_d.get_all(), tb_h.get_all()
        for k in KEYS:
            assert torch.equal(gd[k], gh[k]), k


def _run(policy, venv, n_episode, cap, collects, rng_seed, tb_kw):
    from fsrl_b200.data import FastCollector, TrajectoryBuffer, VectorReplayBuffer
    E = len(venv)
    random.seed(rng_seed)
    np.random.seed(rng_seed)
    tb = TrajectoryBuffer(**tb_kw)
    buf = VectorReplayBuffer(E * cap, E) if cap else None
    col = FastCollector(policy, venv, buf, exploration_noise=True, traj_buffer=tb)
    stats = [col.collect(n_episode=n_episode) for _ in range(collects)]
    torch.cuda.synchronize()
    return tb, stats, col


# task, E, n_episode, ring ("private" or slots beyond the device path's least ring), keep rule
CASES = [
    (CAR_CIRCLE, 6, 6, "private", "all"),          # one episode per env
    (CAR_CIRCLE, 6, 4, 0, "grid"),                 # n < E on a user ring of exactly T: the second collect wraps
    (DRONE_RUN, 6, 13, "private", "all"),          # terminations, surplus retire, several episodes per env
    (DRONE_RUN, 5, 12, 7, "replace"),              # a user ring that wraps inside the collects
    (DRONE_RUN, 4, 4, 0, "window"),
    (HOPPER, 4, 9, 5, "grid"),                     # unhealthy terminations
    (POINT_GOAL1, 3, 3, "private", "replace"),     # a truncating Safety-Gymnasium navigation task
    (POINT_GOAL1, 3, 5, 3, "window"),
]


def _keep_rule(kind, pilot=None):
    if kind == "all":
        return {}
    if kind == "grid":
        return dict(max_trajectory=4, filter_interval=1.5)
    if kind == "replace":
        return dict(max_trajectory=3, use_grid_filter=False)
    rets = np.array([m[0] for m in pilot.metrics])
    costs = np.array([m[1] for m in pilot.metrics])
    return dict(rmin=float(np.quantile(rets, 0.2)), rmax=float(np.quantile(rets, 0.8)), cmin=float(costs.min()),
                cmax=float(costs.max()))


@pytest.mark.parametrize("task,E,n_episode,ring,keep", CASES)
def test_host_harvest_equals_device_harvest(task, E, n_episode, ring, keep):
    from fsrl_b200.envs import DeviceVectorEnv, HostVectorEnv
    seed, collects = 21, 3
    T = _T(task)
    if ring == "private":
        cap = 0
    else:                         # the device path needs T slots (n <= E) or T + 64; both paths get the same ring
        cap = (T if n_episode <= E else T + 64) + ring
    policy = build_ppo(task, n_env=1, seed=5)[0]
    policy.train()
    pilot = None
    if keep == "window":
        # the first collect's episodes, unfiltered: the window keeps the middle of their returns
        pilot = _run(policy, DeviceVectorEnv(task, E, seed=seed), n_episode, cap, 1, 0, {})[0]
    tb_kw = _keep_rule(keep, pilot)
    tb_d, sd, _ = _run(policy, DeviceVectorEnv(task, E, seed=seed), n_episode, cap, collects, 3, tb_kw)
    tb_h, sh, col = _run(policy, HostVectorEnv(twin_fns(task, E, seed)), n_episode, cap, collects, 3, tb_kw)
    assert col.host and (cap or col.buffer.cap == T)
    _assert_stats_equal(sd, sh)
    _assert_same_buffer(tb_d, tb_h)
    assert len(tb_d.buffer) > 0
    if keep == "all":
        assert len(tb_h.buffer) == sum(s["n/ep"] for s in sh)
    if (task, ring) == (CAR_CIRCLE, 0):         # three collects of T steps each through a ring of T slots
        assert (col.buffer.len.cpu().numpy()[:n_episode] == cap).all()     # (the envs past n_episode never step)


def test_collect_checks_the_ring_against_the_horizon():
    from fsrl_b200.data import FastCollector, TrajectoryBuffer, VectorReplayBuffer
    from fsrl_b200.envs import HostVectorEnv
    task, E = DRONE_RUN, 3
    T = _T(task)
    policy = build_ppo(task, n_env=1, seed=5)[0]
    col = FastCollector(policy, HostVectorEnv(twin_fns(task, E, 2)), VectorReplayBuffer(E * (T - 1), E),
                        traj_buffer=TrajectoryBuffer())
    with pytest.raises(ValueError, match=f"at least {T} slots"):
        col.collect(n_episode=E)
    assert col.min_ring_capacity() == T


# ---- the dataset is what the envs saw ---------------------------------------------------------------------------
class Recorder:
    """A gymnasium env that logs every transition (obs, act, rew, cost, terminated, truncated, obs_next) it makes;
    each finished episode goes to the shared ``log`` as it ends.  A reset drops the open episode."""

    def __init__(self, env, log):
        self.env, self.log = env, log
        self.observation_space, self.action_space = env.observation_space, env.action_space
        self.spec = getattr(env, "spec", None)
        self.cur = []

    def reset(self, **kw):
        out = self.env.reset(**kw)
        o = out[0] if isinstance(out, tuple) else out
        self.obs, self.cur = np.asarray(o, np.float32).copy(), []
        return out

    def step(self, a):
        a = np.array(a, copy=True)
        o, r, te, tr, info = self.env.step(a)
        on = np.asarray(o, np.float32).copy()
        self.cur.append((self.obs, a, float(r), float(info.get("cost", 0.0)), bool(te), bool(tr) and not te, on))
        self.obs = on
        if te or tr:
            self.log.append(self.cur)
            self.cur = []
        return o, r, te, tr, info


def _oracle(log, rng_seed, **kw):
    """The recorded episodes, in the order they ended, through the oracle's keep rules."""
    random.seed(rng_seed)
    np.random.seed(rng_seed)
    ob = OracleTrajBuf(**kw)
    for ep in log:
        ret = cost = 0.0
        for t in ep:
            ret += t[2]
            cost += t[3]
        ob.add(dict(observations=np.stack([t[0] for t in ep]), next_observations=np.stack([t[6] for t in ep]),
                    actions=np.stack([t[1] for t in ep]).astype(np.float32),
                    rewards=np.array([t[2] for t in ep], np.float32), costs=np.array([t[3] for t in ep], np.float32),
                    terminals=np.array([t[4] for t in ep]), timeouts=np.array([t[5] for t in ep])), ret, cost)
    return ob


def _assert_is_oracle(tb, ob):
    assert [m.tolist() for m in tb.metrics] == [m.tolist() for m in ob.metrics]
    assert len(tb.buffer) == len(ob.trajs) > 0
    got, want = tb.get_all(), ob.concat()
    for k in KEYS:
        g = got[k].cpu().numpy()
        assert g.dtype == want[k].dtype, (k, g.dtype, want[k].dtype)
        assert np.array_equal(g, want[k]), k


@pytest.mark.parametrize("task,E,n_episode,tb_kw", [
    (DRONE_RUN, 5, 12, dict(max_trajectory=6, filter_interval=1.5)),
    (CAR_CIRCLE, 4, 4, dict(max_trajectory=3, use_grid_filter=False)),
    (HOPPER, 3, 7, {}),
])
def test_dataset_is_what_the_envs_saw(task, E, n_episode, tb_kw):
    from fsrl_b200.data import FastCollector, TrajectoryBuffer
    from fsrl_b200.envs import HostVectorEnv
    log = []
    venv = HostVectorEnv([lambda f=f: Recorder(f(), log) for f in twin_fns(task, E, 8)])
    policy = build_ppo(task, n_env=1, seed=6)[0]
    policy.train()
    random.seed(4)
    np.random.seed(4)
    tb = TrajectoryBuffer(**tb_kw)
    col = FastCollector(policy, venv, exploration_noise=True, traj_buffer=tb)
    for _ in range(2):
        col.collect(n_episode=n_episode)
    torch.cuda.synchronize()
    _assert_is_oracle(tb, _oracle(log, 4, **tb_kw))


# ---- BasicCollector over one env -----------------------------------------------------------------------------
class Gym4:
    """A gymnasium env seen through gym's 4-tuple step (done, TimeLimit.truncated in info)."""

    def __init__(self, env):
        self.env = env
        self.observation_space, self.action_space, self.spec = env.observation_space, env.action_space, env.spec

    def reset(self, **kw):
        return self.env.reset(**kw)[0]

    def step(self, a):
        o, r, te, tr, info = self.env.step(a)
        return o, r, te or tr, dict(info, **{"TimeLimit.truncated": tr and not te})


@pytest.mark.parametrize("task,api", [(DRONE_RUN, 5), (DRONE_RUN, 4), (HOPPER, 5)])
def test_basic_collector_over_one_host_env(task, api):
    from fsrl_b200.data import BasicCollector, TrajectoryBuffer
    from fsrl_b200.envs import DeviceVectorEnv, HostVectorEnv
    seed, n = 13, 5
    out = []
    for host in (False, True):
        policy = build_ppo(task, n_env=1, seed=7)[0]
        policy.train()
        if host:
            env = TwinEnv(twin(task, 1, seed), 0, task)
            env = Gym4(env) if api == 4 else env
        else:
            env = DeviceVectorEnv(task, 1, seed=seed)
        tb = TrajectoryBuffer()
        bc = BasicCollector(policy, env, traj_buffer=tb, exploration_noise=True)
        assert isinstance(bc.env, HostVectorEnv) == host
        stats = [bc.collect(n_episode=n), bc.collect(n_episode=2)]
        torch.cuda.synchronize()
        out.append((tb, stats, bc))
    (tb_d, sd, _), (tb_h, sh, bc_h) = out
    assert bc_h.buffer.cap == _T(task)
    _assert_stats_equal(sd, sh)
    _assert_same_buffer(tb_d, tb_h)
    assert len(tb_h.buffer) == n + 2


# ---- user envs: unknown horizon, ring lifetime, float64 rewards --------------------------------------------------
class UserEnv:
    """A user env with SafetyBallRun-v0's widths (D = 7, A = 2) and scripted episode lengths; rewards and costs are
    float64 values float32 cannot represent.  ``T=None`` leaves the horizon unknown (no spec)."""

    def __init__(self, i, lengths, T=None):
        from fsrl_b200.spaces import Box
        self.i, self.lengths, self.k = i, list(lengths), -1
        self.observation_space = Box(-np.inf, np.inf, (7,), np.float32)
        self.action_space = Box(-1.0, 1.0, (2,), np.float32)
        if T is not None:
            from fsrl_b200.envs import _Spec
            self.spec = _Spec("User-v0", T)

    def _obs(self):
        return np.array([self.i, self.k, self.t, 0.5, -0.5, 0.25, 1.0], np.float32)

    def reset(self, seed=None, options=None):
        self.k, self.t = self.k + 1, 0
        return self._obs(), {}

    def step(self, a):
        self.t += 1
        a = np.asarray(a, np.float64)
        rew = 0.1 + self.t / 3.0 + 1e-9 * self.i + 1e-3 * float(a.sum())
        cost = (self.t % 3) / 7.0
        L = self.lengths[self.k % len(self.lengths)]
        return self._obs(), rew, False, self.t >= L, {"cost": cost}


def _user_collector(lengths, cap, log, **tb_kw):
    from fsrl_b200.data import FastCollector, TrajectoryBuffer, VectorReplayBuffer
    from fsrl_b200.envs import HostVectorEnv
    E = len(lengths)
    venv = HostVectorEnv([lambda i=i: Recorder(UserEnv(i, lengths[i]), log) for i in range(E)])
    assert venv.max_episode_steps is None
    policy = build_ppo("SafetyBallRun-v0", n_env=1, seed=9)[0]
    policy.train()
    tb = TrajectoryBuffer(**tb_kw)
    with pytest.raises(ValueError, match="needs a buffer"):
        FastCollector(policy, venv, exploration_noise=True, traj_buffer=TrajectoryBuffer())
    col = FastCollector(policy, venv, VectorReplayBuffer(E * cap, E), exploration_noise=True, traj_buffer=tb)
    return col, tb


def test_unknown_horizon_and_float64_rewards():
    lengths = [[3, 9, 5], [7, 2, 11, 4], [12, 6]]
    log = []
    random.seed(2)
    np.random.seed(2)
    col, tb = _user_collector(lengths, 12, log)
    for _ in range(3):
        col.collect(n_episode=7)          # the ring of 12 slots wraps on every env
    torch.cuda.synchronize()
    ob = _oracle(log, 2)
    _assert_is_oracle(tb, ob)
    assert len(tb.buffer) == 21 and tb._arena.stride == 12          # the longest kept episode
    # the keep metrics are the float64 sums of what the envs reported, the stored columns their float32 roundings
    # summing the float32 column would not give the returns
    assert any(m[0] != float(np.sum(ep["rewards"].astype(np.float64))) for m, ep in zip(tb.metrics, ob.trajs))
    allr = np.concatenate([[t[2] for t in ep] for ep in log])
    assert not np.array_equal(allr.astype(np.float32).astype(np.float64), allr)


def test_episode_longer_than_the_ring_is_refused_before_any_overwrite():
    # env 0: episodes of 3, 4, then 20 steps; env 1: 2, 5, 6, then 25.  With 10 slots per env, env 0's third episode
    # reaches 11 steps at vector step 18, after five episodes ended (steps 2, 3, 7, 7, 13)
    lengths = [[3, 4, 20], [2, 5, 6, 25]]
    log = []
    col, tb = _user_collector(lengths, 10, log)
    with pytest.raises(ValueError, match="env 0's episode reached 11 steps, longer than the ring's 10 slots"):
        col.collect(n_episode=10)
    torch.cuda.synchronize()
    assert [len(ep) for ep in log] == [2, 3, 4, 5, 6]
    _assert_is_oracle(tb, _oracle(log, 0))


# ---- the example ------------------------------------------------------------------------------------------------
def test_collect_dataset_example_on_a_user_env(tmp_path):
    import sys
    sys.path.insert(0, os.path.join(ROOT, "examples"))
    import collect_dataset
    for n in (1, 8):
        argv = ["--user_env", "True", "--epoch", "2", "--step_per_epoch", "400", "--training_num", str(n),
                "--episode_per_collect", "8", "--testing_num", "2", "--hidden_sizes", "(64,64)",
                "--buffer_size", "3200", "--optim_critic_iters", "2", "--repeat_per_collect", "1",
                "--max_traj_len", "10", "--logdir", str(tmp_path), "--name", f"user{n}", "--epoch_start", "0",
                "--epoch_end", "2"]
        tb, path = collect_dataset.main(argv)
        z = np.load(path)
        assert len(tb.buffer) > 0 and len(z["rewards"]) == len(tb)
        assert z["observations"].shape[1] == 6 and z["actions"].shape[1] == 2
        ends = z["terminals"] | z["timeouts"]
        assert int(ends.sum()) == len(tb.buffer) and ends[-1]
