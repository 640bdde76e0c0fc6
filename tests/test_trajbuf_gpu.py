"""Device harvest of finished episodes into TrajectoryBuffer (csrc/trajbuf.cu) against the ring contents.

The expected dataset is rebuilt on the host from a ring that holds the whole collect: every env's slots in
time order, cut at the done flags, episodes ordered by (finish step, env), open episodes dropped, actions
passed through the policy's host map_action.  Everything is compared bitwise; the returns are fp64 sums of
the fp32 rewards in time order, like the rollout's own episode return."""
import json
import os
import random

import numpy as np
import pytest
import torch

from helpers import buffer_to_numpy, build_ppo, oracle_nets
from oracle.trajbuf import OracleTrajBuf

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TASKS = ["SafetyCarCircle-v0", "SafetyCarRun-v0", "SafetyBallCircle-v0", "SafetyBallRun-v0",
         "SafetyAntCircle-v0", "SafetyPointGoal1Gymnasium-v0"]
KEYS = ("observations", "next_observations", "actions", "rewards", "costs", "terminals", "timeouts")


def _episodes(policy, buf):
    """episodes in a fresh whole-collect ring (written from slot 0), in (finish step, env) order"""
    b = buffer_to_numpy(buf)
    out = []
    for e in range(buf.buffer_num):
        lo, n = e * buf.cap, int(b["len"][e])
        start = 0
        for t in range(n):
            if b["terminated"][lo + t] or b["truncated"][lo + t]:
                s = slice(lo + start, lo + t + 1)
                ret = cost = 0.0
                for r, c in zip(b["rew"][s], b["cost"][s]):
                    ret += float(r)
                    cost += float(c)
                out.append(dict(finish=t + 1, env=e, ret=ret, cost=cost, data=dict(
                    observations=b["obs"][s], next_observations=b["obs_next"][s],
                    actions=policy.map_action(b["act"][s]), rewards=b["rew"][s], costs=b["cost"][s],
                    terminals=b["terminated"][s], timeouts=b["truncated"][s])))
                start = t + 1
    out.sort(key=lambda x: (x["finish"], x["env"]))
    return out


def _host(batch):
    return {k: batch[k].cpu().numpy() for k in KEYS}


def _assert_same(got, want, msg=""):
    for k in KEYS:
        assert got[k].dtype == want[k].dtype or k in ("terminals", "timeouts"), (k, got[k].dtype, want[k].dtype)
        assert np.array_equal(got[k], want[k]), (msg, k)


def _concat(eps):
    return {k: np.concatenate([e["data"][k] for e in eps]) for k in KEYS}


def _collect(task, E, n_episode, cap=None, collects=1, seed=10, rng_seed=None, **tb_kw):
    from fsrl_b200.data import FastCollector, TrajectoryBuffer, VectorReplayBuffer
    policy, venv, _, _ = build_ppo(task, n_env=E, seed=seed)
    if rng_seed is not None:       # the draws of the keep rules
        random.seed(rng_seed)
        np.random.seed(rng_seed)
    T = venv.max_episode_steps
    whole = cap is None
    cap = cap or T * (n_episode // E + 2)
    buf = VectorReplayBuffer(E * cap, E)
    tb = TrajectoryBuffer(**tb_kw)
    col = FastCollector(policy, venv, buf, exploration_noise=True, traj_buffer=tb)
    eps = []
    for _ in range(collects):
        if whole:
            col.reset_buffer()
        stats = col.collect(n_episode=n_episode)
        if whole:
            eps.append(_episodes(policy, buf))
    return policy, tb, stats, eps


@pytest.mark.parametrize("task", TASKS)
@pytest.mark.parametrize("E,n_episode", [(6, 6), (6, 4), (4, 11)])
def test_harvest_is_bit_exact(task, E, n_episode):
    policy, tb, stats, (eps,) = _collect(task, E, n_episode)
    assert len(tb.buffer) == len(eps) == stats["n/ep"]
    _assert_same(_host(tb.get_all()), _concat(eps), task)
    for i, ep in enumerate(eps):
        assert tb.metrics[i].tolist() == [ep["ret"], ep["cost"]]
        _assert_same(_host(tb.buffer[i]), ep["data"], (task, i))
    assert len(tb) == sum(len(e["data"]["rewards"]) for e in eps)
    if n_episode <= E:        # every ready env runs one whole episode: no partial episode to drop
        assert len(tb) == stats["n/st"]
    else:
        assert len(tb) <= stats["n/st"]
    # the episode returns are the rollout's own: their mean is the collect's "rew"
    assert sum(e["ret"] for e in eps) / len(eps) == pytest.approx(stats["rew"], rel=1e-12, abs=1e-12)


@pytest.mark.parametrize("task,E,n_episode", [("SafetyBallRun-v0", 4, 11), ("SafetyCarCircle-v0", 6, 6),
                                              ("SafetyPointGoal1Gymnasium-v0", 3, 7)])
def test_minimal_ring_gives_the_same_dataset(task, E, n_episode):
    from fsrl_b200.data import FastCollector, TrajectoryBuffer, VectorReplayBuffer
    _, tb_whole, _, _ = _collect(task, E, n_episode)
    policy, venv, _, _ = build_ppo(task, n_env=E, seed=10)
    T = venv.max_episode_steps
    tb = TrajectoryBuffer()
    if n_episode > E:              # below the least capacity: refused before any step
        p0, v0, _, _ = build_ppo(task, n_env=E, seed=10)
        small = FastCollector(p0, v0, VectorReplayBuffer(E * T, E), traj_buffer=TrajectoryBuffer())
        with pytest.raises(ValueError, match=str(T + 64)):
            small.collect(n_episode=n_episode)
    cap = T if n_episode <= E else T + 64
    col = FastCollector(policy, venv, VectorReplayBuffer(E * cap, E), exploration_noise=True, traj_buffer=tb)
    col.collect(n_episode=n_episode)
    assert [m.tolist() for m in tb.metrics] == [m.tolist() for m in tb_whole.metrics]
    _assert_same(_host(tb.get_all()), _host(tb_whole.get_all()), task)


def test_basic_collector_matches_fast_collector_and_oracle():
    from fsrl_b200.data import BasicCollector, FastCollector, TrajectoryBuffer, VectorReplayBuffer
    task, n = "SafetyBallCircle-v0", 3
    policy, venv, _, _ = build_ppo(task, n_env=1, seed=4)
    tb1 = TrajectoryBuffer()
    bc = BasicCollector(policy, venv, traj_buffer=tb1)
    assert bc.buffer.cap == venv.max_episode_steps + 64
    with pytest.raises(ValueError):
        bc.collect()
    stats = bc.collect(n_episode=n)
    policy2, venv2, _, _ = build_ppo(task, n_env=1, seed=4)
    T = venv2.max_episode_steps
    tb2 = TrajectoryBuffer()
    FastCollector(policy2, venv2, VectorReplayBuffer(T * (n + 1), 1), traj_buffer=tb2).collect(n_episode=n)
    assert len(tb1.buffer) == n
    _assert_same(_host(tb1.get_all()), _host(tb2.get_all()))
    # the oracle collector over one env
    from oracle import collector as ocol
    from oracle.envs import OracleVecEnv
    policy3, venv3, _, _ = build_ppo(task, n_env=1, seed=4)
    actor, _ = oracle_nets(policy3, (64, 64))
    oenv = OracleVecEnv(venv3.kind, 1, venv3.seed_value)
    oenv.reset()
    oenv.reset()                   # build_ppo's collector and the BasicCollector each reset the env once
    obuf = ocol.OracleBuffer(T * (n + 1), 1, venv3.D, venv3.A)
    ost = ocol.collect(oenv, actor, n, policy3._act_seed, np.zeros(1, np.uint32), obuf)
    for k in ("n/ep", "n/st", "truncated", "terminated"):
        assert stats[k] == ost[k], k
    assert abs(stats["rew"] - ost["rew"]) <= 1e-2 * max(1.0, abs(ost["rew"]))
    assert abs(stats["cost"] - ost["cost"]) <= 1.0


def _replay(eps_per_collect, seed, **kw):
    random.seed(seed)
    np.random.seed(seed)
    ob = OracleTrajBuf(**kw)
    for eps in eps_per_collect:
        for ep in eps:
            ob.add(ep["data"], ep["ret"], ep["cost"])
    return ob


@pytest.mark.parametrize("kind", ["grid", "replace", "window"])
def test_filters_on_device_match_the_oracle(kind):
    task, E, n_episode, collects = "SafetyCarCircle-v0", 16, 16, 4
    kw = dict(max_trajectory=4, filter_interval=1.5)
    if kind == "replace":
        kw = dict(max_trajectory=5, use_grid_filter=False)
    if kind == "window":
        _, _, _, pilot = _collect(task, E, n_episode, collects=1, max_trajectory=1)
        rets = np.array([e["ret"] for e in pilot[0]])
        kw.update(rmin=float(np.quantile(rets, 0.2)), rmax=float(np.quantile(rets, 0.8)))
    _, tb, _, eps = _collect(task, E, n_episode, collects=collects, rng_seed=3, **kw)
    ob = _replay(eps, 3, **kw)
    assert [m.tolist() for m in tb.metrics] == [m.tolist() for m in ob.metrics]
    assert len(tb.buffer) == len(ob.trajs)
    _assert_same(_host(tb.get_all()), ob.concat(), kind)
    if kind == "grid":       # filter_interval 1.5 over 16 episodes per harvest: the filter ran inside harvests
        assert sum(len(e) for e in eps) > 3 * 6 and len(tb.buffer) < 6


def test_host_store_reproduces_the_reference():
    from fsrl_b200.data import Batch, TrajectoryBuffer
    g = json.load(open(os.path.join(ROOT, "tests", "golden", "trajbuf_golden.json")))
    for s in g["scenarios"]:
        random.seed(s["seed"])
        np.random.seed(s["seed"])
        tb = TrajectoryBuffer(**s["kwargs"])
        for k, ep in enumerate(s["episodes"]):
            for t in range(ep["len"]):
                last = t == ep["len"] - 1
                obs = np.array([[1000 * k + t, k, t]], np.float32)
                tb.store(Batch(observations=obs, next_observations=obs + 0.5,
                               actions=np.array([[0.25 * t, -0.5 * k]], np.float32),
                               rewards=np.array([ep["rew"][t]], np.float32), costs=np.array([ep["cost"][t]], np.float32),
                               terminals=np.array([last and ep["terminal"]]),
                               timeouts=np.array([last and not ep["terminal"]])))
            want = s["after"][k]
            assert [int(tr["observations"][0, 0].item()) // 1000 for tr in tb.buffer] == want["kept"], (s["name"], k)
            assert [m.tolist() for m in tb.metrics] == want["metrics"]
            assert len(tb) == want["n_transitions"]
        got = _host(tb.get_all())
        ids = got["observations"][:, 0].astype(np.int64)
        want_ids = np.concatenate([1000 * k + np.arange(s["episodes"][k]["len"]) for k in s["after"][-1]["kept"]])
        assert np.array_equal(ids, want_ids)
        assert np.array_equal(got["next_observations"], got["observations"] + np.float32(0.5))


def test_read_out_api_and_save(tmp_path):
    policy, tb, stats, (eps,) = _collect("SafetyBallRun-v0", 5, 12)
    allb = tb.get_all()
    N = len(tb)
    D, A = eps[0]["data"]["observations"].shape[1], eps[0]["data"]["actions"].shape[1]
    assert allb["observations"].shape == (N, D) and allb["actions"].shape == (N, A)
    assert allb["rewards"].shape == (N,) and allb["terminals"].dtype == torch.bool
    assert allb["observations"].is_cuda and len(tb.buffer) == len(eps)
    assert len(tb.buffer[-1]["rewards"]) == len(eps[-1]["data"]["rewards"])
    # sample: the reference's draws (trajectory, then a transition inside it)
    np.random.seed(8)
    s = tb.sample(64)
    np.random.seed(8)
    traj = np.random.randint(0, len(eps), size=64)
    rows = []
    for i in range(64):
        rows.append((traj[i], np.random.randint(0, len(eps[traj[i]]["data"]["rewards"]))))
    want = {k: np.stack([eps[i]["data"][k][t] for i, t in rows]) for k in KEYS}
    _assert_same(_host(s), want, "sample")
    # save: <log_dir>/<stem>.npz with the seven keys
    tb.save(str(tmp_path / "out"), "data.hdf5")
    z = np.load(tmp_path / "out" / "data.npz")
    assert sorted(z.files) == sorted(KEYS)
    for k in KEYS:
        assert z[k].dtype == (np.bool_ if k in ("terminals", "timeouts") else np.float32)
        assert np.array_equal(z[k], allb[k].cpu().numpy()), k


def test_collect_dataset_example_both_paths(tmp_path):
    import sys
    sys.path.insert(0, os.path.join(ROOT, "examples"))
    import collect_dataset
    for n in (1, 8):
        argv = ["--task", "SafetyBallRun-v0", "--epoch", "2", "--step_per_epoch", "400", "--training_num", str(n),
                "--episode_per_collect", "8", "--testing_num", "2", "--hidden_sizes", "(64,64)",
                "--buffer_size", "3200", "--optim_critic_iters", "2", "--repeat_per_collect", "1",
                "--max_traj_len", "10", "--logdir", str(tmp_path), "--name", f"n{n}", "--epoch_start", "0",
                "--epoch_end", "2"]
        tb, path = collect_dataset.main(argv)
        z = np.load(path)
        assert len(tb.buffer) > 0 and len(z["rewards"]) == len(tb)
        ends = z["terminals"] | z["timeouts"]
        assert int(ends.sum()) == len(tb.buffer) and ends[-1]
