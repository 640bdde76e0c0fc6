"""SafetyAntRun-v0, SafetyDroneCircle-v0 and SafetyDroneRun-v0 on the device, against the CPU env twin
(oracle/envs_flight.py), the oracle collector and the oracle returns.

The Drone tasks are the first device environments that terminate (a crash or a flip), so besides the
env models these tests drive the termination paths end to end with real flags: the rollout kernel's
``terminated`` store and count, the resolve kernel's reset after a termination, the value mask of GAE,
the cut of the n-step targets and the ``terminals`` of the trajectory harvest.

Random-mode actions come from the Philox stream with no MLP, so a random-mode collect is compared with
the oracle collector bit for bit.  A train-mode collect is replayed through the twin env by env from
the device's own stored actions: float noise of the actor MLP may move a crash by a step, so a
train-mode trajectory is never compared with an independent oracle collect."""
import math
import os
import sys

import numpy as np
import pytest
import torch

from helpers import buffer_to_numpy, build_ppo

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TASKS = ["SafetyAntRun-v0", "SafetyDroneCircle-v0", "SafetyDroneRun-v0"]
DRONES = ["SafetyDroneCircle-v0", "SafetyDroneRun-v0"]
COLS = ("obs", "obs_next", "act", "rew", "cost", "terminated", "truncated")


def _twin(venv, E=None):
    from oracle.envs_flight import OracleVecEnvExt
    return OracleVecEnvExt(venv.kind, venv.env_num if E is None else E, venv.seed_value)


def _ulp_diff(a, b):
    ai = a.view(np.int32).astype(np.int64)
    bi = b.view(np.int32).astype(np.int64)
    ai = np.where(ai < 0, np.int64(-2**31) - ai, ai)
    bi = np.where(bi < 0, np.int64(-2**31) - bi, bi)
    return np.abs(ai - bi)


@pytest.mark.parametrize("task", TASKS)
def test_env_reset_matches_twin_bitwise(task):
    _, venv, _, _ = build_ppo(task, n_env=33)
    oenv = _twin(venv)
    obs = oenv.reset()
    assert np.array_equal(venv.obs_cur.cpu().numpy(), obs)
    assert np.array_equal(venv.env_state.cpu().numpy(), oenv.st)


@pytest.mark.parametrize("task", TASKS)
@pytest.mark.parametrize("E,n_episode", [(16, 16), (16, 10), (6, 20)])
def test_random_collect_matches_oracle_bitwise(task, E, n_episode):
    """n_episode <= E retires every finished env inline; n_episode > E resets envs after their episode
    ends (after a termination, for the Drone tasks) in the resolve kernel."""
    from oracle import collector as ocol
    T = 300
    rounds = n_episode // E + 2
    policy, venv, buf, col = build_ppo(task, n_env=E, buffer_size=E * T * rounds)
    stats = col.collect(n_episode=n_episode, random=True)
    oenv = _twin(venv)
    oenv.reset()
    obuf = ocol.OracleBuffer(E * T * rounds, E, venv.D, venv.A)
    ctr = np.zeros(E, np.uint32)
    ostats = ocol.collect(oenv, None, n_episode, policy._act_seed, ctr, obuf, mode="random",
                          action_bound=policy.action_bound_method or "none")
    assert buf.cap == obuf.cap
    for k in ("n/ep", "n/st", "terminated", "truncated", "total_cost"):
        assert stats[k] == ostats[k], k
    assert stats["len"] == ostats["len"]
    assert stats["rew"] == pytest.approx(ostats["rew"], rel=1e-12, abs=1e-12)
    b = buffer_to_numpy(buf)
    assert np.array_equal(b["ptr"], obuf.ptr) and np.array_equal(b["len"], obuf.len)
    for k in COLS:
        assert np.array_equal(b[k], getattr(obuf, k)), k
    # the collect ends with a reset of every env: same episode counters, same fresh observations
    assert np.array_equal(venv.ep_idx.cpu().numpy().astype(np.uint32), oenv.ep_idx)
    assert np.array_equal(venv.obs_cur.cpu().numpy(), oenv.observe())
    assert np.array_equal(venv.act_ctr.cpu().numpy().astype(np.uint32), ctr)
    if task in DRONES:
        assert b["terminated"].any() and stats["terminated"] > 0
    else:
        assert not b["terminated"].any() and stats["truncated"] == 1.0


def _replay(policy, venv, buf):
    """Step the twin env by env with the device's stored actions; every stored column must match.
    Returns the number of terminated steps seen."""
    b = buffer_to_numpy(buf)
    oenv = _twin(venv)
    oenv.reset()
    n_term = 0
    for e in range(venv.env_num):
        for t in range(int(b["len"][e])):
            p = e * buf.cap + t
            assert np.array_equal(b["obs"][p], oenv.observe([e])[0]), (e, t)
            a = np.asarray(policy.map_action(b["act"][p][None]), np.float32)
            obs, rew, cost, term, trunc = oenv.step(a, [e])
            trunc = trunc & ~term
            assert np.array_equal(b["obs_next"][p], obs[0]), (e, t)
            assert b["rew"][p] == rew[0] and b["cost"][p] == cost[0], (e, t)
            assert b["terminated"][p] == term[0] and b["truncated"][p] == trunc[0], (e, t)
            if term[0] or trunc[0]:
                n_term += int(term[0])
                oenv.reset([e])
    return n_term


@pytest.mark.parametrize("task", TASKS)
@pytest.mark.parametrize("E,n_episode", [(8, 8), (5, 17)])
def test_train_collect_replays_through_twin(task, E, n_episode):
    T = 300
    rounds = n_episode // E + 2
    policy, venv, buf, col = build_ppo(task, n_env=E, buffer_size=E * T * rounds)
    policy.train()
    stats = col.collect(n_episode=n_episode)
    assert stats["n/ep"] == n_episode
    n_term = _replay(policy, venv, buf)
    b = buffer_to_numpy(buf)
    assert n_term == int(b["terminated"].sum())
    assert stats["terminated"] == n_term / stats["n/ep"]
    if task in DRONES:
        assert n_term > 0


def test_gae_with_real_terminations():
    """process_fn on a Drone-Circle ring against oracle.returns.dual_gae fed the device's own critic
    values; a terminated row bootstraps from zero, a truncated one from V(obs_next)."""
    from oracle import returns
    E = 32
    policy, venv, buf, col = build_ppo("SafetyDroneCircle-v0", n_env=E)
    col.collect(n_episode=E)
    idx = buf.sample_indices(0)
    batch = policy.process_fn(None, buf, idx)
    b = buffer_to_numpy(buf)
    sel = idx.cpu().numpy()
    term, trunc = b["terminated"][sel], b["truncated"][sel]
    assert term.any()
    v = batch.values.cpu().numpy().T.copy()                      # (C, n)
    # V(obs_next): the device's value of the identical next row inside an episode, a critic pass elsewhere
    obs, obs_next = b["obs"][sel], b["obs_next"][sel]
    n = len(sel)
    same = np.zeros(n, bool)
    same[:-1] = (obs_next[:-1] == obs[1:]).all(1)
    vnext = np.zeros_like(v)
    vnext[:, :-1] = v[:, 1:]
    rest = np.nonzero(~same)[0]
    on = torch.from_numpy(np.ascontiguousarray(obs_next)).cuda()
    ridx = torch.from_numpy(rest.astype(np.int32)).cuda()
    for i in range(v.shape[0]):
        vnext[i, rest] = policy.net_forward(1 + i, on, idx=ridx).flatten().cpu().numpy()
    assert np.all(vnext[:, term] != 0)                           # the mask, not the critic, zeroes them
    unf = np.zeros(n, bool)
    _, rets, advs = returns.dual_gae(v, vnext, b["rew"][sel], b["cost"][sel], term, trunc, unf, 0.99, 0.95)
    adv, ret = batch.advs.cpu().numpy(), batch.rets.cpu().numpy()
    for c in range(v.shape[0]):
        assert _ulp_diff(adv[:, c], advs[:, c]).max() <= 1
        assert _ulp_diff(ret[:, c], rets[:, c]).max() <= 1
    # terminated rows: adv = r - V(s); truncated rows: adv = r + gamma V(s') - V(s)
    m = [b["rew"][sel].astype(np.float64), b["cost"][sel].astype(np.float64)]
    for c in range(v.shape[0]):
        want_t = (m[c][term] - v[c, term].astype(np.float64)).astype(np.float32)
        assert _ulp_diff(adv[term, c], want_t).max() <= 1
        want_u = (m[c][trunc] + vnext[c, trunc].astype(np.float64) * 0.99 - v[c, trunc]).astype(np.float32)
        assert _ulp_diff(adv[trunc, c], want_u).max(initial=0) <= 1


def test_nstep_targets_cut_at_terminations():
    """compute_nstep_returns of SAC-Lagrangian on a Drone-Run ring against oracle.returns.nstep_return."""
    from fsrl_b200 import envs
    from fsrl_b200.agent import SACLagAgent
    from fsrl_b200.data import FastCollector, VectorReplayBuffer
    from oracle import offpolicy as ooff
    from oracle.collector import OracleBuffer
    task, E = "SafetyDroneRun-v0", 4
    env = envs.make(task)
    agent = SACLagAgent(env, seed=10, hidden_sizes=(64, 64), unbounded=True, n_step=2, tau=0.05)
    policy = agent.policy
    venv = envs.DeviceVectorEnv(task, E, seed=12)
    buf = VectorReplayBuffer(E * env.spec.max_episode_steps, E)
    col = FastCollector(policy, venv, buf, exploration_noise=True)
    col.collect(n_episode=12)
    b = buffer_to_numpy(buf)
    assert b["terminated"].any()
    ob = OracleBuffer(buf.maxsize, buf.buffer_num, buf.D, buf.A)
    for k in COLS:
        setattr(ob, k, b[k])
    ob.ptr = b["ptr"].astype(np.int64); ob.len = b["len"].astype(np.int64)
    rng = np.random.default_rng(1)
    valid = ob.sample_all()
    # every terminated row and its predecessors, plus a uniform draw
    tr = valid[ob.terminated[valid]]
    idx = np.concatenate([tr, tr - 1, tr - 2, rng.choice(valid, 200)]).astype(np.int64)
    idx = idx[np.isin(idx, valid)]
    B = len(idx)
    for n_step in (1, 2, 3, 5):
        tq = [rng.standard_normal(B).astype(np.float32) for _ in range(2)]
        seen = {}

        def target_q_fn(buffer, terminal):
            seen["terminal"] = terminal.cpu().numpy().copy()
            return [torch.from_numpy(t).cuda().reshape(-1, 1) for t in tq]

        batch = policy.compute_nstep_returns(None, buf, idx, target_q_fn, n_step)
        rets, terminal = ooff.nstep_targets(ob, idx, tq, policy._gamma, n_step)
        assert np.array_equal(seen["terminal"], terminal.astype(np.int32))
        got = batch.rets.cpu().numpy()
        assert got.shape == (B, 1, 2)
        np.testing.assert_allclose(got[:, 0, :], rets, rtol=1e-6, atol=1e-6)
        # a terminated transition's target is its own reward and cost: nothing is bootstrapped
        hit = ob.terminated[idx]
        np.testing.assert_allclose(got[hit, 0, 0], b["rew"][idx[hit]], rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(got[hit, 0, 1], b["cost"][idx[hit]], rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("E,n_episode", [(8, 8), (6, 15)])
def test_trajectory_harvest_keeps_terminals(E, n_episode):
    from test_trajbuf_gpu import _assert_same, _collect, _concat, _host
    policy, tb, stats, (eps,) = _collect("SafetyDroneCircle-v0", E, n_episode)
    assert len(tb.buffer) == len(eps) == stats["n/ep"]
    got = _host(tb.get_all())
    _assert_same(got, _concat(eps))
    for i, ep in enumerate(eps):
        assert tb.metrics[i].tolist() == [ep["ret"], ep["cost"]]
        d = ep["data"]
        # one flag per episode, on its last row, and it is the ring's own flag
        assert d["terminals"][:-1].sum() == 0 and d["timeouts"][:-1].sum() == 0
        assert bool(d["terminals"][-1]) != bool(d["timeouts"][-1])
    n_term = sum(bool(ep["data"]["terminals"][-1]) for ep in eps)
    assert n_term > 0 and int(got["terminals"].sum()) == n_term
    assert stats["terminated"] == n_term / len(eps)


@pytest.mark.parametrize("algo,task,extra", [
    ("ppol", "SafetyDroneCircle-v0", ["--repeat_per_collect", "2", "--batch_size", "256"]),
    ("ppol", "SafetyAntRun-v0", ["--repeat_per_collect", "2", "--batch_size", "256"]),
    ("sacl", "SafetyDroneRun-v0", ["--update_per_step", "0.05"]),
])
def test_agents_train_on_new_tasks_through_reference_imports(algo, task, extra, tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "examples"))
    import train_agent
    argv = ["--algo", algo, "--task", task, "--epoch", "2", "--step_per_epoch", "1600",
            "--training_num", "16", "--episode_per_collect", "16", "--testing_num", "2", "--hidden_sizes", "(64,64)",
            "--buffer_size", "6400", "--logdir", str(tmp_path), "--verbose", "False", "--save_interval", "1"] + extra
    epoch, stats, info = train_agent.main(argv)     # ends with agent.evaluate on the test envs
    assert epoch == 2 and info["train_speed"] > 0
    nums = {k: v for k, v in stats.items() if isinstance(v, (int, float))}
    assert "train/reward" in nums and all(math.isfinite(v) for v in nums.values()), nums
    run_dirs = os.listdir(tmp_path)
    assert run_dirs
    from fsrl_b200.utils.exp_util import load_config_and_model
    cfg, model = load_config_and_model(os.path.join(tmp_path, run_dirs[0]))
    assert cfg["task"] == task and any(k.startswith("actor.") for k in model["model"])
