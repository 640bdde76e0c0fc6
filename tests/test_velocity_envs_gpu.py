"""The Safety-Gymnasium velocity tasks (HalfCheetah, Hopper, Swimmer, Walker2d, Ant) on the device, against the CPU
env twin (oracle/envs_velocity.py), the oracle collector and the oracle returns.

Hopper, Walker2d and Ant end an episode on an unhealthy pose, so terminations are the common case here.  The env
battery of test_nav_envs_gpu.py is restated for episodes that may terminate: resets, random-mode collects against
the oracle collector on the inline and the resolve path, train-mode rings replayed through the twin, ``step`` /
``reset(id)`` on id subsets and the trajectory harvest.  The termination paths of test_drone_ant_run_gpu.py
(GAE's value mask, the cut of the n-step targets, the harvest's ``terminals``) run on Hopper and Walker2d.  The
persistent PPO launch is checked at action widths 3, 6 and 8 against the three-launch chain, and
examples/train_agent.py trains every learner end to end on one of the tasks."""
import copy
import ctypes

import numpy as np
import pytest
import torch

import test_drone_ant_run_gpu as drone
import test_nav_envs_gpu as nav
import test_rollout_one_launch_gpu as one
from helpers import buffer_to_numpy, build_ppo
from oracle.envs_velocity import OracleVecEnvVel

pytestmark = pytest.mark.gpu
TASKS = ["SafetyHalfCheetahVelocityGymnasium-v1", "SafetyHopperVelocityGymnasium-v1",
         "SafetySwimmerVelocityGymnasium-v1", "SafetyWalker2dVelocityGymnasium-v1", "SafetyAntVelocityGymnasium-v1"]
HOPPER, WALKER2D = "SafetyHopperVelocityGymnasium-v1", "SafetyWalker2dVelocityGymnasium-v1"
TERMINATING = (HOPPER, WALKER2D, "SafetyAntVelocityGymnasium-v1")
COLS = ("obs", "obs_next", "act", "rew", "cost", "terminated", "truncated")
T = 1000


def _twin(venv, E=None):
    return OracleVecEnvVel(venv.kind, venv.env_num if E is None else E, venv.seed_value)


def _h(t):
    return t.detach().cpu().numpy()


@pytest.fixture
def vel_twin(monkeypatch):
    """Point the twin test_nav_envs_gpu.py builds at the subclass that also takes kinds 33-37."""
    import oracle.envs_nav
    monkeypatch.setattr(oracle.envs_nav, "OracleVecEnvNav", OracleVecEnvVel)


@pytest.mark.parametrize("task", TASKS)
def test_env_reset_matches_twin_bitwise(task, vel_twin):
    nav.test_env_reset_matches_twin_bitwise(task)


@pytest.mark.parametrize("task", TASKS)
@pytest.mark.parametrize("E,n_episode", [(16, 16), (6, 14)])
def test_random_collect_matches_oracle_bitwise(task, E, n_episode):
    """n_episode <= E retires every finished env inline; n_episode > E resets envs after their episode ends (after a
    termination, on the terminating tasks) in the resolve kernel."""
    from oracle import collector as ocol
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
    assert np.array_equal(_h(venv.ep_idx).astype(np.uint32), oenv.ep_idx)
    assert np.array_equal(_h(venv.obs_cur), oenv.observe())
    assert np.array_equal(_h(venv.act_ctr).astype(np.uint32), ctr)
    if task in (HOPPER, WALKER2D):              # random play topples them (test_velocity_envs_host.py)
        assert b["terminated"].any() and stats["terminated"] > 0.5
    if task not in TERMINATING:
        assert not b["terminated"].any() and stats["truncated"] == 1.0


@pytest.mark.parametrize("task", TASKS)
@pytest.mark.parametrize("E,n_episode", [(8, 8), (5, 7)])
def test_train_collect_replays_through_twin(task, E, n_episode, monkeypatch):
    rounds = n_episode // E + 2
    policy, venv, buf, col = build_ppo(task, n_env=E, buffer_size=E * T * rounds)
    policy.train()
    stats = col.collect(n_episode=n_episode)
    assert stats["n/ep"] == n_episode
    monkeypatch.setattr(drone, "_twin", _twin)
    n_term = drone._replay(policy, venv, buf)
    assert n_term == int(buffer_to_numpy(buf)["terminated"].sum())
    assert stats["terminated"] == n_term / stats["n/ep"]
    if task in (HOPPER, WALKER2D):
        assert n_term > 0


@pytest.mark.parametrize("task", TASKS)
def test_step_and_reset_ids_match_twin(task):
    """DeviceVectorEnv.step / reset(id) on id subsets; envs that terminate or reach the horizon are reset."""
    from fsrl_b200.envs import DeviceVectorEnv
    from oracle.philox import action_uniform
    E = 24
    venv = DeviceVectorEnv(task, E, device="cuda", seed=5)
    oenv = _twin(venv)
    obs, _ = venv.reset()
    assert np.array_equal(_h(obs), oenv.reset())
    rng = np.random.default_rng(3)
    n_term = 0
    for t in range(1100 if task not in TERMINATING else 300):
        ids = np.sort(rng.permutation(E)[:rng.integers(1, E + 1)]) if t % 3 else None
        sel = np.arange(E) if ids is None else ids
        a = action_uniform(77, sel, np.full(len(sel), t, np.uint32), venv.A)
        o, rew, term, trunc, info = venv.step(torch.from_numpy(a).cuda(), ids)
        oo, orew, ocost, oterm, otrunc = oenv.step(a, ids)
        otrunc = otrunc & ~oterm
        assert np.array_equal(_h(o), oo) and np.array_equal(_h(rew), orew), t
        assert np.array_equal(_h(info.cost), ocost) and np.array_equal(_h(term), oterm), t
        assert np.array_equal(_h(trunc), otrunc), t
        n_term += int(oterm.sum())
        done = sel[oterm | otrunc]
        if t % 7 == 0:
            done = np.union1d(done, sel[:2])
        if len(done):
            robs, _ = venv.reset(done)
            assert np.array_equal(_h(robs), oenv.reset(done)), t
    assert np.array_equal(_h(venv.obs_cur), oenv.observe())
    assert np.array_equal(_h(venv.env_state), oenv.st)
    assert np.array_equal(_h(venv.ep_idx).astype(np.uint32), oenv.ep_idx)
    if task in (HOPPER, WALKER2D):
        assert n_term > 0


@pytest.mark.parametrize("task", [HOPPER, "SafetySwimmerVelocityGymnasium-v1", "SafetyAntVelocityGymnasium-v1"])
@pytest.mark.parametrize("E,n_episode", [(6, 6), (4, 11)])
def test_trajectory_harvest_matches_ring(task, E, n_episode):
    from test_trajbuf_gpu import _assert_same, _collect, _concat, _host
    policy, tb, stats, (eps,) = _collect(task, E, n_episode)
    assert len(tb.buffer) == len(eps) == stats["n/ep"]
    got = _host(tb.get_all())
    _assert_same(got, _concat(eps), task)
    for i, ep in enumerate(eps):
        assert tb.metrics[i].tolist() == [ep["ret"], ep["cost"]]
        d = ep["data"]
        # one flag per episode, on its last row, and it is the ring's own flag
        assert d["terminals"][:-1].sum() == 0 and d["timeouts"][:-1].sum() == 0
        assert bool(d["terminals"][-1]) != bool(d["timeouts"][-1])
    n_term = sum(bool(ep["data"]["terminals"][-1]) for ep in eps)
    assert int(got["terminals"].sum()) == n_term and stats["terminated"] == n_term / len(eps)
    if task == HOPPER:
        assert n_term > 0


# ---- terminations end to end --------------------------------------------------------------------------------
@pytest.mark.parametrize("task", [HOPPER])
def test_gae_with_real_terminations(task):
    """process_fn on a ring against oracle.returns.dual_gae fed the device's own critic values; a terminated row
    bootstraps from zero, a truncated one from V(obs_next)."""
    from oracle import returns
    E = 32
    policy, venv, buf, col = build_ppo(task, n_env=E)
    col.collect(n_episode=E)
    idx = buf.sample_indices(0)
    batch = policy.process_fn(None, buf, idx)
    b = buffer_to_numpy(buf)
    sel = idx.cpu().numpy()
    term, trunc = b["terminated"][sel], b["truncated"][sel]
    assert term.any()
    v = batch.values.cpu().numpy().T.copy()                      # (C, n)
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
        assert drone._ulp_diff(adv[:, c], advs[:, c]).max() <= 1
        assert drone._ulp_diff(ret[:, c], rets[:, c]).max() <= 1
    m = [b["rew"][sel].astype(np.float64), b["cost"][sel].astype(np.float64)]
    for c in range(v.shape[0]):
        want_t = (m[c][term] - v[c, term].astype(np.float64)).astype(np.float32)
        assert drone._ulp_diff(adv[term, c], want_t).max() <= 1


@pytest.mark.parametrize("task", [WALKER2D])
def test_nstep_targets_cut_at_terminations(task):
    """compute_nstep_returns of SAC-Lagrangian on a ring against oracle.offpolicy.nstep_targets."""
    from fsrl_b200 import envs
    from fsrl_b200.agent import SACLagAgent
    from fsrl_b200.data import FastCollector, VectorReplayBuffer
    from oracle import offpolicy as ooff
    from oracle.collector import OracleBuffer
    E = 4
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
        np.testing.assert_allclose(got[:, 0, :], rets, rtol=1e-6, atol=1e-6)
        hit = ob.terminated[idx]
        np.testing.assert_allclose(got[hit, 0, 0], b["rew"][idx[hit]], rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(got[hit, 0, 1], b["cost"][idx[hit]], rtol=1e-6, atol=1e-6)


# ---- one launch per collect ---------------------------------------------------------------------------------
@pytest.mark.parametrize("task", TASKS)
@pytest.mark.parametrize("H", [128, 256])
def test_one_launch_every_new_env(task, H, monkeypatch):
    ref = one._compare(task, H, "indep", "train", 2048, 2048, T, monkeypatch)
    assert ref["finished"] == 1 and ref["episode_count"] == 2048
    if task in (HOPPER, WALKER2D):
        assert ref["term_count"] > 0
    one._compare(task, H, "indep", "train", 17, 17, 41, monkeypatch)            # cut short: episodes still running


# ---- the persistent PPO launch at action widths 3, 6 and 8 --------------------------------------------------
@pytest.mark.parametrize("task,D,A", [(HOPPER, 11, 3), (WALKER2D, 17, 6), ("SafetyAntVelocityGymnasium-v1", 27, 8)])
def test_persistent_update_matches_chain(task, D, A):
    """At H = 256, batch 256 the gate admits these tasks; one repeat of the persistent launch against the three-launch
    chain, within the bounds test_nav_envs_gpu.py keeps on a Circle task."""
    from fsrl_b200 import _lib
    from test_ppo_scale_gpu import KEYS, _collect, _sub_batch
    lag, lr = 0.3, 5e-4
    policy, batch, _, _, _ = _collect(task, (256, 256), 256, lag)      # 256 envs: short episodes still fill 8 batches
    assert batch.obs.shape[0] >= 8 * 256
    sub = _sub_batch(policy, batch, 8 * 256)
    policy._target_kl = 1e9
    policy._ensure_update_state(256, sub.n, 1)
    u = policy._descriptor(sub, torch.zeros(sub.n, dtype=torch.int32, device="cuda"))
    assert (u.D, u.A) == (D, A)
    assert _lib.lib.fsrl_ppo_persist_active(ctypes.byref(u), sub.n, 256) == 1
    sd0 = copy.deepcopy(policy.state_dict())
    out = []
    for off in (False, True):
        policy.load_state_dict(sd0)
        policy.optim.m.zero_(); policy.optim.v.zero_(); policy.optim.step_count = 0
        policy._persist_off = off
        np.random.seed(41)
        policy.learn(sub, batch_size=256, repeat=1)
        torch.cuda.synchronize()
        out.append((copy.deepcopy(policy.last_stats), policy.arena.theta.double().cpu().numpy().copy()))
    policy._persist_off = False
    (sp, pp), (sc, pc) = out
    for key in KEYS:
        assert len(sp[key]) == 8
        np.testing.assert_allclose(np.asarray(sp[key]), np.asarray(sc[key]), rtol=3e-4, atol=3e-6, err_msg=key)
    d = np.abs(pp - pc)
    assert (d > 2e-5).mean() <= 1e-3 and d.max() <= 0.5 * lr * 8 and np.median(d) <= 1e-7, d.max()


# ---- training end to end ------------------------------------------------------------------------------------
@pytest.mark.parametrize("algo,task,extra", [
    ("ppol", HOPPER, ["--repeat_per_collect", "2", "--batch_size", "256"]),
    ("cpo", "SafetyHalfCheetahVelocityGymnasium-v1", []),
    ("focops", "SafetySwimmerVelocityGymnasium-v1", []),
    ("trpol", WALKER2D, []),
    ("sacl", WALKER2D, ["--update_per_step", "0.05"]),
    ("ddpgl", "SafetyAntVelocityGymnasium-v1", ["--update_per_step", "0.05"]),
    ("cvpo", HOPPER, ["--update_per_step", "0.05"]),
])
def test_agents_train_on_velocity_tasks(algo, task, extra, tmp_path):
    nav.test_agents_train_on_new_tasks_through_reference_imports(algo, task, extra, tmp_path)
