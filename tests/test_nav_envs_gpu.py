"""The Safety-Gymnasium navigation tasks (Point / Car on Circle 1-2 and Goal 1-2) on the device, against the
CPU env twin (oracle/envs_nav.py) and the oracle collector.

Random-mode actions come from the Philox stream with no MLP, so a random-mode collect is compared with the
oracle collector bit for bit.  A train-mode collect is replayed through the twin env by env from the
device's own stored actions.  The Goal2 tasks regenerate their layout from the reset's Philox stream inside
step and observe, so every comparison of them also checks that the device and the twin key it alike."""
import copy
import ctypes
import math
import os
import sys

import numpy as np
import pytest
import torch

from helpers import buffer_to_numpy, build_ppo

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TASKS = ["SafetyPointCircle1Gymnasium-v0", "SafetyPointCircle2Gymnasium-v0", "SafetyCarCircle1Gymnasium-v0",
         "SafetyCarCircle2Gymnasium-v0", "SafetyPointGoal2Gymnasium-v0", "SafetyCarGoal1Gymnasium-v0",
         "SafetyCarGoal2Gymnasium-v0"]
COLS = ("obs", "obs_next", "act", "rew", "cost", "terminated", "truncated")


def _twin(venv, E=None):
    from oracle.envs_nav import OracleVecEnvNav
    return OracleVecEnvNav(venv.kind, venv.env_num if E is None else E, venv.seed_value)


def _h(t):
    return t.detach().cpu().numpy()


@pytest.mark.parametrize("task", TASKS)
def test_env_reset_matches_twin_bitwise(task):
    _, venv, _, _ = build_ppo(task, n_env=33)
    oenv = _twin(venv)
    obs = oenv.reset()
    assert np.array_equal(_h(venv.obs_cur), obs)
    assert np.array_equal(_h(venv.env_state), oenv.st)


@pytest.mark.parametrize("task", TASKS)
@pytest.mark.parametrize("E,n_episode", [(16, 16), (6, 14)])
def test_random_collect_matches_oracle_bitwise(task, E, n_episode):
    """n_episode <= E retires every finished env inline; n_episode > E resets envs in the resolve kernel."""
    from oracle import collector as ocol
    T = 1000
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
    assert not b["terminated"].any() and stats["truncated"] == 1.0
    assert stats["total_cost"] > 0


@pytest.mark.parametrize("task", TASKS)
@pytest.mark.parametrize("E,n_episode", [(8, 8), (5, 7)])
def test_train_collect_replays_through_twin(task, E, n_episode):
    T = 1000
    rounds = n_episode // E + 2
    policy, venv, buf, col = build_ppo(task, n_env=E, buffer_size=E * T * rounds)
    policy.train()
    stats = col.collect(n_episode=n_episode)
    assert stats["n/ep"] == n_episode
    b = buffer_to_numpy(buf)
    oenv = _twin(venv)
    oenv.reset()
    L = b["len"].astype(np.int64)
    assert L.sum() == stats["n/st"]
    for t in range(int(L.max())):           # every env whose ring reaches row t, stepped together
        ids = np.nonzero(L > t)[0]
        p = ids * buf.cap + t
        assert np.array_equal(b["obs"][p], oenv.observe(ids)), t
        a = np.asarray(policy.map_action(b["act"][p]), np.float32)
        obs, rew, cost, term, trunc = oenv.step(a, ids)
        assert np.array_equal(b["obs_next"][p], obs), t
        assert np.array_equal(b["rew"][p], rew) and np.array_equal(b["cost"][p], cost), t
        assert not b["terminated"][p].any() and np.array_equal(b["truncated"][p], trunc), t
        if trunc.any():
            oenv.reset(ids[trunc])


@pytest.mark.parametrize("task", TASKS)
def test_step_and_reset_ids_match_twin(task):
    """DeviceVectorEnv.step / reset(id) on id subsets, past a horizon for the Circle tasks."""
    from fsrl_b200.envs import DeviceVectorEnv
    from oracle.philox import action_uniform
    E = 24
    venv = DeviceVectorEnv(task, E, device="cuda", seed=5)
    oenv = _twin(venv)
    obs, _ = venv.reset()
    assert np.array_equal(_h(obs), oenv.reset())
    rng = np.random.default_rng(3)
    for t in range(venv.max_episode_steps + 10 if venv.max_episode_steps <= 500 else 120):
        ids = np.sort(rng.permutation(E)[:rng.integers(1, E + 1)]) if t % 3 else None
        sel = np.arange(E) if ids is None else ids
        a = action_uniform(77, sel, np.full(len(sel), t, np.uint32), venv.A)
        o, rew, term, trunc, info = venv.step(torch.from_numpy(a).cuda(), ids)
        oo, orew, ocost, oterm, otrunc = oenv.step(a, ids)
        assert np.array_equal(_h(o), oo) and np.array_equal(_h(rew), orew), t
        assert np.array_equal(_h(info.cost), ocost) and np.array_equal(_h(trunc), otrunc) and not _h(term).any(), t
        done = sel[otrunc]
        if t % 7 == 0:
            done = np.union1d(done, sel[:2])
        if len(done):
            robs, _ = venv.reset(done)
            assert np.array_equal(_h(robs), oenv.reset(done)), t
    assert np.array_equal(_h(venv.obs_cur), oenv.observe())
    assert np.array_equal(_h(venv.env_state), oenv.st)
    assert np.array_equal(_h(venv.ep_idx).astype(np.uint32), oenv.ep_idx)


@pytest.mark.parametrize("task", ["SafetyCarCircle2Gymnasium-v0", "SafetyPointGoal2Gymnasium-v0"])
@pytest.mark.parametrize("E,n_episode", [(6, 6), (4, 7)])
def test_trajectory_harvest_matches_ring(task, E, n_episode):
    from test_trajbuf_gpu import _assert_same, _collect, _concat, _host
    policy, tb, stats, (eps,) = _collect(task, E, n_episode)
    assert len(tb.buffer) == len(eps) == stats["n/ep"]
    _assert_same(_host(tb.get_all()), _concat(eps), task)
    for i, ep in enumerate(eps):
        assert tb.metrics[i].tolist() == [ep["ret"], ep["cost"]]
        d = ep["data"]
        assert not d["terminals"].any() and d["timeouts"][-1] and not d["timeouts"][:-1].any()


def test_persistent_update_matches_chain_on_circle():
    """SafetyPointCircle1Gymnasium-v0 (D = 28) at H = 256, batch 256: the persistent launch against the
    three-launch chain, within the bounds the persistent path keeps against the fp32 oracle."""
    from fsrl_b200 import _lib
    from test_ppo_scale_gpu import KEYS, _collect, _sub_batch
    lag, lr = 0.3, 5e-4
    policy, batch, _, _, _ = _collect("SafetyPointCircle1Gymnasium-v0", (256, 256), 64, lag)
    sub = _sub_batch(policy, batch, 8 * 256)
    policy._target_kl = 1e9
    policy._ensure_update_state(256, sub.n, 1)
    u = policy._descriptor(sub, torch.zeros(sub.n, dtype=torch.int32, device="cuda"))
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


@pytest.mark.parametrize("algo,task,extra", [
    ("ppol", "SafetyPointCircle1Gymnasium-v0", ["--repeat_per_collect", "2", "--batch_size", "256"]),
    ("sacl", "SafetyCarGoal2Gymnasium-v0", ["--update_per_step", "0.05"]),
    ("cvpo", "SafetyCarCircle2Gymnasium-v0", ["--update_per_step", "0.05"]),
])
def test_agents_train_on_new_tasks_through_reference_imports(algo, task, extra, tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "examples"))
    import train_agent
    argv = ["--algo", algo, "--task", task, "--epoch", "2", "--step_per_epoch", "1600",
            "--training_num", "16", "--episode_per_collect", "16", "--testing_num", "2", "--hidden_sizes", "(64,64)",
            "--buffer_size", "32000", "--logdir", str(tmp_path), "--verbose", "False", "--save_interval", "1",
            "--cost_limit", "25"] + extra
    epoch, stats, info = train_agent.main(argv)
    assert epoch == 2 and info["train_speed"] > 0
    nums = {k: v for k, v in stats.items() if isinstance(v, (int, float))}
    assert "train/reward" in nums and all(math.isfinite(v) for v in nums.values()), nums
    run_dirs = os.listdir(tmp_path)
    assert run_dirs
    from fsrl_b200.utils.exp_util import load_config_and_model
    cfg, model = load_config_and_model(os.path.join(tmp_path, run_dirs[0]))
    assert cfg["task"] == task and any(k.startswith("actor.") for k in model["model"])
