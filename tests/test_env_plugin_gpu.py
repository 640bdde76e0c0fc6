"""User-defined device envs (plugins built by fsrl_b200.envs.build_device_env) on the device.

- A plugin of a built-in env struct is bit-identical to the built-in kind: collects in every mode on the inline and
  the resolve path, step() / reset(id), the observation-normalizing wrapper, the trajectory harvest, a PPO-Lagrangian
  epoch and SAC-Lagrangian gradient steps.
- HazardDash (tests/envs/hazard_dash.h), an env the library does not have, replays bit for bit on its numpy twin
  (tests/env_plugin_twin.py), and every agent trains on it.
- Two plugins coexist in one process; rendering, a foreign ABI version and unregistered plugin kinds are refused.

The plugins are built by build() into PLUGIN_DIR; these tests only load them."""
import os

import numpy as np
import pytest
import torch

from env_plugin_twin import PLUGIN_DIR, HazardDashTwin, header
from helpers import buffer_to_numpy, build_ppo

pytestmark = pytest.mark.gpu
SAME = {"car_circle": "SafetyCarCircle-v0", "drone_circle": "SafetyDroneCircle-v0",
        "car_button1": "SafetyCarButton1Gymnasium-v0"}
COLS = ("obs", "obs_next", "act", "rew", "cost", "logp", "terminated", "truncated", "ptr", "len")
STATE = ("env_state", "obs_cur", "env_t", "ep_idx", "act_ctr", "active", "done_now", "ep_rew", "ep_len")
DASH = "HazardDash-v0"


def _register(name, task=None):
    from fsrl_b200 import envs
    path = envs.plugin_path(header(name), PLUGIN_DIR)
    assert os.path.exists(path), f"{path} is missing: build() builds the test env plugins"
    task = task or f"Plugin{name.title().replace('_', '')}-v0"
    envs.register_device_env(task, path)
    return task


def _h(t):
    return t.detach().cpu().numpy()


def _same_state(v0, v1):
    for k in STATE:
        assert np.array_equal(_h(getattr(v0, k)), _h(getattr(v1, k))), k


def _same_buffer(b0, b1):
    n0, n1 = buffer_to_numpy(b0), buffer_to_numpy(b1)
    for k in COLS:
        assert np.array_equal(n0[k], n1[k]), k


def _params(policy):
    return {k: _h(v) for k, v in policy.state_dict().items() if isinstance(v, torch.Tensor)}


def _same_params(p0, p1):
    assert p0.keys() == p1.keys()
    for k in p0:
        assert np.array_equal(p0[k], p1[k]), k


@pytest.mark.parametrize("name", sorted(SAME))
def test_same_struct_collects_are_bit_identical(name):
    """Train- and random-mode collects, inline (n_episode <= E) and resolve (n_episode > E): the ring, the env state
    with its noise counters, and the statistics."""
    task = _register(name)
    E = 6
    T = build_ppo(SAME[name], n_env=1)[1].max_episode_steps
    runs = [build_ppo(t, n_env=E, buffer_size=E * (T + 40)) for t in (SAME[name], task)]
    assert runs[1][1].kind >= 64 and runs[1][3].fused
    for n_episode, random in ((4, False), (4, True), (15, False), (9, True)):
        stats = [col.collect(n_episode=n_episode, random=random) for _, _, _, col in runs]
        assert stats[0] == stats[1], (n_episode, random)
        _same_buffer(runs[0][2], runs[1][2])
        _same_state(runs[0][1], runs[1][1])


@pytest.mark.parametrize("name", sorted(SAME))
def test_same_struct_step_and_reset_ids(name):
    from fsrl_b200.envs import DeviceVectorEnv
    from oracle.philox import action_uniform
    task = _register(name)
    E = 12
    venvs = [DeviceVectorEnv(t, E, seed=3) for t in (SAME[name], task)]
    outs = [v.reset() for v in venvs]
    assert torch.equal(outs[0][0], outs[1][0])
    n_done = 0
    for t in range(venvs[0].max_episode_steps + 30):
        a = action_uniform(9, np.arange(E), np.full(E, t, np.uint32), venvs[0].A)
        ids = None if t % 3 else np.arange(0, E, 2)
        act = a if ids is None else a[ids]
        outs = [v.step(act, ids) for v in venvs]
        for x, y in zip(outs[0][:4], outs[1][:4]):
            assert torch.equal(x, y), t
        assert torch.equal(outs[0][4].cost, outs[1][4].cost)
        done = (outs[0][2] | outs[0][3]).cpu().numpy()
        if done.any():
            env_id = np.arange(E) if ids is None else ids
            r = [v.reset(env_id[done]) for v in venvs]
            assert torch.equal(r[0][0], r[1][0])
            n_done += int(done.sum())
    assert n_done > 0
    _same_state(*venvs)


@pytest.mark.parametrize("name", sorted(SAME))
def test_same_struct_norm_obs_and_trajectory_harvest(name):
    from fsrl_b200.data import FastCollector, TrajectoryBuffer, VectorReplayBuffer
    from fsrl_b200.envs import VectorEnvNormObs
    task = _register(name)
    E = 5
    cols, tbs, norms = [], [], []
    for t in (SAME[name], task):
        policy, venv, buf, _ = build_ppo(t, n_env=E)
        norm = VectorEnvNormObs(venv)
        cols.append((FastCollector(policy, norm, buf, exploration_noise=True), buf))
        norms.append(norm)
        tb = TrajectoryBuffer()
        T = venv.max_episode_steps      # the harvest needs a ring longer than an episode
        policy2, venv2, buf2, _ = build_ppo(t, n_env=E, seed=21, buffer_size=E * (T + 100))
        tbs.append((FastCollector(policy2, venv2, buf2, exploration_noise=True, traj_buffer=tb), buf2, tb))
    for n_episode in (3, 8):
        s = [c.collect(n_episode=n_episode) for c, _ in cols]
        assert s[0] == s[1]
        _same_buffer(cols[0][1], cols[1][1])
        r0, r1 = (n.get_obs_rms() for n in norms)
        for k in ("mean", "var", "count"):
            assert np.array_equal(np.asarray(_h_any(getattr(r0, k))), np.asarray(_h_any(getattr(r1, k)))), k
        s = [c.collect(n_episode=n_episode) for c, _, _ in tbs]
        assert s[0] == s[1]
        _same_buffer(tbs[0][1], tbs[1][1])
    d0, d1 = (tb.get_all() for _, _, tb in tbs)
    assert len(d0) == len(d1) > 0
    for k in ("observations", "next_observations", "actions", "rewards", "costs", "terminals", "timeouts"):
        assert np.array_equal(_h_any(d0[k]), _h_any(d1[k])), k


def _h_any(x):
    return _h(x) if isinstance(x, torch.Tensor) else np.asarray(x)


@pytest.mark.parametrize("name", sorted(SAME))
def test_same_struct_training_is_bit_identical(name):
    """One PPOLagAgent.learn epoch and a few SAC-Lagrangian gradient steps end with the same parameters."""
    from fsrl_b200 import envs
    from fsrl_b200.agent import PPOLagAgent, SACLagAgent
    task = _register(name)
    kw = dict(epoch=1, testing_num=2, save_ckpt=False, verbose=False, show_progress=False)
    params = []
    for t in (SAME[name], task):
        agent = PPOLagAgent(envs.make(t), seed=4, hidden_sizes=(64, 64))
        agent.learn(envs.DeviceVectorEnv(t, 8, seed=5), envs.DeviceVectorEnv(t, 2, seed=6), episode_per_collect=8,
                    step_per_epoch=2 * 8 * 300, repeat_per_collect=2, buffer_size=8 * 1000, batch_size=256, **kw)
        params.append(_params(agent.policy))
    _same_params(*params)
    params = []
    for t in (SAME[name], task):
        agent = SACLagAgent(envs.make(t), seed=4, hidden_sizes=(64, 64))
        agent.learn(envs.DeviceVectorEnv(t, 4, seed=5), envs.DeviceVectorEnv(t, 2, seed=6), episode_per_collect=4,
                    step_per_epoch=20, update_per_step=0.25, buffer_size=4 * 1000, batch_size=64, **kw)
        params.append(_params(agent.policy))
    _same_params(*params)


# ---- HazardDash: an env the library does not have ---------------------------------------------------------------
@pytest.mark.parametrize("E,n_episode", [(16, 16), (16, 9), (6, 20)])
def test_new_env_random_collect_matches_twin(E, n_episode):
    from oracle import collector as ocol
    _register("hazard_dash", DASH)
    policy, venv, buf, col = build_ppo(DASH, n_env=E, buffer_size=E * 200 * 4)
    assert (venv.D, venv.A, venv.S) == (19, 3, 32)
    oenv = HazardDashTwin(E, venv.seed_value)
    assert np.array_equal(_h(venv.obs_cur), oenv.reset())
    ctr = _h(venv.act_ctr).astype(np.uint32)
    stats = col.collect(n_episode=n_episode, random=True)
    obuf = ocol.OracleBuffer(E * 200 * 4, E, venv.D, venv.A)
    ostats = ocol.collect(oenv, None, n_episode, policy._act_seed, ctr, obuf, mode="random",
                          action_bound=policy.action_bound_method or "none")
    for k in ("n/ep", "n/st", "terminated", "truncated", "total_cost", "len"):
        assert stats[k] == ostats[k], k
    assert stats["rew"] == pytest.approx(ostats["rew"], rel=1e-12, abs=1e-12)
    assert stats["terminated"] > 0 and stats["truncated"] > 0     # shares of the finished episodes
    b = buffer_to_numpy(buf)
    assert np.array_equal(b["ptr"], obuf.ptr) and np.array_equal(b["len"], obuf.len)
    for k in COLS[:-2]:
        assert np.array_equal(b[k], getattr(obuf, k)), k
    assert np.array_equal(_h(venv.act_ctr).astype(np.uint32), ctr)
    assert np.array_equal(_h(venv.env_state), oenv.st)


def test_new_env_step_and_reset_ids_match_twin():
    from fsrl_b200.envs import DeviceVectorEnv
    from oracle.philox import action_uniform
    _register("hazard_dash", DASH)
    E = 40
    venv = DeviceVectorEnv(DASH, E, seed=11)
    oenv = HazardDashTwin(E, 11)
    assert np.array_equal(_h(venv.reset()[0]), oenv.reset())
    n_term = n_trunc = 0
    for t in range(450):
        a = action_uniform(5, np.arange(E), np.full(E, t, np.uint32), 3)
        ids = None if t % 4 else np.arange(1, E, 3)
        act = a if ids is None else a[ids]
        obs, rew, term, trunc, info = venv.step(act, ids)
        oobs, orew, ocost, oterm, otrunc = oenv.step(act, ids)
        assert np.array_equal(_h(obs), oobs) and np.array_equal(_h(rew), orew), t
        assert np.array_equal(_h(info.cost), ocost) and np.array_equal(_h(term), oterm), t
        assert np.array_equal(_h(trunc), otrunc & ~oterm), t
        done = oterm | otrunc
        n_term += int(oterm.sum()); n_trunc += int((otrunc & ~oterm).sum())
        if done.any():
            env_id = (np.arange(E) if ids is None else ids)[done]
            assert np.array_equal(_h(venv.reset(env_id)[0]), oenv.reset(env_id))
    assert n_term > 0 and n_trunc > 0
    assert np.array_equal(_h(venv.env_state), oenv.st)


@pytest.mark.parametrize("agent_name", ["PPOLagAgent", "TRPOLagAgent", "CPOAgent", "FOCOPSAgent", "SACLagAgent",
                                        "DDPGLagAgent", "CVPOAgent"])
def test_every_agent_learns_on_new_env(agent_name):
    from fsrl_b200 import agent as agents
    from fsrl_b200 import envs
    from fsrl_b200.utils.logger import BaseLogger
    _register("hazard_dash", DASH)

    class Logged(BaseLogger):
        """BaseLogger that also keeps the last value of every key stored."""

        def __init__(self):
            super().__init__(None, log_txt=False, name="plugin")
            self.seen = {}

        def store(self, tab=None, **kwargs):
            super().store(tab, **kwargs)
            for k, v in kwargs.items():
                self.seen[f"{tab}/{k}" if tab else k] = v

        def store_many(self, tab, key, values):
            super().store_many(tab, key, values)
            self.seen[f"{tab}/{key}" if tab else key] = np.asarray(_h_any(values), dtype=np.float64)

    logger = Logged()
    cls = getattr(agents, agent_name)
    agent = cls(envs.make(DASH), logger, seed=3, hidden_sizes=(64, 64))
    kw = dict(epoch=1, testing_num=2, save_ckpt=False, verbose=False, show_progress=False)
    train, test = envs.DeviceVectorEnv(DASH, 8, seed=1), envs.DeviceVectorEnv(DASH, 2, seed=2)
    if isinstance(agent, agents.OffpolicyAgent):
        agent.learn(train, test, episode_per_collect=8, step_per_epoch=64, update_per_step=0.25, buffer_size=8000,
                    batch_size=64, **kw)
    else:
        agent.learn(train, test, episode_per_collect=8, step_per_epoch=1600, repeat_per_collect=2, buffer_size=8000,
                    batch_size=256, **kw)
    for k, v in _params(agent.policy).items():
        assert np.isfinite(v).all(), k
    stats = {k: v for k, v in logger.seen.items() if isinstance(v, (int, float, np.floating, np.ndarray))}
    assert any("loss" in k for k in stats) and any("rew" in k for k in stats), sorted(stats)
    assert all(np.isfinite(np.asarray(v, dtype=np.float64)).all() for v in stats.values()), stats


# ---- several plugins, refusals ----------------------------------------------------------------------------------
def test_two_plugins_in_one_process_do_not_interfere():
    from fsrl_b200.envs import DeviceVectorEnv, task_kind
    a, b = _register("hazard_dash", DASH), _register("car_circle")
    assert task_kind(a) != task_kind(b) and 64 <= min(task_kind(a), task_kind(b)) < 128
    venvs = {t: DeviceVectorEnv(t, 8, seed=4) for t in (a, b, "SafetyCarCircle-v0")}
    twin = HazardDashTwin(8, 4)
    twin.reset()
    for v in venvs.values():
        v.reset()
    for t in range(50):
        for name, v in venvs.items():
            act = np.full((8, v.A), 0.25 * ((t % 5) - 2), np.float32)
            out = v.step(act)
            if name == a:
                assert np.array_equal(_h(out[0]), twin.step(act)[0]), t
    _same_state(venvs[b], venvs["SafetyCarCircle-v0"])
    assert np.array_equal(_h(venvs[a].env_state), twin.st)


def test_refusals():
    from fsrl_b200 import _lib, envs
    import ctypes
    _register("hazard_dash", DASH)
    with pytest.raises(ValueError, match="no renderer"):
        envs.DeviceVectorEnv(DASH, 2, render_mode="rgb_array")
    # the C entry point refuses the kind as well
    v = envs.DeviceVectorEnv(DASH, 2)
    r = _lib.Rollout()
    v.fill(r)
    out = torch.empty((2, 16, 16, 3), dtype=torch.uint8, device="cuda")
    rc = _lib.lib.fsrl_env_render(ctypes.byref(r), None, 2, 16, 16, None, out.data_ptr(), None)
    assert rc == _lib.FSRL_EINVAL and "no renderer" in _lib.last_error()
    # a table of another ABI version
    _, table = envs._load_plugin(envs.PLUGINS[DASH].path)
    t = _lib.EnvPlugin.from_buffer_copy(table.contents)
    t.abi_version = _lib.lib.fsrl_abi_version() + 1
    kind = ctypes.c_int(-1)
    assert _lib.lib.fsrl_env_register(ctypes.byref(t), ctypes.byref(kind)) == _lib.FSRL_EINVAL
    assert "ABI version" in _lib.last_error() and kind.value == -1
    # a kind of the plugin range that nobody registered
    r.kind = 127
    with pytest.raises(ValueError, match="unknown env kind 127"):
        _lib.check(_lib.lib.fsrl_env_reset_all(ctypes.byref(r), None))
    with pytest.raises(ValueError, match="unknown env kind 127"):
        envs.env_dims(127)
