"""Rendering user-defined device envs (plugins whose struct defines draw) on the device.

- The drawn Car Circle plugin (tests/envs_render/car_circle_drawn.h) renders bit-identical frames to the built-in
  SafetyCarCircle-v0 in lockstep: the library and the plugin instantiate the same rasterizer.
- The drawn HazardDash plugin matches its float32 twin (tests/render_plugin_twin.py) bit for bit through resets,
  steps, each of its terminations and reset(id); crowded.h checks the default window and the primitive cap.
- Rendering is read-only, VectorEnvNormObs renders the raw state, several renderers coexist with an undrawn plugin,
  a draw leaves training bit-identical, and examples/render_agent.py renders a plugin end to end.

The plugins are built by build() into PLUGIN_DIR; these tests only load them."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import render_plugin_twin as rpt
from env_plugin_twin import ARENA, GOAL_R, PLUGIN_DIR, HazardDashTwin
from env_plugin_twin import header as env_header
from helpers import buffer_to_numpy, build_ppo

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAR = "PluginCarCircleDrawn-v0"
DASH_DRAWN, DASH = "HazardDashDrawn-v0", "HazardDash-v0"
CROWDED = "PluginCrowded-v0"
STATE = ("env_state", "obs_cur", "env_t", "ep_idx", "act_ctr", "active", "done_now", "ep_rew", "ep_len", "stats")


def _register(task, header):
    from fsrl_b200 import envs
    path = envs.plugin_path(header, PLUGIN_DIR)
    assert os.path.exists(path), f"{path} is missing: build() builds the test env plugins"
    envs.register_device_env(task, path)
    return task


def _car():
    return _register(CAR, rpt.header("car_circle_drawn"))


def _dash_drawn():
    return _register(DASH_DRAWN, rpt.header("hazard_dash_drawn"))


def _dash():
    return _register(DASH, env_header("hazard_dash"))


def _crowded():
    return _register(CROWDED, rpt.header("crowded"))


def _venv(task, E, seed=7, size=(48, 64), mode="rgb_array"):
    from fsrl_b200.envs import DeviceVectorEnv
    return DeviceVectorEnv(task, E, device="cuda", seed=seed, render_mode=mode, render_size=size)


def _h(t):
    return t.detach().cpu().numpy()


def _raw(venv, ids=None, last_cost=None):
    """fsrl_env_render called directly (last_cost may be None, which render() never passes)."""
    from fsrl_b200 import _lib
    n = venv.env_num if ids is None else len(ids)
    h, w = venv.render_size
    out = torch.empty((n, h, w, 3), dtype=torch.uint8, device="cuda")
    r = _lib.Rollout()
    venv.fill(r)
    p = None if ids is None else np.asarray(ids, np.int32)
    _lib.check(_lib.lib.fsrl_env_render(ctypes.byref(r), None if p is None else p.ctypes.data, n, h, w,
                                        None if last_cost is None else last_cost.data_ptr(), out.data_ptr(),
                                        torch.cuda.current_stream().cuda_stream))
    return out.cpu().numpy()


def _same_frames(v0, v1, where):
    np.testing.assert_array_equal(_h(v0.render()), _h(v1.render()), err_msg=where)
    np.testing.assert_array_equal(_raw(v0), _raw(v1), err_msg=f"{where}: without last_cost")
    ids = [3, 0, 3, 1]
    np.testing.assert_array_equal(_h(v0.render(id=ids)), _h(v1.render(id=ids)), err_msg=f"{where}: ids {ids}")


@pytest.mark.parametrize("size", [(48, 64), (256, 256)])
def test_drawn_car_circle_is_bit_identical_to_the_built_in(size):
    task = _car()
    E = 6
    venvs = [_venv(t, E, seed=3, size=size) for t in ("SafetyCarCircle-v0", task)]
    for v in venvs:
        v.reset()
    _same_frames(*venvs, "after reset")
    rng = np.random.default_rng(1)
    for t in range(120):
        act = rng.uniform(-1, 1, (E, 2)).astype(np.float32)
        ids = None if t % 3 else np.array([5, 1, 2])
        outs = [v.step(act if ids is None else act[ids], ids) for v in venvs]
        assert torch.equal(outs[0][4].cost, outs[1][4].cost)
        if t % 10 == 0:
            _same_frames(*venvs, f"step {t}")
        if t % 25 == 24:
            for v in venvs:
                v.reset(np.array([0, 4]))
            _same_frames(*venvs, f"after reset(id) at step {t}")
    assert torch.equal(venvs[0].last_cost, venvs[1].last_cost)
    _same_frames(*venvs, "end")
    # the cost colour (random actions seldom leave the band |x| <= XLIM): forced on every other env of both
    lc = torch.tensor([1.0, 0.0] * (E // 2), device="cuda")
    for v in venvs:
        v.last_cost.copy_(lc)
    _same_frames(*venvs, "with last_cost")
    cost_rgb = np.array([240, 60, 40], np.uint8)
    assert (_h(venvs[1].render())[::2] == cost_rgb).all(-1).any(axis=(1, 2)).all()


def _dash_actions(twin, t):
    """Three groups of four envs: 0-3 steer to the goal, 4-7 run for the +x wall, 8-11 burn energy in place."""
    E = twin.E
    a = np.zeros((E, 3), np.float32)
    st = twin.st
    g = np.clip(2.0 * (st[4:6, :4] - st[0:2, :4]) - 2.0 * st[2:4, :4], -1, 1).T
    a[:4, :2] = g
    a[4:8, 0], a[4:8, 2] = 1.0, 1.0
    sgn = 1.0 if t % 2 else -1.0
    a[8:, 0], a[8:, 1], a[8:, 2] = sgn, -sgn, 1.0
    return a


def test_drawn_hazard_dash_matches_the_twin():
    task = _dash_drawn()
    E, size = 12, (64, 80)
    venv = _venv(task, E, seed=5, size=size)
    twin = HazardDashTwin(E, 5)
    T = HazardDashTwin.T

    def check(where, ids=None):
        assert np.array_equal(_h(venv.env_state), twin.st) and np.array_equal(_h(venv.env_t), twin.t), where
        lc = _h(venv.last_cost)
        got = _h(venv.render(id=ids))
        want = rpt.render(rpt.hazard_dash_draw, T, twin.st, twin.t, *size, ids=ids, last_cost=lc)
        bad = np.argwhere((got != want).any(-1))
        assert len(bad) == 0, f"{where}: {len(bad)} pixels differ, first {bad[:3].tolist()}"
        np.testing.assert_array_equal(_raw(venv, ids), rpt.render(rpt.hazard_dash_draw, T, twin.st, twin.t, *size,
                                                                  ids=ids), err_msg=f"{where}: without last_cost")
        return got

    venv.reset()
    twin.reset()
    check("after reset")
    seen = {"goal": 0, "energy": 0, "arena": 0}
    cost_rgb = np.array([240, 60, 40], np.uint8)
    for t in range(300):
        act = _dash_actions(twin, t)
        _, _, term, trunc, info = venv.step(act)
        _, _, ocost, oterm, otrunc = twin.step(act)
        assert np.array_equal(_h(info.cost), ocost) and np.array_equal(_h(term), oterm), t
        if oterm.any():
            st = twin.st
            d = np.sqrt((st[4] - st[0]) ** 2 + (st[5] - st[1]) ** 2)
            kinds = {"goal": d < GOAL_R, "energy": st[6] <= 0,
                     "arena": (np.abs(st[0]) > ARENA) | (np.abs(st[1]) > ARENA)}
            for k, m in kinds.items():
                seen[k] += int((m & oterm).sum())
            check(f"at a termination, step {t}")              # the terminal state, before its reset
        elif t % 7 == 0:
            check(f"step {t}")
        done = oterm | otrunc
        if done.any():
            ids = np.nonzero(done)[0]
            venv.reset(ids)
            twin.reset(ids)
            check(f"after reset(id) at step {t}", ids=np.concatenate([ids, ids[:1]]))
    assert all(v > 0 for v in seen.values()), seen
    lc = np.zeros(E, np.float32)
    lc[::2] = 1.0                      # the cost colour, forced on every other env
    venv.last_cost.copy_(torch.from_numpy(lc))
    got = check("forced cost")
    assert (got[::2] == cost_rgb).all(-1).any(axis=(1, 2)).all()


def test_crowded_default_window_and_cap():
    task = _crowded()
    E = 5
    venv = _venv(task, E, seed=2, size=(96, 96))
    venv.reset()
    rng = np.random.default_rng(8)
    for t in range(12):
        venv.step(rng.uniform(-1, 1, (E, 1)).astype(np.float32))
        want = rpt.render(rpt.crowded_draw, 20, _h(venv.env_state), _h(venv.env_t), 96, 96,
                          last_cost=_h(venv.last_cost))
        np.testing.assert_array_equal(_h(venv.render()), want, err_msg=f"step {t}")


def test_rendering_is_read_only_and_wrapper_renders_raw_state():
    from fsrl_b200.envs import VectorEnvNormObs
    task = _dash_drawn()
    E = 6
    venv = _venv(task, E, seed=9)
    venv.reset()
    rng = np.random.default_rng(6)
    for _ in range(20):
        venv.step(rng.uniform(-1, 1, (E, 3)).astype(np.float32))
    torch.cuda.synchronize()
    before = {k: _h(getattr(venv, k)).copy() for k in STATE + ("last_cost",)}
    venv.render()
    venv.render(id=[2, 2, 5])
    torch.cuda.synchronize()
    for k, v in before.items():
        assert np.array_equal(_h(getattr(venv, k)), v), k
    wvenv = _venv(task, 4, seed=4)
    wrapped = VectorEnvNormObs(wvenv)
    wrapped.reset()
    for _ in range(15):
        wrapped.step(rng.uniform(-1, 1, (4, 3)).astype(np.float32))
    frames = wrapped.render()
    assert torch.equal(frames, wvenv.render())
    assert torch.equal(wrapped.render(id=[1]), frames[[1]])
    np.testing.assert_array_equal(_h(frames), rpt.render(rpt.hazard_dash_draw, HazardDashTwin.T,
                                                         _h(wvenv.env_state), _h(wvenv.env_t), *wvenv.render_size,
                                                         last_cost=_h(wvenv.last_cost)))


def test_two_renderers_and_an_undrawn_plugin_in_one_process():
    from fsrl_b200.envs import PLUGINS, task_kind
    car, dash_drawn, dash = _car(), _dash_drawn(), _dash()
    assert len({task_kind(t) for t in (car, dash_drawn, dash)}) == 3
    assert PLUGINS[car].renders and PLUGINS[dash_drawn].renders and not PLUGINS[dash].renders
    with pytest.raises(ValueError, match="no renderer"):
        _venv(dash, 2)
    E = 4
    builtin, vcar, vdash = _venv("SafetyCarCircle-v0", E, seed=1), _venv(car, E, seed=1), _venv(dash_drawn, E, seed=1)
    for v in (builtin, vcar, vdash):
        v.reset()
    rng = np.random.default_rng(0)
    for t in range(30):
        a2, a3 = rng.uniform(-1, 1, (E, 2)).astype(np.float32), rng.uniform(-1, 1, (E, 3)).astype(np.float32)
        builtin.step(a2)
        vcar.step(a2)
        vdash.step(a3)
    np.testing.assert_array_equal(_h(vcar.render()), _h(builtin.render()))
    np.testing.assert_array_equal(_h(vdash.render()), rpt.render(rpt.hazard_dash_draw, HazardDashTwin.T,
                                                                 _h(vdash.env_state), _h(vdash.env_t),
                                                                 *vdash.render_size, last_cost=_h(vdash.last_cost)))
    assert not np.array_equal(_h(vcar.render())[:, :, :, 0], _h(vdash.render())[:, :, :, 0])


def test_draw_does_not_touch_training():
    """Collects and a PPO-Lagrangian epoch of the drawn HazardDash are bit-identical to the undrawn plugin's."""
    from fsrl_b200 import envs
    from fsrl_b200.agent import PPOLagAgent
    tasks = (_dash(), _dash_drawn())
    E = 8
    runs = [build_ppo(t, n_env=E, buffer_size=E * 400) for t in tasks]
    for n_episode, random in ((8, False), (5, True), (17, False)):
        stats = [col.collect(n_episode=n_episode, random=random) for _, _, _, col in runs]
        assert stats[0] == stats[1], (n_episode, random)
        b0, b1 = buffer_to_numpy(runs[0][2]), buffer_to_numpy(runs[1][2])
        for k in ("obs", "obs_next", "act", "rew", "cost", "logp", "terminated", "truncated", "ptr", "len"):
            assert np.array_equal(b0[k], b1[k]), k
        for k in STATE:
            assert np.array_equal(_h(getattr(runs[0][1], k)), _h(getattr(runs[1][1], k))), k
    params = []
    kw = dict(epoch=1, testing_num=2, save_ckpt=False, verbose=False, show_progress=False)
    for t in tasks:
        agent = PPOLagAgent(envs.make(t), seed=4, hidden_sizes=(64, 64))
        agent.learn(envs.DeviceVectorEnv(t, 8, seed=5), envs.DeviceVectorEnv(t, 2, seed=6), episode_per_collect=8,
                    step_per_epoch=1600, repeat_per_collect=2, buffer_size=8000, batch_size=256, **kw)
        params.append({k: _h(v) for k, v in agent.policy.state_dict().items() if isinstance(v, torch.Tensor)})
    assert params[0].keys() == params[1].keys()
    for k in params[0]:
        assert np.array_equal(params[0][k], params[1][k]), k


def test_example_renders_a_plugin(tmp_path):
    """examples/render_agent.py --header: builds (here: finds in the cache) the plugin, registers it and writes one
    frame per vector step; the first frame is the twin's after the agent's first deterministic action."""
    out = tmp_path / "clip"
    E, H, W = 2, 32, 48
    res = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "render_agent.py"),
                          "--header", rpt.header("hazard_dash_drawn"), "--plugin_dir", PLUGIN_DIR,
                          "--task_name", "ExampleDash-v0", "--envs", str(E), "--size", str(H), str(W),
                          "--out", str(out), "--format", "npz", "--max_steps", "40", "--seed", "0"],
                         capture_output=True, text=True, cwd=str(tmp_path), timeout=600)
    assert res.returncode == 0, res.stdout + res.stderr
    steps = int([ln for ln in res.stdout.splitlines() if ln.startswith("frames:")][0].split()[1])
    assert 1 <= steps <= 40
    frames = np.load(str(out) + ".npz")["frames"]
    assert frames.shape == (steps, E, H, W, 3) and frames.dtype == np.uint8
    # the example's first step, restated: its agent, seed and deterministic policy, on the twin
    sys.path.insert(0, os.path.join(ROOT, "examples"))
    import render_agent
    from fsrl_b200 import envs
    from fsrl_b200.data import Batch
    task = _dash_drawn()
    agent = render_agent.ALGOS["ppol"](env=envs.make(task), hidden_sizes=(128, 128), seed=0)
    policy = agent.policy
    policy.eval()
    venv = _venv(task, E, seed=0, size=(H, W))
    obs, _ = venv.reset()
    twin = HazardDashTwin(E, 0)
    assert np.array_equal(twin.reset(), _h(obs))
    with torch.no_grad():
        act = policy(Batch(obs=obs)).act
    act = policy.map_action(act.cpu().numpy() if isinstance(act, torch.Tensor) else np.asarray(act))
    _, _, cost, _, _ = twin.step(np.asarray(act, np.float32))
    want = rpt.render(rpt.hazard_dash_draw, HazardDashTwin.T, twin.st, twin.t, H, W, last_cost=cost)
    np.testing.assert_array_equal(frames[0], want)
