"""fsrl_env_render on the device against the float32 twin of tests/render_twin.py: every task bit for bit after resets,
steps and terminations, with and without the last cost; frame sizes and id subsets; read-only on the env; the
observation-normalizing wrapper; and examples/render_agent.py end to end."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import render_twin as rt
from fsrl_b200.envs import KINDS

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TERMINATING = {"SafetyDroneCircle-v0", "SafetyDroneRun-v0", "SafetyHopperVelocityGymnasium-v1",
               "SafetyWalker2dVelocityGymnasium-v1"}
FAMILY_TASKS = ["SafetyCarCircle-v0", "SafetyBallRun-v0", "SafetyPointButton2Gymnasium-v0",
                "SafetyWalker2dVelocityGymnasium-v1", "SafetyAntVelocityGymnasium-v1"]


def _venv(task, E, seed=7, size=(48, 64), mode="rgb_array"):
    from fsrl_b200.envs import DeviceVectorEnv
    return DeviceVectorEnv(task, E, device="cuda", seed=seed, render_mode=mode, render_size=size)


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


def _twin(venv, ids=None, last_cost=None):
    h, w = venv.render_size
    lc = None if last_cost is None else last_cost.cpu().numpy()
    return rt.render(venv.kind, venv.env_state.cpu().numpy(), venv.env_t.cpu().numpy(), venv.ep_idx.cpu().numpy(),
                     venv.seed_value, h, w, ids=ids, last_cost=lc)


def _check(venv, where):
    got = venv.render()
    assert got.dtype == torch.uint8 and got.is_cuda and got.is_contiguous()
    assert tuple(got.shape) == (venv.env_num,) + venv.render_size + (3,)
    want = _twin(venv, last_cost=venv.last_cost)
    bad = np.argwhere((got.cpu().numpy() != want).any(-1))
    assert len(bad) == 0, f"{venv.task} {where}: {len(bad)} pixels differ, first {bad[:3].tolist()}"
    np.testing.assert_array_equal(_raw(venv), _twin(venv), err_msg=f"{venv.task} {where}: without last_cost")


def _policy(task, A, rng, E):
    if task in ("SafetyHopperVelocityGymnasium-v1", "SafetyWalker2dVelocityGymnasium-v1"):
        return np.zeros((E, A), np.float32)            # holding the joints still topples the torso
    return rng.uniform(-1, 1, (E, A)).astype(np.float32)


@pytest.mark.parametrize("task", sorted(KINDS))
def test_every_task_matches_the_twin(task):
    E = 5
    venv = _venv(task, E)
    venv.reset()
    _check(venv, "after reset")
    rng = np.random.default_rng(3)
    terms, shown_terminal = 0, False
    for block in range(4):
        for t in range(40):
            _, _, term, trunc, info = venv.step(_policy(task, venv.A, rng, E))
            done = (term | trunc).cpu().numpy()
            terms += int(term.sum())
            if done.any():
                if term.any() and not shown_terminal:     # the terminal pose, before its reset
                    _check(venv, f"at a termination, block {block} step {t}")
                    shown_terminal = True
                venv.reset(np.nonzero(done)[0])
        _check(venv, f"after block {block}")
    if task in TERMINATING:
        assert terms > 0 and shown_terminal, task


@pytest.mark.parametrize("task", FAMILY_TASKS)
@pytest.mark.parametrize("size", [(16, 16), (64, 200), (256, 256), (1024, 1024)])
def test_sizes_and_id_subsets(task, size):
    E = 4
    venv = _venv(task, E, size=size)
    venv.reset()
    rng = np.random.default_rng(5)
    for _ in range(25):
        venv.step(rng.uniform(-1, 1, (E, venv.A)).astype(np.float32))
    full = venv.render()
    ids = [0, 3] if size[0] == 1024 else None
    np.testing.assert_array_equal(full.cpu().numpy()[ids] if ids else full.cpu().numpy(),
                                  _twin(venv, ids=ids, last_cost=venv.last_cost))
    sub = venv.render(id=[3, 0])
    assert torch.equal(sub, full[[3, 0]])
    dup = venv.render(id=np.array([2, 2, 1]))
    assert torch.equal(dup, full[[2, 2, 1]])


def test_more_ctas_than_one_wave():
    venv = _venv("SafetyPointGoal2Gymnasium-v0", 300, size=(64, 64))
    venv.reset()
    rng = np.random.default_rng(9)
    for _ in range(10):
        venv.step(rng.uniform(-1, 1, (300, venv.A)).astype(np.float32))
    np.testing.assert_array_equal(venv.render().cpu().numpy(), _twin(venv, last_cost=venv.last_cost))


@pytest.mark.parametrize("task", ["SafetyCarButton2Gymnasium-v0", "SafetyDroneRun-v0"])
def test_rendering_is_read_only(task):
    E = 6
    runs = []
    for mode in (None, "rgb_array"):
        venv = _venv(task, E, seed=11, mode=mode)
        rng = np.random.default_rng(2)
        venv.reset()
        outs = []
        for t in range(60):
            out = venv.step(rng.uniform(-1, 1, (E, venv.A)).astype(np.float32))
            if mode is not None:
                venv.render()
                venv.render(id=[1, 1, 4])
            outs.append([x.cpu().numpy() for x in out[:4]] + [out[4].cost.cpu().numpy()])
            done = (out[2] | out[3]).cpu().numpy()
            if done.any():
                venv.reset(np.nonzero(done)[0])
        torch.cuda.synchronize()
        runs.append((outs, [getattr(venv, f).cpu().numpy() for f in ("env_state", "env_t", "ep_idx", "act_ctr",
                                                                       "obs_cur", "stats")]))
    (o0, s0), (o1, s1) = runs
    for a, b in zip(o0, o1):
        for x, y in zip(a, b):
            np.testing.assert_array_equal(x, y)
    for x, y in zip(s0, s1):
        np.testing.assert_array_equal(x, y)


def test_wrapped_env_renders_the_raw_state():
    from fsrl_b200.envs import VectorEnvNormObs
    venv = _venv("SafetyPointPush2Gymnasium-v0", 4)
    wrapped = VectorEnvNormObs(venv)
    wrapped.reset()
    rng = np.random.default_rng(4)
    for _ in range(15):
        wrapped.step(rng.uniform(-1, 1, (4, venv.A)).astype(np.float32))
    rms = wrapped.get_obs_rms()
    before = (rms.mean, rms.var, rms.count)
    frames = wrapped.render()
    assert torch.equal(frames, venv.render())
    assert torch.equal(wrapped.render(id=[2]), frames[[2]])
    after = (rms.mean, rms.var, rms.count)
    np.testing.assert_array_equal(before[0], after[0])
    np.testing.assert_array_equal(before[1], after[1])
    assert before[2] == after[2]
    np.testing.assert_array_equal(frames.cpu().numpy(), _twin(venv, last_cost=venv.last_cost))


def _has_pil():
    try:
        import PIL  # noqa: F401
        return True
    except ImportError:
        return False


@pytest.mark.parametrize("task", ["SafetyCarCircle-v0", "SafetyDroneRun-v0", "SafetyPointButton2Gymnasium-v0",
                                  "SafetyHopperVelocityGymnasium-v1", "SafetyAntVelocityGymnasium-v1"])
def test_example_writes_one_frame_per_vector_step(task, tmp_path):
    out = tmp_path / "clip"
    fmt = "gif" if _has_pil() else "npz"
    res = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "render_agent.py"), "--task", task,
                          "--envs", "2", "--size", "32", "48", "--out", str(out), "--format", fmt, "--max_steps", "60",
                          "--fps", "20"],
                         capture_output=True, text=True, cwd=str(tmp_path), timeout=600)
    assert res.returncode == 0, res.stdout + res.stderr
    steps = int([ln for ln in res.stdout.splitlines() if ln.startswith("frames:")][0].split()[1])
    assert 1 <= steps <= 60
    if fmt == "gif":
        from PIL import Image
        with Image.open(str(out) + ".gif") as im:
            # PIL merges identical consecutive frames into one longer frame: one frame per step in time
            assert 1 <= im.n_frames <= steps and im.size == (2 * 48, 32)
            total = 0
            for k in range(im.n_frames):
                im.seek(k)
                total += im.info["duration"]
            assert total == steps * 50, (total, steps)
    else:
        frames = np.load(str(out) + ".npz")["frames"]
        assert frames.shape == (steps, 2, 32, 48, 3) and frames.dtype == np.uint8
    assert "return" in res.stdout and "cost" in res.stdout
