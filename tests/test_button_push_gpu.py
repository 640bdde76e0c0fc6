"""The Safety-Gymnasium Button and Push tasks on the device, and the learners' paths at their 76-wide
observations.

The env battery of test_nav_envs_gpu.py runs over the eight tasks against the CPU twin that takes them
(oracle/envs_button_push.py): resets, random-mode collects against the oracle collector on the inline and the
resolve path, train-mode rings replayed through the twin, ``step`` / ``reset(id)`` on id subsets and the
trajectory harvest.  The Button tasks regenerate their whole layout from the reset's Philox stream inside
step and observe, so every comparison of them also checks that the device and the twin key it alike.

The one-launch collect is compared with one launch per step as test_rollout_one_launch_gpu.py does; the MLP
engine is checked against float64 at inputs wider than 64 (obs + act = 78 is the critic input of the
off-policy learners here); the critic pass is compared with its 16-row kernel at D = 76; and
examples/train_agent.py trains every learner end to end on one of the tasks."""
import ctypes

import pytest
import torch

import test_engine_gpu as eng
import test_mlp_forward_rows_gpu as rows
import test_nav_envs_gpu as nav
import test_rollout_one_launch_gpu as one
from oracle.envs_button_push import OracleVecEnvBP

pytestmark = pytest.mark.gpu
TASKS = ["SafetyPointButton1Gymnasium-v0", "SafetyPointButton2Gymnasium-v0", "SafetyCarButton1Gymnasium-v0",
         "SafetyCarButton2Gymnasium-v0", "SafetyPointPush1Gymnasium-v0", "SafetyPointPush2Gymnasium-v0",
         "SafetyCarPush1Gymnasium-v0", "SafetyCarPush2Gymnasium-v0"]


@pytest.fixture
def bp_twin(monkeypatch):
    """The battery of test_nav_envs_gpu.py builds its twin from oracle.envs_nav.OracleVecEnvNav: point that name at
    the subclass that also takes kinds 24-31 for the duration of a test."""
    import oracle.envs_nav
    monkeypatch.setattr(oracle.envs_nav, "OracleVecEnvNav", OracleVecEnvBP)


@pytest.mark.parametrize("task", TASKS)
def test_env_reset_matches_twin_bitwise(task, bp_twin):
    nav.test_env_reset_matches_twin_bitwise(task)


@pytest.mark.parametrize("task", TASKS)
@pytest.mark.parametrize("E,n_episode", [(16, 16), (6, 14)])
def test_random_collect_matches_oracle_bitwise(task, E, n_episode, bp_twin):
    nav.test_random_collect_matches_oracle_bitwise(task, E, n_episode)


@pytest.mark.parametrize("task", TASKS)
@pytest.mark.parametrize("E,n_episode", [(8, 8), (5, 7)])
def test_train_collect_replays_through_twin(task, E, n_episode, bp_twin):
    nav.test_train_collect_replays_through_twin(task, E, n_episode)


@pytest.mark.parametrize("task", TASKS)
def test_step_and_reset_ids_match_twin(task, bp_twin):
    nav.test_step_and_reset_ids_match_twin(task)


@pytest.mark.parametrize("task", ["SafetyCarButton2Gymnasium-v0", "SafetyPointPush1Gymnasium-v0"])
@pytest.mark.parametrize("E,n_episode", [(6, 6), (4, 7)])
def test_trajectory_harvest_matches_ring(task, E, n_episode):
    nav.test_trajectory_harvest_matches_ring(task, E, n_episode)


@pytest.mark.parametrize("task", TASKS)
@pytest.mark.parametrize("H", [128, 256])
def test_one_launch_every_new_env(task, H, monkeypatch):
    ref = one._compare(task, H, "indep", "train", 2048, 2048, 1000, monkeypatch)
    assert ref["finished"] == 1 and ref["episode_count"] == 2048
    one._compare(task, H, "indep", "train", 17, 17, 41, monkeypatch)            # cut short: episodes still running


@pytest.mark.parametrize("H", [64, 512])
def test_one_launch_other_widths(H, monkeypatch):
    one._compare("SafetyCarPush2Gymnasium-v0", H, "indep", "train", 2048, 2048, 1000, monkeypatch)


@pytest.mark.parametrize("H,D,heads,B,mode", [
    (64, 65, ((1, 0), (3, 3)), 1000, "plain"),
    (128, 78, ((1, 0), (1, 0)), 4097, "critic"),     # the SAC / DDPG critic input of these tasks, past the row split
    (256, 80, ((16, 0), (8, 8)), 300, "gather"),
    (512, 78, ((3, 3), (1, 0)), 600, "critic"),
    (256, 76, ((4, 4), (2, 2)), 257, "gather"),      # an actor on these tasks
])
def test_engine_wide_inputs_match_float64(H, D, heads, B, mode):
    eng.test_forward_backward_wgrad_match_float64(H, D, heads, B, mode)


def test_engine_rejects_inputs_wider_than_the_dx_stride():
    from fsrl_b200.engine import DX_LD
    with pytest.raises(ValueError, match=f"input dim {DX_LD + 1} unsupported"):
        eng.Rig(64, [(DX_LD + 1, 1, 0)], bmax=4, seed=1)


@pytest.mark.parametrize("H", [128, 256])
@pytest.mark.parametrize("out", [1, 2])
def test_critic_pass_at_76_wide_inputs(H, out, monkeypatch):
    for n_rows in (65, 132 * 64 + 1, 2048 * 40):
        rows._check(H, 76, out, n_rows, n_rows % 2 == 1, monkeypatch, seed=n_rows)


def test_ppo_takes_the_chain_on_76_wide_observations():
    """The persistent PPO launch admits D <= 40: at the shape where test_nav_envs_gpu.py sees it admit a Circle task
    (H = 256, batch 256), a Button task's update runs the three-launch chain."""
    from fsrl_b200 import _lib
    from test_ppo_scale_gpu import _collect, _sub_batch
    policy, batch, _, _, _ = _collect("SafetyPointButton1Gymnasium-v0", (256, 256), 16, 0.3)
    sub = _sub_batch(policy, batch, 4 * 256)
    policy._ensure_update_state(256, sub.n, 1)
    u = policy._descriptor(sub, torch.zeros(sub.n, dtype=torch.int32, device="cuda"))
    assert u.D == 76 and _lib.lib.fsrl_ppo_persist_active(ctypes.byref(u), sub.n, 256) == 0


@pytest.mark.parametrize("algo,task,extra", [
    ("ppol", "SafetyPointButton1Gymnasium-v0", ["--repeat_per_collect", "2", "--batch_size", "256"]),
    ("cpo", "SafetyCarButton2Gymnasium-v0", []),
    ("focops", "SafetyPointButton2Gymnasium-v0", []),
    ("sacl", "SafetyPointPush1Gymnasium-v0", ["--update_per_step", "0.05"]),
    ("ddpgl", "SafetyCarPush2Gymnasium-v0", ["--update_per_step", "0.05"]),
    ("cvpo", "SafetyCarPush1Gymnasium-v0", ["--update_per_step", "0.05"]),
])
def test_agents_train_on_button_and_push(algo, task, extra, tmp_path):
    nav.test_agents_train_on_new_tasks_through_reference_imports(algo, task, extra, tmp_path)
