"""fsrl_rollout_steps with inline bookkeeping runs all its steps in one launch; against one launch per step
(FSRL_ROLLOUT_PER_STEP=1) everything the collect writes must be bit-identical: the ring, the env state, obs_cur,
the per-env bookkeeping and the integer counters.  The fp64 sums of rewards and costs are accumulated by atomics
whose order differs between runs anyway, so they are compared to a relative 1e-12.

Every env kind at H = 128 and 256 (and one at 64 and 512); every head in train and eval mode plus random mode
at E in {1, 17, 2048, 4096} and H = 128 and 256; collects cut short and run to the end, and the Drone tasks,
whose episodes terminate early.  With n_episode > E the resolve path must still take one launch per step and agree as well.
"""
import ctypes

import numpy as np
import pytest
import torch
from torch import nn

pytestmark = pytest.mark.gpu

TASKS = ["SafetyCarCircle-v0", "SafetyCarRun-v0", "SafetyBallCircle-v0", "SafetyBallRun-v0", "SafetyAntCircle-v0",
         "SafetyPointGoal1Gymnasium-v0", "SafetyAntRun-v0", "SafetyDroneCircle-v0", "SafetyDroneRun-v0",
         "SafetyPointCircle1Gymnasium-v0", "SafetyPointCircle2Gymnasium-v0", "SafetyCarCircle1Gymnasium-v0",
         "SafetyCarCircle2Gymnasium-v0", "SafetyPointGoal2Gymnasium-v0", "SafetyCarGoal1Gymnasium-v0",
         "SafetyCarGoal2Gymnasium-v0"]
STAT_INTS = ("step_count", "sum_ep_len", "episode_count", "n_episode", "n_ready", "term_count", "trunc_count",
             "finished", "finished_next")


class _Policy:
    """fill_rollout() for FastCollector: an arena actor with the head and mode under test"""

    def __init__(self, arena, slot, head, mode):
        self.arena, self.slot, self.head, self.mode = arena, slot, head, mode

    def fill_rollout(self, r, exploration_noise=False):
        from fsrl_b200 import _lib
        from fsrl_b200.nets import SIGMA_MAX, SIGMA_MIN
        r.actor = self.arena.mlp3(self.slot)
        r.head = {"indep": _lib.HEAD_GAUSS_INDEP, "cond": _lib.HEAD_GAUSS_COND, "cond_raw": _lib.HEAD_GAUSS_COND_RAW,
                  "det": _lib.HEAD_DETERMINISTIC}[self.head]
        r.mode = {"train": _lib.MODE_TRAIN, "eval": _lib.MODE_EVAL, "random": _lib.MODE_RANDOM}[self.mode]
        r.bounded = int(self.head != "cond_raw")
        r.action_bound = _lib.BOUND_CLIP
        r.action_scaling = 1
        r.max_action = 1.0
        r.expl_sigma = 0.3 if self.head == "det" else 0.0
        r.sigma_min, r.sigma_max = SIGMA_MIN, SIGMA_MAX
        r.tanh_eps = float(np.finfo(np.float32).eps)
        r.seed_act = 11
        r.log_sigma = self.arena.extra_ptr(self.slot)


def _actor(D, H, A, head, seed=0):
    from fsrl_b200.nets import Arena, NetSlot
    gen = torch.Generator().manual_seed(seed)

    def lin(i, o):
        m = nn.Linear(i, o)
        with torch.no_grad():
            m.weight.copy_(torch.randn(o, i, generator=gen) * (2.0 / i) ** 0.5)
            m.bias.copy_(0.1 * torch.randn(o, generator=gen))
        return m

    heads = [lin(H, A), lin(H, A)] if head in ("cond", "cond_raw") else [lin(H, A)]
    extra = nn.Parameter(-0.5 * torch.ones(A)) if head == "indep" else None
    slot = NetSlot("actor", None, lin(D, H), lin(H, H), heads, extra)
    return Arena([slot], "cuda"), slot


def _run(task, H, head, mode, E, n_episode, n_steps, per_step, monkeypatch):
    """collect_begin and n_steps fused steps on a fresh rig; returns everything the collect wrote"""
    from fsrl_b200 import _lib
    from fsrl_b200.data import FastCollector, VectorReplayBuffer
    from fsrl_b200.envs import DeviceVectorEnv
    if per_step:
        monkeypatch.setenv("FSRL_ROLLOUT_PER_STEP", "1")
    else:
        monkeypatch.delenv("FSRL_ROLLOUT_PER_STEP", raising=False)
    venv = DeviceVectorEnv(task, E, device="cuda", seed=3)
    buf = VectorReplayBuffer(E * venv.max_episode_steps, E, device="cuda")
    arena, slot = _actor(venv.D, H, venv.A, head, seed=H)
    col = FastCollector(_Policy(arena, slot, head, mode), venv, buf)
    col.reset_buffer()
    r = col._descriptor(mode == "random")
    r.inline_done = int(n_episode <= E)
    stream = torch.cuda.current_stream().cuda_stream
    _lib.check(_lib.lib.fsrl_collect_begin(ctypes.byref(r), n_episode, stream))
    l0 = int(_lib.lib.fsrl_launch_count())
    _lib.check(_lib.lib.fsrl_rollout_steps(ctypes.byref(r), n_steps, stream))
    launches = int(_lib.lib.fsrl_launch_count()) - l0
    torch.cuda.synchronize()
    st = venv.read_stats()
    out = {k: getattr(buf, k).clone() for k in ("obs", "obs_next", "act", "rew", "cost", "logp", "terminated",
                                                 "truncated", "ptr", "len")}
    out.update({k: getattr(venv, k).clone() for k in ("env_state", "obs_cur", "env_t", "ep_idx", "act_ctr", "active",
                                                       "done_now", "ep_rew", "ep_len")})
    out.update({k: int(getattr(st, k)) for k in STAT_INTS})
    return out, (float(st.sum_ep_rew), float(st.total_cost)), launches


def _compare(task, H, head, mode, E, n_episode, n_steps, monkeypatch):
    one, sums1, l1 = _run(task, H, head, mode, E, n_episode, n_steps, False, monkeypatch)
    ref, sums0, l0 = _run(task, H, head, mode, E, n_episode, n_steps, True, monkeypatch)
    case = f"{task} H={H} {head}/{mode} E={E} n_episode={n_episode} steps={n_steps}"
    assert l0 == 2 * n_steps, case
    assert l1 == (2 if n_episode <= E else 2 * n_steps), f"{case}: {l1} launches"
    for k, v in ref.items():
        w = one[k]
        if torch.is_tensor(v):
            same = v.shape == w.shape and bool((v.view(torch.uint8) == w.view(torch.uint8)).all())
        else:
            same = v == w
        assert same, f"{case}: {k} differs"
    for a, b in zip(sums1, sums0):
        assert abs(a - b) <= 1e-12 * max(abs(b), 1.0), f"{case}: fp64 sums {sums1} vs {sums0}"
    return ref


@pytest.mark.parametrize("task", TASKS)
@pytest.mark.parametrize("H", [128, 256])
def test_one_launch_every_env(task, H, monkeypatch):
    from fsrl_b200.envs import DeviceVectorEnv
    T = DeviceVectorEnv(task, 1, device="cuda").max_episode_steps
    ref = _compare(task, H, "indep", "train", 2048, 2048, T, monkeypatch)
    assert ref["finished"] == 1 and ref["episode_count"] == 2048
    _compare(task, H, "indep", "train", 17, 17, 41, monkeypatch)           # cut short: episodes still running


@pytest.mark.parametrize("head,mode", [("indep", "train"), ("indep", "eval"), ("cond", "train"), ("cond", "eval"),
                                       ("cond_raw", "train"), ("cond_raw", "eval"), ("det", "train"),
                                       ("det", "eval"), ("indep", "random")])
@pytest.mark.parametrize("E", [1, 17, 2048, 4096])
@pytest.mark.parametrize("H", [128, 256])
def test_one_launch_heads_and_sizes(H, head, mode, E, monkeypatch):
    _compare("SafetyCarCircle-v0", H, head, mode, E, E, 300, monkeypatch)


@pytest.mark.parametrize("H", [64, 512])
def test_one_launch_other_widths(H, monkeypatch):
    _compare("SafetyBallRun-v0", H, "indep", "train", 2048, 2048, 300, monkeypatch)


@pytest.mark.parametrize("task", ["SafetyDroneCircle-v0", "SafetyDroneRun-v0"])
def test_one_launch_early_terminations(task, monkeypatch):
    from fsrl_b200.envs import DeviceVectorEnv
    T = DeviceVectorEnv(task, 1, device="cuda").max_episode_steps
    ref = _compare(task, 256, "indep", "train", 4096, 3000, T, monkeypatch)
    assert ref["term_count"] > 0, "no episode terminated early: the case does not test terminations"


def test_resolve_path_keeps_per_step_launches(monkeypatch):
    _compare("SafetyCarCircle-v0", 256, "indep", "train", 64, 200, 500, monkeypatch)
