"""Offline datasets from host-stepped envs without a GPU: the collector's refusals and their messages, BasicCollector
turning a gymnasium-style env (or a one-env vector env) into a one-env HostVectorEnv, and the argument checks of
``fsrl_traj_copy_host`` (EINVAL before any device call)."""
import ctypes
import re

import numpy as np
import pytest


class _Spec:
    def __init__(self, id, T):
        self.id, self.max_episode_steps = id, T


class ToyEnv:
    """A gymnasium-style env (api 5) or a gym one (api 4, TimeLimit.truncated in info)."""

    def __init__(self, api=5, D=3, A=2, T=5):
        from fsrl_b200.spaces import Box
        self.api, self.D, self.T = api, D, T
        self.observation_space = Box(-np.inf, np.inf, (D,), np.float32)
        self.action_space = Box(-1.0, 1.0, (A,), np.float32)
        self.spec = _Spec("Toy-v0", T)
        self.t = 0

    def reset(self, seed=None, options=None):
        self.t = 0
        return np.zeros(self.D, np.float32), {}

    def step(self, a):
        self.t += 1
        trunc = self.T is not None and self.t >= self.T
        o = np.full(self.D, self.t, np.float32)
        if self.api == 5:
            return o, 1.0, False, trunc, {"cost": 0.0}
        return o, 1.0, trunc, {"cost": 0.0, "TimeLimit.truncated": trunc}


class FusedStub:
    """A policy the collector would run in the fused kernel (it brings its own fill_rollout); never called here."""
    device = "cuda"

    def fill_rollout(self, r, exploration_noise=False):
        raise AssertionError("no collect runs in these tests")


def _host(envs, device="cuda"):
    from fsrl_b200.envs import HostVectorEnv
    return HostVectorEnv._from_envs(envs, device=device)


# ---- refusals ---------------------------------------------------------------------------------------------------
def test_generic_path_policy_with_traj_buffer_is_refused():
    from fsrl_b200.data import FastCollector, TrajectoryBuffer
    with pytest.raises(NotImplementedError, match="traj_buffer") as ei:
        FastCollector(object(), _host([ToyEnv()]), traj_buffer=TrajectoryBuffer(10))
    assert "generic path" in str(ei.value)


def test_norm_obs_with_traj_buffer_is_refused():
    from fsrl_b200.data import FastCollector, TrajectoryBuffer
    from fsrl_b200.envs import VectorEnvNormObs
    venv = VectorEnvNormObs(_host([ToyEnv(), ToyEnv()], device="cpu"))
    with pytest.raises(NotImplementedError, match="traj_buffer with a VectorEnvNormObs env"):
        FastCollector(FusedStub(), venv, traj_buffer=TrajectoryBuffer(10))


@pytest.mark.parametrize("how", ["env_spec", "no_spec"])
def test_unknown_horizon_without_buffer_is_refused(how):
    from fsrl_b200.data import FastCollector, TrajectoryBuffer
    env = ToyEnv(T=None)
    if how == "no_spec":
        del env.spec
    venv = _host([env, ToyEnv(T=None)])
    assert venv.max_episode_steps is None
    with pytest.raises(ValueError, match="needs a buffer"):
        FastCollector(FusedStub(), venv, traj_buffer=TrajectoryBuffer(10))
    FastCollector(FusedStub(), venv)              # without a traj_buffer no ring is needed


def test_basic_collector_refuses_more_than_one_env():
    from fsrl_b200.data import BasicCollector

    from host_twin import TwinVectorEnv, twin
    with pytest.raises(TypeError, match="of 2 envs"):
        BasicCollector(FusedStub(), _host([ToyEnv(), ToyEnv()]))
    with pytest.raises(TypeError, match="of 3 envs"):
        BasicCollector(FusedStub(), TwinVectorEnv(twin("SafetyCarCircle-v0", 3, 0), "SafetyCarCircle-v0"))
    with pytest.raises(TypeError, match="one env"):
        BasicCollector(FusedStub(), object())


# ---- BasicCollector over host envs, no GPU touched ----------------------------------------------------------------
@pytest.mark.parametrize("api", [4, 5])
def test_basic_collector_wraps_a_gymnasium_env(api):
    from fsrl_b200.data import BasicCollector
    from fsrl_b200.envs import HostVectorEnv
    env = ToyEnv(api=api, D=4, A=3, T=7)
    bc = BasicCollector(FusedStub(), env)
    assert isinstance(bc.env, HostVectorEnv) and len(bc.env) == 1
    assert (bc.env.D, bc.env.A, bc.env.max_episode_steps) == (4, 3, 7)
    assert bc.env._envs == [env] and bc.env._dev is None          # no device state yet
    assert bc._fast.host and bc.buffer is None
    # the env as the collector sees it: one row, the protocol normalised
    obs, rew, term, trunc, cost = bc.env.step_envs(np.zeros((1, 3), np.float32))
    assert obs.shape == (1, 4) and rew.dtype == np.float64 and not term[0] and not trunc[0]


def test_basic_collector_takes_one_env_vector_envs():
    from fsrl_b200.data import BasicCollector
    from fsrl_b200.envs import HostVectorEnv

    from host_twin import TwinVectorEnv, twin
    venv = _host([ToyEnv()])
    assert BasicCollector(FusedStub(), venv).env is venv
    tv = TwinVectorEnv(twin("SafetyDroneRun-v0", 1, 0), "SafetyDroneRun-v0")
    bc = BasicCollector(FusedStub(), tv)
    assert isinstance(bc.env, HostVectorEnv) and bc.env._venv is tv and bc.env.max_episode_steps == 200


# ---- fsrl_traj_copy_host: argument checks -----------------------------------------------------------------------
def _copy_args(kind=-1, D=3, A=2, aD=3, aA=2, n_jobs=1, jobs_off=0, null=None, ring=True):
    from fsrl_b200 import _lib
    r = _lib.Rollout()
    r.kind, r.E, r.cap = kind, 2, 8
    if ring:
        for f in ("b_obs", "b_obs_next", "b_act", "b_rew", "b_cost", "b_term", "b_trunc", "b_ptr"):
            setattr(r, f, 1 << 20)
    a = _lib.TrajArena()
    for f in ("obs", "obs_next", "act", "rew", "cost", "term", "trunc"):
        setattr(a, f, None if f == null else 1 << 20)
    a.stride, a.n_slots, a.D, a.A = 8, 4, aD, aA
    return r, a, D, A, (1 << 20) + jobs_off, n_jobs


@pytest.mark.parametrize("case,msg", [
    (dict(kind=0), "host ring has env kind -1"), (dict(kind=3), "host ring has env kind -1"),
    (dict(D=0, aD=0), "bad dims"), (dict(D=0), "bad host ring dims"), (dict(A=0), "bad host ring dims"),
    (dict(A=9), "bad host ring dims"), (dict(D=5), "arena dims \\(3, 2\\) != env dims \\(5, 2\\)"),
    (dict(A=1), "arena dims \\(3, 2\\) != env dims \\(3, 1\\)"), (dict(ring=False), "no transition ring"),
    (dict(null="act"), "null pointer"), (dict(n_jobs=-1), "bad job list"), (dict(jobs_off=4), "16-byte aligned"),
])
def test_traj_copy_host_einval_before_the_device(case, msg):
    from fsrl_b200 import _lib
    r, a, D, A, jobs, n = _copy_args(**case)
    rc = _lib.lib.fsrl_traj_copy_host(ctypes.byref(r), ctypes.byref(a), D, A, jobs, n, None)
    assert rc == _lib.FSRL_EINVAL
    assert re.search(msg, _lib.last_error()), _lib.last_error()


def test_traj_copy_host_without_jobs_launches_nothing():
    from fsrl_b200 import _lib
    r, a, D, A, jobs, _ = _copy_args()
    assert _lib.lib.fsrl_traj_copy_host(ctypes.byref(r), ctypes.byref(a), D, A, jobs, 0, None) == _lib.FSRL_OK
    # the device form keeps refusing a host descriptor: its widths come from the env kind
    assert _lib.lib.fsrl_traj_copy(ctypes.byref(r), ctypes.byref(a), jobs, 0, None) == _lib.FSRL_EINVAL
    assert "unknown env kind -1" in _lib.last_error()


def test_traj_copy_host_is_bound_and_declared():
    import os

    from fsrl_b200 import _lib
    assert "fsrl_traj_copy_host" in _lib.SIGNATURES
    hdr = open(os.path.join(os.path.dirname(_lib.__file__), "..", "include", "fsrl_b200.h")).read()
    assert re.search(r"int fsrl_traj_copy_host\(const fsrl_rollout_t\* r, const fsrl_traj_arena_t\* a, int D, int A,",
                     hdr)
