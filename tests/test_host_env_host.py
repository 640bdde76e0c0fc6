"""Host-stepped envs without a GPU: the protocol normalisation of HostVectorEnv (step 4- / 5-tuples, the three
shapes of ``info``, ``reset`` with and without info), every limit it rejects, construction without a device, the
collector's refusals, and the argument checks of ``fsrl_host_collect_step`` (EINVAL before any device call)."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest


class _Spec:
    def __init__(self, id, T):
        self.id, self.max_episode_steps = id, T


class ToyEnv:
    """A deterministic numpy env: api 5 (gymnasium), 4 (gym with TimeLimit.truncated)."""

    def __init__(self, api=5, D=3, A=2, T=3, reset_info=True, cost=True, i=0):
        from fsrl_b200.spaces import Box
        self.api, self.D, self.A, self.T, self.reset_info, self.with_cost, self.i = api, D, A, T, reset_info, cost, i
        self.observation_space = Box(-np.inf, np.inf, (D,), np.float32)
        self.action_space = Box(-1.0, 1.0, (A,), np.float32)
        self.spec = _Spec("Toy-v0", T)
        self.t = 0
        self.seen = []

    def reset(self, seed=None, options=None):
        self.t = 0
        o = np.full(self.D, 10.0 * self.i, np.float32)
        return (o, {"i": self.i}) if self.reset_info else o

    def step(self, a):
        self.seen.append(np.asarray(a).copy())
        self.t += 1
        o = np.full(self.D, 10.0 * self.i + self.t, np.float32)
        rew = float(self.i + 0.5)
        term = self.i == 1 and self.t == 2
        trunc = self.t >= self.T
        info = {"cost": float(self.i)} if self.with_cost else {}
        if self.api == 5:
            return o, rew, term, trunc, info
        info["TimeLimit.truncated"] = trunc and not term
        return o, rew, term or trunc, info


def _host(envs):
    from fsrl_b200.envs import HostVectorEnv
    return HostVectorEnv([lambda e=e: e for e in envs])


@pytest.mark.parametrize("api", [4, 5])
@pytest.mark.parametrize("reset_info", [False, True])
def test_step_and_reset_normalised(api, reset_info):
    envs = [ToyEnv(api, reset_info=reset_info, i=i) for i in range(3)]
    venv = _host(envs)
    assert (len(venv), venv.D, venv.A, venv.spec.max_episode_steps) == (3, 3, 2, 3)
    obs = venv.reset_obs()
    assert obs.dtype == np.float32 and obs.shape == (3, 3) and obs[2, 0] == 20.0
    act = np.arange(4, dtype=np.float32).reshape(2, 2)
    for t in (1, 2):
        o, rew, term, trunc, cost = venv.step_envs(act, [0, 1])
        assert o.shape == (2, 3) and o[1, 0] == 10.0 + t
        assert rew.dtype == np.float64 and rew.tolist() == [0.5, 1.5]
        assert cost.tolist() == [0.0, 1.0]
        assert term.tolist() == [False, t == 2] and not trunc.any()
    assert np.array_equal(envs[1].seen[0], act[1])
    o, _, term, trunc, _ = venv.step_envs(act[:1], [0])
    assert trunc.tolist() == [True] and term.tolist() == [False]
    obs = venv.reset_obs([1])
    assert obs.shape == (1, 3) and obs[0, 0] == 10.0


def test_terminated_wins_over_truncated():
    """gymnasium's TimeLimit reports truncated on a terminal step at the horizon; the ring keeps terminated only."""
    from fsrl_b200.host_envs import normalize_step
    o = np.zeros((2, 1), np.float32)
    _, _, term, trunc, _ = normalize_step((o, [1, 2], [True, False], [True, True], {}), 2, 1)
    assert term.tolist() == [True, False] and trunc.tolist() == [False, True]


@pytest.mark.parametrize("shape", ["dict", "list", "batch", "absent"])
def test_cost_from_every_info_shape(shape):
    from fsrl_b200.data import Batch
    from fsrl_b200.host_envs import normalize_step
    c = np.array([0.0, 2.5, 1.0], np.float32)
    info = {"dict": {"cost": c}, "list": [{"cost": float(x)} for x in c], "batch": Batch(cost=c),
            "absent": [{} for _ in c]}[shape]
    o = np.zeros((3, 2), np.float32)
    _, _, _, _, cost = normalize_step((o, np.zeros(3), np.zeros(3, bool), np.zeros(3, bool), info), 3, 2)
    assert cost.dtype == np.float64
    assert cost.tolist() == ([0.0] * 3 if shape == "absent" else c.tolist())


def test_rewards_and_costs_are_not_rounded():
    """The collect statistics sum what the env reported (the reference accumulates the env's own dtype); only the
    ring rounds to float32."""
    from fsrl_b200.host_envs import normalize_step
    r = [0.1, 1.0 / 3.0]
    _, rew, _, _, cost = normalize_step((np.zeros((2, 1)), r, [False] * 2, [False] * 2, [{"cost": 0.7}, {}]), 2, 1)
    assert rew.tolist() == r and cost.tolist() == [0.7, 0.0]


@pytest.mark.parametrize("shape", ["dict", "list"])
def test_four_tuple_truncation_from_info(shape):
    from fsrl_b200.host_envs import normalize_step
    tl = [False, True, False]
    info = {"TimeLimit.truncated": np.array(tl)} if shape == "dict" else [{"TimeLimit.truncated": x} for x in tl]
    o = np.zeros((3, 1), np.float32)
    _, _, term, trunc, cost = normalize_step((o, np.zeros(3), np.array([True, True, False]), info), 3, 1)
    assert term.tolist() == [True, False, False] and trunc.tolist() == [False, True, False]
    assert not cost.any()


def test_vector_reset_with_and_without_info():
    from fsrl_b200.host_envs import normalize_reset
    o = np.ones((2, 3))
    for rval in (o, (o, [{}, {}]), (o, {"x": 1})):
        got = normalize_reset(rval, 2, 3)
        assert got.dtype == np.float32 and np.array_equal(got, o)


def test_from_vector_env_adopts_the_protocol():
    from fsrl_b200.envs import HostVectorEnv
    from fsrl_b200.spaces import Box

    class Vec:
        observation_space = [Box(-1, 1, (4,))] * 3
        action_space = [Box(-1, 1, (1,))] * 3
        spec = [_Spec("V", 7)] * 3

        def __len__(self):
            return 3

        def reset(self, id=None, **kw):
            n = 3 if id is None else len(id)
            self.kw = kw
            return np.zeros((n, 4)), [{}] * n

        def step(self, action, id=None):
            n = len(action)
            return np.ones((n, 4)), np.ones(n), np.zeros(n, bool), np.zeros(n, bool), [{"cost": 3.0}] * n

    v = Vec()
    venv = HostVectorEnv.from_vector_env(v)
    assert (len(venv), venv.D, venv.A, venv.max_episode_steps) == (3, 4, 1, 7)
    assert venv.reset_obs([0, 2], seed=4).shape == (2, 4) and v.kw == {"seed": 4}
    o, rew, term, trunc, cost = venv.step_envs(np.zeros((2, 1)), [1, 2])
    assert cost.tolist() == [3.0, 3.0]


def test_rejections_name_the_limit():
    from fsrl_b200.spaces import Box, Discrete

    class Env(ToyEnv):
        pass

    e = Env()
    e.action_space = Discrete(3)
    with pytest.raises(ValueError, match="Box action"):
        _host([e])
    e = Env()
    e.observation_space = Box(-1, 1, (2, 3))
    with pytest.raises(ValueError, match="flat"):
        _host([e])
    with pytest.raises(ValueError, match="same spaces"):
        _host([ToyEnv(D=3), ToyEnv(D=4)])
    with pytest.raises(ValueError, match="at most 8"):
        _host([ToyEnv(A=9)])
    with pytest.raises(ValueError, match="D \\+ A = 80"):
        _host([ToyEnv(D=75, A=6)])
    _host([ToyEnv(D=72, A=8)])                            # the widest admitted


def test_built_without_a_gpu():
    venv = _host([ToyEnv(i=i) for i in range(2)])
    assert venv._dev is None                              # nothing on a device until a collect step
    assert venv.device.type == "cuda" and venv.seed_value == 0


def test_collector_refusals():
    from fsrl_b200.data import FastCollector, TrajectoryBuffer
    venv = _host([ToyEnv()])
    with pytest.raises(NotImplementedError, match="traj_buffer"):
        FastCollector(object(), venv, traj_buffer=TrajectoryBuffer(10))
    with pytest.raises(NotImplementedError, match="generic path"):
        FastCollector(object(), venv)
    with pytest.raises(TypeError, match="vector-env protocol"):
        FastCollector(object(), object())


def test_compat_vector_class_builds_host_envs():
    from fsrl_b200.compat import _vector_env_class
    from fsrl_b200.envs import HostVectorEnv
    made = []

    def fn():
        made.append(ToyEnv())
        return made[-1]

    venv = _vector_env_class("DummyVectorEnv")([fn, fn, fn])
    assert isinstance(venv, HostVectorEnv) and len(venv) == 3 and len(made) == 3


# ---- the C entry ------------------------------------------------------------------------------------------------
def _descriptors(E=4, D=3, A=2, H=64, n_store=0, n_act=1, ids=(0,), head=0, out=None):
    from fsrl_b200 import _lib
    r = _lib.Rollout()
    r.E, r.head = E, head
    r.act_ctr = 1 << 20
    r.actor.in_, r.actor.H, r.actor.out = D, H, 2 * A if out is None else out
    for f in ("w1t", "b1", "w2t", "b2", "w3t", "b3"):
        setattr(r.actor, f, 1 << 20)
    r.log_sigma = 1 << 20
    pack = np.zeros(int(_lib.lib.fsrl_host_pack_bytes(D, n_store, n_act)) + 16, np.uint8)
    pack[:4 * len(ids)] = np.asarray(ids, np.int32).view(np.uint8)
    h = _lib.HostStep(D=D, A=A, n_store=n_store, n_act=n_act, parity=0, pack_host=pack.ctypes.data,
                      pack_dev=1 << 20, scratch=1 << 20, act_dev=1 << 20, act_host=1 << 20)
    return r, h, pack


def test_pack_size():
    from fsrl_b200 import _lib
    assert _lib.lib.fsrl_host_pack_bytes(5, 3, 4) == 4 * (3 + 4) + 4 * (4 * 5 + 3 * 5 + 2 * 3) + 2 * 3


@pytest.mark.parametrize("case,msg", [
    (dict(A=0), "action width"), (dict(A=9), "action width"), (dict(D=78, A=3), "D \\+ A"),
    (dict(H=96), "hidden width"), (dict(n_act=5), "outside \\[0, E"), (dict(ids=(4,)), "outside \\[0, E"),
    (dict(n_act=2, ids=(1, 1)), "listed twice"), (dict(n_store=1, n_act=0), "complete ring"),
    (dict(obs_dim=5), "actor input dim"), (dict(parity=2), "parity"), (dict(null="scratch"), "null pointer"),
    (dict(null="w2t"), "null actor weights"), (dict(head=1, out=2), "actor out dim"), (dict(out=1), "actor out dim"),
])
def test_host_step_einval_before_the_device(case, msg):
    from fsrl_b200 import _lib
    case = dict(case)
    null, parity, obs_dim = case.pop("null", None), case.pop("parity", 0), case.pop("obs_dim", None)
    r, h, pack = _descriptors(**case)
    if obs_dim is not None:            # an observation width the actor was not built for
        h.D = obs_dim
    h.parity = parity
    if null == "scratch":
        h.scratch = None
    elif null:
        setattr(r.actor, null, None)
    rc = _lib.lib.fsrl_host_collect_step(ctypes.byref(r), ctypes.byref(h), None)
    assert rc == _lib.FSRL_EINVAL
    import re
    assert re.search(msg, _lib.last_error()), _lib.last_error()


def test_host_step_abi_size_and_c99_header(tmp_path):
    from fsrl_b200 import _lib
    assert ctypes.sizeof(_lib.HostStep) == _lib.lib.fsrl_abi_sizeof(14) == 64
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "abi.c"
    src.write_text('#include <stdio.h>\n#include "fsrl_b200.h"\n'
                   'int main(void){ printf("%zu\\n", sizeof(fsrl_host_step_t)); return 0; }\n')
    exe = tmp_path / "abi"
    subprocess.check_call([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(root, "include"),
                           "-o", str(exe), str(src)])
    assert int(subprocess.check_output([str(exe)], text=True)) == _lib.lib.fsrl_abi_sizeof(14)
