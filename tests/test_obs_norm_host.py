"""VectorEnvNormObs without a GPU: the float64 restatement (tests/obs_norm_twin.py) against a direct numpy
statement of the update and the normalization, the wrapper's forwarding and sharing, the collector's refusals and
the EINVAL paths of the new entry points."""
import ctypes

import numpy as np
import pytest

from obs_norm_twin import EPS32, OracleNormObs, OracleObsRms
from oracle.envs_velocity import OracleVecEnvVel


def _direct(batches, D, clip=10.0):
    """mean / var / count after the batches, by the textbook parallel update, and the last batch normalized."""
    mean, var, count = np.zeros(D), np.ones(D), 0
    y = None
    for x in batches:
        x = np.asarray(x, np.float64)
        if len(x):
            n = len(x)
            bm, bv = x.mean(0), ((x - x.mean(0)) ** 2).mean(0)
            tot = count + n
            d = bm - mean
            mean, var = mean + d * n / tot, (var * count + bv * n + d * d * count * n / tot) / tot
            count = tot
        y = np.clip((x - mean) / np.sqrt(var + EPS32), -clip, clip).astype(np.float32)
    return mean, var, count, y


def test_oracle_rms_matches_direct_statement():
    rng = np.random.default_rng(0)
    batches = [rng.normal(3.0, 2.0, (n, 5)) for n in (1, 7, 0, 64, 3)]
    r = OracleObsRms(5)
    for x in batches:
        r.update(x)
        y = r.norm(x)
    mean, var, count, yd = _direct(batches, 5)
    assert r.count == count == 75
    np.testing.assert_allclose(r.mean, mean, rtol=1e-12)
    np.testing.assert_allclose(r.var, var, rtol=1e-12)
    assert np.array_equal(y, yd)


def test_empty_batch_is_not_an_update_and_clip_holds():
    r = OracleObsRms(3)
    r.update(np.zeros((0, 3)))
    assert r.count == 0 and np.array_equal(r.mean, np.zeros(3)) and np.array_equal(r.var, np.ones(3))
    r.update(np.array([[0.0, 0.0, 0.0], [1e-3, 0.0, 0.0]]))
    y = r.norm(np.array([[1e3, -1e3, 0.0]]))
    assert y[0, 0] == 10.0 and y[0, 1] == -10.0 and y[0, 2] == 0.0


def test_oracle_wrapper_updates_then_normalizes():
    inner = OracleVecEnvVel(34, 4, 3)               # Hopper velocity
    w = OracleNormObs(inner)
    o = w.reset()
    mean, var, count, y = _direct([inner.observe()], inner.D)
    assert w.rms.count == 4 and np.array_equal(o, y) and np.array_equal(w.observe(), y)
    a = np.zeros((2, inner.A), np.float32)
    raw0 = inner.observe()
    obs, *_ = w.step(a, [3, 1])
    raw = inner.observe([3, 1])
    _, _, count, y = _direct([raw0, raw], inner.D)
    assert w.rms.count == count == 6 and np.array_equal(obs, y)
    assert np.array_equal(w.observe([1]), y[1:2])
    frozen = OracleNormObs(OracleVecEnvVel(34, 4, 3), update=False, rms=w.rms)
    frozen.reset()
    assert w.rms.count == 6


def test_wrapper_forwards_and_shares_statistics():
    from fsrl_b200.envs import DeviceVectorEnv, ObsRunningMeanStd, VectorEnvNormObs
    venv = DeviceVectorEnv("SafetyPointButton1Gymnasium-v0", 3, device="cpu", seed=4)
    w = VectorEnvNormObs(venv)
    assert len(w) == 3 and w.D == 76 and w.A == venv.A and w.device == venv.device
    assert w.observation_space is venv.observation_space and w.action_space is venv.action_space
    assert w.spec is venv.spec and w.max_episode_steps == venv.max_episode_steps
    assert w.seed(9) == [9, 9, 9] and venv.seed_value == 9
    assert w.render() is None
    rms = w.get_obs_rms()
    assert isinstance(rms, ObsRunningMeanStd) and rms.count == 0
    assert np.array_equal(rms.mean, np.zeros(76)) and np.array_equal(rms.var, np.ones(76))
    t = VectorEnvNormObs(DeviceVectorEnv("SafetyPointButton1Gymnasium-v0", 2, device="cpu"), update_obs_rms=False)
    t.set_obs_rms(rms)
    assert t.get_obs_rms() is rms
    rms.copy_from(np.arange(76.0), np.full(76, 2.0), 5)
    assert t.get_obs_rms().count == 5                        # shared: the train env's updates reach the test env

    class Plain:
        mean, var, count = np.full(76, 1.5), np.full(76, 3.0), 11
    u = VectorEnvNormObs(DeviceVectorEnv("SafetyPointButton1Gymnasium-v0", 2, device="cpu"))
    u.set_obs_rms(Plain())
    assert u.get_obs_rms() is not rms and u.get_obs_rms().count == 11
    assert np.array_equal(u.get_obs_rms().var, np.full(76, 3.0))
    sd = u.get_obs_rms().state_dict()
    v = VectorEnvNormObs(DeviceVectorEnv("SafetyPointButton1Gymnasium-v0", 2, device="cpu"))
    v.get_obs_rms().load_state_dict(sd)
    assert v.get_obs_rms().count == 11 and np.array_equal(v.get_obs_rms().mean, sd["mean"])
    with pytest.raises(ValueError):
        VectorEnvNormObs(DeviceVectorEnv("SafetyCarCircle-v0", 2, device="cpu")).set_obs_rms(rms)
    with pytest.raises(TypeError):
        VectorEnvNormObs(w)
    with w.frozen():
        assert not w.update_obs_rms
    assert w.update_obs_rms


def test_wrapper_adopts_vector_protocol_objects_and_compat_exports_it():
    from fsrl_b200 import compat
    from fsrl_b200.envs import HostVectorEnv, VectorEnvNormObs
    from host_twin import TwinVectorEnv
    w = VectorEnvNormObs(TwinVectorEnv(OracleVecEnvVel(33, 2, 0), "SafetyHalfCheetahVelocityGymnasium-v1", 1000))
    assert isinstance(w.venv, HostVectorEnv) and w.D == 17 and w.A == 6
    compat.install()
    import tianshou.env
    assert tianshou.env.VectorEnvNormObs is VectorEnvNormObs


@pytest.mark.parametrize("first", ["fsrl_b200.obs_norm", "fsrl_b200.envs"])
def test_obs_norm_imports_in_either_order(first):
    """envs re-exports obs_norm's classes and obs_norm wraps envs' DeviceVectorEnv: a fresh interpreter can import
    either module first."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = (f"import {first}\nfrom fsrl_b200.obs_norm import ObsRunningMeanStd, VectorEnvNormObs\n"
            "from fsrl_b200 import envs\nassert envs.VectorEnvNormObs is VectorEnvNormObs\n"
            "assert envs.ObsRunningMeanStd is ObsRunningMeanStd\n")
    subprocess.run([sys.executable, "-c", code], cwd=root, check=True)


def test_agents_pass_the_wrapper_through():
    from fsrl_b200.agent.base_agent import _as_vector
    from fsrl_b200.envs import DeviceVectorEnv, VectorEnvNormObs
    w = VectorEnvNormObs(DeviceVectorEnv("SafetyCarCircle-v0", 2, device="cpu"))
    assert _as_vector(w, "cpu") is w


def test_collector_refusals():
    """traj_buffer= and a data-parallel policy are refused before the collector touches the env."""
    from fsrl_b200.data import FastCollector, TrajectoryBuffer
    from fsrl_b200.envs import DeviceVectorEnv, VectorEnvNormObs
    w = VectorEnvNormObs(DeviceVectorEnv("SafetyCarCircle-v0", 2, device="cpu"))

    class Policy:
        device = "cpu"
    with pytest.raises(NotImplementedError, match="normalized observations"):
        FastCollector(Policy(), w, traj_buffer=TrajectoryBuffer(10))
    p = Policy()
    p._dp = object()
    with pytest.raises(NotImplementedError, match="data parallelism"):
        FastCollector(p, w)


def test_entry_points_refuse_bad_arguments_without_gpu():
    from fsrl_b200 import _lib
    L = _lib.lib
    assert L.fsrl_obs_rms_work_bytes(0, 4) == 0 and L.fsrl_obs_rms_work_bytes(300, 17) > 300
    assert int(L.fsrl_abi_sizeof(15)) == ctypes.sizeof(_lib.ObsRms)
    fake = 1 << 20                                 # never dereferenced: every call below fails its checks first
    n = _lib.ObsRms(mean=fake, var=fake, count=fake, work=fake, D=17, update=1, clip_max=10.0, eps=1e-7)
    x = fake

    def rows(desc, E, ids, count, x=x):
        arr = None if ids is None else np.asarray(ids, np.int32)
        rc = L.fsrl_obs_rms_rows(None if desc is None else ctypes.byref(desc), x, E,
                                 None if arr is None else arr.ctypes.data, count, None, None, None)
        return rc, _lib.last_error()

    assert rows(None, 4, None, 4) == (_lib.FSRL_EINVAL, "fsrl_obs_rms_rows: null obs_rms descriptor")
    rc, msg = rows(n, 4, [0, 4], 2)
    assert rc == _lib.FSRL_EINVAL and "outside [0, E = 4)" in msg
    rc, msg = rows(n, 4, [1, 1], 2)
    assert rc == _lib.FSRL_EINVAL and "listed twice" in msg
    rc, msg = rows(n, 4, None, 3)
    assert rc == _lib.FSRL_EINVAL and "count must be E" in msg
    rc, msg = rows(n, 4, [0], 5)
    assert rc == _lib.FSRL_EINVAL and "outside [0, E = 4]" in msg
    rc, msg = rows(n, 4, [0], 1, x=None)
    assert rc == _lib.FSRL_EINVAL and "null observation" in msg
    bad = _lib.ObsRms(mean=fake, var=fake, count=fake, work=None, D=17, update=1, clip_max=10.0, eps=1e-7)
    rc, msg = rows(bad, 4, [0], 1)
    assert rc == _lib.FSRL_EINVAL and "null obs_rms pointer" in msg
    wide = _lib.ObsRms(mean=fake, var=fake, count=fake, work=fake, D=81, update=1, clip_max=10.0, eps=1e-7)
    rc, msg = rows(wide, 4, [0], 1)
    assert rc == _lib.FSRL_EINVAL and "outside [1, 80]" in msg
    # the collect entry: a rollout descriptor of HalfCheetah-velocity (D = 17) with a D = 11 descriptor
    from fsrl_b200.envs import DeviceVectorEnv
    venv = DeviceVectorEnv("SafetyHalfCheetahVelocityGymnasium-v1", 2, device="cpu")
    r = _lib.Rollout()
    venv.fill(r)
    r.mode = _lib.MODE_RANDOM
    n11 = _lib.ObsRms(mean=fake, var=fake, count=fake, work=fake, D=11, update=1, clip_max=10.0, eps=1e-7)
    assert L.fsrl_rollout_norm_steps(ctypes.byref(r), ctypes.byref(n11), 1, None, None) == _lib.FSRL_EINVAL
    assert "!= observation width 17" in _lib.last_error()
    assert L.fsrl_rollout_norm_steps(ctypes.byref(r), ctypes.byref(n), 2, fake, None) == _lib.FSRL_EINVAL
    assert "caller actions cover one step" in _lib.last_error()
    # the host step: a wrapped call checks the descriptor and n_fresh
    D, A, E = 17, 6, 2
    pack = np.zeros(int(L.fsrl_host_pack_norm_bytes(D, E, E, E)), np.uint8)
    h = _lib.HostStep(D=D, A=A, n_store=0, n_act=0, parity=0, pack_host=pack.ctypes.data, pack_dev=fake,
                      scratch=fake, act_dev=fake, act_host=fake)
    rh = _lib.Rollout()
    rh.E, rh.act_ctr, rh.mode = E, fake, _lib.MODE_RANDOM
    rh.actor.H = 64
    assert int(L.fsrl_abi_sizeof(16)) == ctypes.sizeof(_lib.HostNorm)

    def host(hn):
        return L.fsrl_host_collect_step_norm(ctypes.byref(rh), ctypes.byref(h), hn, None), _lib.last_error()

    rc, msg = host(None)
    assert rc == _lib.FSRL_EINVAL and "null normalization descriptor" in msg
    hn = _lib.HostNorm(obs_rms=ctypes.addressof(n11), obs_norm=fake, n_fresh=0)
    rc, msg = host(ctypes.byref(hn))
    assert rc == _lib.FSRL_EINVAL and "!= observation width 17" in msg
    hn.obs_rms, hn.n_fresh = ctypes.addressof(n), 3
    rc, msg = host(ctypes.byref(hn))
    assert rc == _lib.FSRL_EINVAL and "n_fresh = 3" in msg
    hn.n_fresh, hn.obs_norm = 1, None
    rc, msg = host(ctypes.byref(hn))
    assert rc == _lib.FSRL_EINVAL and "null obs_norm" in msg
    hn.obs_norm = fake
    off = int(L.fsrl_host_pack_norm_bytes(D, 0, 0, 0))
    pack[off:off + 4] = np.frombuffer(np.int32(7).tobytes(), np.uint8)
    rc, msg = host(ctypes.byref(hn))
    assert rc == _lib.FSRL_EINVAL and "fresh_ids[0] = 7" in msg
    # without a ring, store rows are refused unwrapped
    h.n_store = 1
    pack[:4] = 0
    assert L.fsrl_host_collect_step(ctypes.byref(rh), ctypes.byref(h), None) == _lib.FSRL_EINVAL
    assert "without a complete ring" in _lib.last_error()
