"""Host-stepped envs on the GPU (fsrl_b200/host_envs.py, csrc/rollout_host.cu).

The CPU env twins (oracle/envs_velocity.py takes every device kind) are bit-exact models of the device envs, so a
FastCollector over a HostVectorEnv of twins and one over the DeviceVectorEnv of the same task and seed must fill
identical rings: the host path runs the fused path's actor, sampling, noise stream, map_action and episode rules,
only the env step happens on the host.  Whole training runs must then end in bit-identical parameters.  User envs
that are no twin check the protocol normalisation, the costs in the ring and that every learner trains on them."""
import copy
import math

import numpy as np
import pytest
import torch

from helpers import buffer_to_numpy, build_ppo
from host_twin import host_twin

pytestmark = pytest.mark.gpu

CAR_CIRCLE, DRONE_CIRCLE = "SafetyCarCircle-v0", "SafetyDroneCircle-v0"
POINT_GOAL1, CHEETAH, CAR_BUTTON1 = ("SafetyPointGoal1Gymnasium-v0", "SafetyHalfCheetahVelocityGymnasium-v1",
                                     "SafetyCarButton1Gymnasium-v0")
COLS = ("obs", "obs_next", "act", "rew", "cost", "logp", "terminated", "truncated", "ptr", "len")


# ---- policies of every head ---------------------------------------------------------------------------------
def _policy(head, task, H):
    from fsrl_b200 import envs
    if head == "ppo":
        return build_ppo(task, hidden=(H, H))[0]
    from fsrl_b200.agent import CVPOAgent, DDPGLagAgent, SACLagAgent
    env = envs.make(task)
    cls = {"sac": SACLagAgent, "ddpg": DDPGLagAgent, "cvpo": CVPOAgent}[head]
    kw = dict(exploration_noise=0.3) if head == "ddpg" else {}
    return cls(env, seed=3, hidden_sizes=(H, H), **kw).policy


def _collect(policy, venv, mode, n_episode, cap, store=True, rounds=2):
    from fsrl_b200.data import FastCollector, VectorReplayBuffer
    E = len(venv)
    buf = VectorReplayBuffer(E * cap, E) if store else None
    col = FastCollector(policy, venv, buf, exploration_noise=True)
    policy.eval() if mode == "eval" else policy.train()
    stats = [col.collect(n_episode=n_episode, random=(mode == "random")) for _ in range(rounds)]
    torch.cuda.synchronize()
    ring = buffer_to_numpy(buf) if store else None
    return stats, ring, venv.act_ctr.cpu().numpy().copy()


def _assert_stats_equal(sd, sh):
    for a, b in zip(sd, sh):
        for k in ("n/ep", "n/st", "terminated", "truncated"):
            assert a[k] == b[k], k
        for k in ("rew", "len", "cost", "total_cost"):
            assert b[k] == pytest.approx(a[k], rel=1e-12, abs=1e-12), k


CASES = [
    # task, H, head, mode, n_episode as a multiple of E ("half", "one", "surplus" = 3E + 1), per-env host envs
    (CAR_CIRCLE, 64, "ppo", "train", "half", True),
    (CAR_CIRCLE, 256, "sac", "train", "surplus", False),
    (CAR_CIRCLE, 64, "ddpg", "train", "one", False),
    (DRONE_CIRCLE, 64, "ppo", "train", "surplus", False),
    (DRONE_CIRCLE, 256, "cvpo", "eval", "one", False),
    (DRONE_CIRCLE, 64, "sac", "random", "half", False),
    (POINT_GOAL1, 64, "sac", "random", "surplus", False),
    (POINT_GOAL1, 512, "ppo", "train", "one", False),
    (CHEETAH, 256, "ddpg", "train", "half", False),
    (CHEETAH, 64, "cvpo", "train", "surplus", True),
    (CAR_BUTTON1, 64, "ppo", "eval", "surplus", False),
    (CAR_BUTTON1, 256, "sac", "train", "one", False),
]


@pytest.mark.parametrize("task,H,head,mode,n_ep,per_env", CASES)
def test_host_twin_matches_device_bitwise(task, H, head, mode, n_ep, per_env):
    from fsrl_b200.envs import DeviceVectorEnv
    E, seed = 6, 21
    n_episode = {"half": E // 2, "one": E, "surplus": 3 * E + 1}[n_ep]
    policy = _policy(head, task, H)
    T = DeviceVectorEnv(task, 1).max_episode_steps
    cap = T * (n_episode // E + 2)          # two collects; the second one wraps the ring on the surplus cases
    sd, rd, cd = _collect(policy, DeviceVectorEnv(task, E, seed=seed), mode, n_episode, cap)
    sh, rh, ch = _collect(policy, host_twin(task, E, seed, per_env), mode, n_episode, cap)
    _assert_stats_equal(sd, sh)
    for k in COLS:
        assert np.array_equal(rd[k], rh[k]), k
    assert np.array_equal(cd, ch)
    assert rd["len"].sum() > 0
    if mode != "eval":
        assert ch.sum() > 0


@pytest.mark.parametrize("task", [DRONE_CIRCLE, CHEETAH])
def test_host_twin_without_buffer_matches_device(task):
    """evaluate()'s collect stores nothing; the statistics and the noise counters still match."""
    from fsrl_b200.envs import DeviceVectorEnv
    E = 5
    policy = _policy("ppo", task, 64)
    sd, _, cd = _collect(policy, DeviceVectorEnv(task, E, seed=4), "train", 2 * E + 1, 0, store=False)
    sh, _, ch = _collect(policy, host_twin(task, E, 4), "train", 2 * E + 1, 0, store=False)
    _assert_stats_equal(sd, sh)
    assert np.array_equal(cd, ch)


def test_second_collector_continues_the_noise_stream():
    """act_ctr lives with the envs: a second collector over the same host envs continues the stream, as on the
    device."""
    from fsrl_b200.data import FastCollector, VectorReplayBuffer
    from fsrl_b200.envs import DeviceVectorEnv
    E, task = 4, CAR_CIRCLE
    policy = _policy("ppo", task, 64)
    T = DeviceVectorEnv(task, 1).max_episode_steps
    out = []
    for venv in (DeviceVectorEnv(task, E, seed=9), host_twin(task, E, 9)):
        FastCollector(policy, venv, exploration_noise=True).collect(n_episode=E)
        buf = VectorReplayBuffer(E * T, E)
        FastCollector(policy, venv, buf, exploration_noise=True).collect(n_episode=E)
        out.append((buffer_to_numpy(buf), venv.act_ctr.cpu().numpy()))
    for k in COLS:
        assert np.array_equal(out[0][0][k], out[1][0][k]), k
    assert np.array_equal(out[0][1], out[1][1]) and out[0][1].min() == 2 * T


# ---- pinned to the reference ----------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["E4_n4", "E4_n9", "E3_n7", "E5_n2", "E2_n1", "E4_n11_term41", "E5_n13_term29",
                                  "E3_n5_term41", "E6_n4_term17"])
def test_host_collect_replays_reference_fast_collector(golden_dir, case):
    """The reference's own FastCollector runs (collector_golden.npz: a deterministic eval-mode H = 16 Gaussian actor on
    the SafetyBallRun-v0 twin; the *_term cases add scripted terminations at different times per env) replayed
    through a HostVectorEnv: episode counting, the surplus rule and the reset order of the host loop against the
    reference itself, with the tolerances of test_oracle_golden.py's replay (the reward's is explained below).  The
    ring's rewards are also checked to be exactly the ones the env reported.  The H = 16 actor is zero-padded to
    H = 64: the extra hidden units are ReLU(0) = 0 and add nothing to the head."""
    from host_twin import TwinVectorEnv
    from test_oracle_golden import _load_policy_golden

    from fsrl_b200.data import FastCollector, VectorReplayBuffer
    from fsrl_b200.envs import HostVectorEnv
    from oracle.envs import OracleVecEnv
    from oracle.trainer_scenario import TerminatingEnv
    g = _load_policy_golden(golden_dir, "collector_golden.npz")[case]
    E, n_ep, period = (int(g["data"][k]) for k in ("E", "n_episode", "period"))
    want = g["final"]
    inner = TerminatingEnv("ball_run", E, 77, period) if period else OracleVecEnv("ball_run", E, 77)
    seen = [[] for _ in range(E)]              # every reward the env reported, per env, in step order

    class Recording(TwinVectorEnv):
        def step(self, action, id=None):
            out = super().step(action, id)
            for e, r in zip(np.arange(E) if id is None else id, out[1]):
                seen[e].append(r)
            return out
    venv = HostVectorEnv.from_vector_env(Recording(inner))
    policy = build_ppo("SafetyBallRun-v0", hidden=(64, 64), n_env=1)[0]
    sd = policy.state_dict()
    for k, v in g["init"].items():
        pad = torch.zeros_like(sd[k])
        pad[tuple(slice(0, n) for n in v.shape)] = torch.from_numpy(v).to(pad.device)
        sd[k] = pad
    policy.load_state_dict(sd)
    policy.eval()
    buf = VectorReplayBuffer(E * 100 * 4, E)
    col = FastCollector(policy, venv, buf)
    st = col.collect(n_episode=n_ep)
    torch.cuda.synchronize()
    got = np.array([st[k] for k in ("n/ep", "n/st", "rew", "len", "total_cost", "cost", "truncated", "terminated")])
    np.testing.assert_allclose(got, want["stats"], rtol=1e-6, atol=1e-9)
    assert int(want["collect_episode"]) == n_ep == col.collect_episode and int(want["collect_step"]) == col.collect_step
    b = buffer_to_numpy(buf)
    np.testing.assert_array_equal(b["ptr"], want["ptr"])
    np.testing.assert_array_equal(b["len"], want["len"])
    for k in ("terminated", "truncated"):
        np.testing.assert_array_equal(b[k], want[k].astype(bool), err_msg=k)
    for k in ("obs", "obs_next", "act", "cost"):
        np.testing.assert_allclose(b[k].reshape(want[k].shape), want[k], rtol=1e-6, atol=1e-6, err_msg=k)
    # The ring holds exactly the rewards the env reported ...
    cap = len(b["rew"]) // E
    for e in range(E):
        assert np.array_equal(b["rew"][e * cap:e * cap + len(seen[e])], np.asarray(seen[e], np.float32)), e
    # ... and BallRun's reward is 40 (x' - x): a difference of two positions.  The actor runs on the tensor cores
    # (3xTF32, ~1e-7 relative), the reference's on the CPU in fp32; actions and observations agree to 1e-6 above,
    # and the cancellation turns a position difference of one float32 ulp (4.8e-7 for positions in [4, 8)) into 40
    # such ulps of the reward.  The bound allows 80 (one ulp in each of the two positions).
    np.testing.assert_allclose(b["rew"], want["rew"], rtol=1e-6, atol=80 * np.spacing(np.float32(4.0)), err_msg="rew")
    if period:
        assert want["terminated"].any()


# ---- whole training runs ------------------------------------------------------------------------------------
def _strip(d):
    """The logged statistics without the wall-clock ones."""
    return {k: v for k, v in d.items() if not any(w in k for w in ("time", "speed", "duration"))}


@pytest.mark.parametrize("H,batch", [(64, 512), (256, 256)])
def test_ppo_lag_learn_on_host_twin_is_bitwise_device(H, batch):
    """H = 64 updates through the kernel chain, H = 256 with batch 256 through the persistent launch."""
    from fsrl_b200 import envs
    from fsrl_b200.agent import PPOLagAgent
    from fsrl_b200.envs import DeviceVectorEnv
    task, E = CAR_CIRCLE, 8
    runs = []
    for host in (False, True):
        agent = PPOLagAgent(envs.make(task), seed=5, hidden_sizes=(H, H))
        mk = (lambda n, s: host_twin(task, n, s)) if host else (lambda n, s: DeviceVectorEnv(task, n, seed=s))
        epoch, stat, info = agent.learn(mk(E, 11), mk(2, 12), epoch=2, episode_per_collect=E, step_per_epoch=2 * E * 500,
                                        repeat_per_collect=2, buffer_size=E * 1000, testing_num=2, batch_size=batch,
                                        save_ckpt=False, verbose=False, show_progress=False)
        torch.cuda.synchronize()
        runs.append((copy.deepcopy(agent.state_dict), _strip(stat), _strip(info), epoch))
    (sd0, st0, in0, ep0), (sd1, st1, in1, ep1) = runs
    assert ep0 == ep1 == 2
    assert sd0.keys() == sd1.keys()
    for k in sd0:
        a, b = sd0[k], sd1[k]
        if isinstance(a, torch.Tensor):
            assert torch.equal(a.cpu(), b.cpu()), k
    assert st0 == st1
    assert in0 == in1


# ---- user envs that are not twins ---------------------------------------------------------------------------
class UserEnv:
    """A small numpy env with a cost, gymnasium's 5-tuple API (api=5) or gym's 4-tuple with TimeLimit.truncated."""

    def __init__(self, api=5, T=40, seed=0):
        from fsrl_b200.envs import _Spec
        from fsrl_b200.spaces import Box
        self.api, self.T = api, T
        self.observation_space = Box(-np.inf, np.inf, (5,), np.float32)
        self.action_space = Box(-2.0, 2.0, (2,), np.float32)
        self.spec = _Spec("UserEnv-v0", T)
        self.rng = np.random.default_rng(seed)
        self.costs = []

    def reset(self, seed=None, options=None):
        self.x = self.rng.normal(size=5).astype(np.float32)
        self.t = 0
        return (self.x.copy(), {}) if self.api == 5 else self.x.copy()

    def step(self, a):
        a = np.asarray(a, np.float32)
        self.t += 1
        drive = np.concatenate([a, a, a[:1]]).astype(np.float32)
        self.x = (np.float32(0.9) * self.x + np.float32(0.2) * drive).astype(np.float32)
        rew = float(1.0 - np.sum(self.x * self.x) * 0.1)
        cost = float(abs(self.x[0]) > 0.8)
        self.costs.append(cost)
        term = bool(np.abs(self.x).max() > 4.0)
        trunc = self.t >= self.T and not term
        if self.api == 5:
            return self.x.copy(), rew, term, trunc, {"cost": cost}
        return self.x.copy(), rew, term or trunc, {"cost": cost, "TimeLimit.truncated": trunc}


@pytest.mark.parametrize("api", [4, 5])
def test_user_env_costs_land_in_the_ring(api):
    from fsrl_b200.data import FastCollector, VectorReplayBuffer
    from fsrl_b200.envs import HostVectorEnv
    E = 4
    made = [UserEnv(api, seed=i) for i in range(E)]
    venv = HostVectorEnv([lambda e=e: e for e in made])
    policy = _policy_for_user("ppo").policy
    buf = VectorReplayBuffer(E * 200, E)
    col = FastCollector(policy, venv, buf, exploration_noise=True)
    stats = col.collect(n_episode=E)
    ring = buffer_to_numpy(buf)
    assert stats["n/st"] == int(ring["len"].sum())
    total = 0.0
    for e in range(E):
        n = int(ring["len"][e])
        assert np.array_equal(ring["cost"][e * 200:e * 200 + n], np.asarray(made[e].costs[:n], np.float32))
        total += sum(made[e].costs[:n])
    assert stats["total_cost"] == pytest.approx(total) and total > 0


def _policy_for_user(algo, **kw):
    from fsrl_b200.agent import CPOAgent, CVPOAgent, DDPGLagAgent, PPOLagAgent, SACLagAgent
    cls = dict(ppo=PPOLagAgent, sac=SACLagAgent, ddpg=DDPGLagAgent, cpo=CPOAgent, cvpo=CVPOAgent)[algo]
    return cls(UserEnv(), seed=1, hidden_sizes=(64, 64), **kw)


def _finite(x):
    if isinstance(x, torch.Tensor):
        return bool(torch.isfinite(x).all())
    if isinstance(x, (float, int, np.floating)):
        return math.isfinite(float(x))
    return True


@pytest.mark.parametrize("algo", ["sac", "ddpg", "cpo", "cvpo"])
@pytest.mark.parametrize("api", [4, 5])
def test_learners_train_on_user_envs(algo, api):
    from fsrl_b200.envs import HostVectorEnv
    agent = _policy_for_user(algo)
    train = HostVectorEnv([lambda i=i: UserEnv(api, seed=i) for i in range(4)])
    test = HostVectorEnv([lambda i=i: UserEnv(api, seed=10 + i) for i in range(2)])
    kw = dict(epoch=1, episode_per_collect=4, step_per_epoch=400, buffer_size=4000, testing_num=2, batch_size=64,
              save_ckpt=False, verbose=False, show_progress=False)
    if algo in ("sac", "ddpg", "cvpo"):
        kw["update_per_step"] = 0.1
    epoch, stat, info = agent.learn(train, test, **kw)
    assert epoch == 1
    for k, v in list(stat.items()) + list(info.items()):
        assert _finite(v), k
    for k, v in agent.state_dict.items():
        assert _finite(v), k
    rew, length, cost = agent.evaluate(test, eval_episodes=2)
    assert math.isfinite(rew) and length > 0 and math.isfinite(cost)


def test_host_env_example_trains():
    import importlib.util
    import os
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples", "train_host_env.py")
    spec = importlib.util.spec_from_file_location("train_host_env", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    epoch, rew, cost = mod.main(["--epoch", "1", "--training_num", "4", "--step_per_epoch", "1000"])
    assert epoch == 1 and math.isfinite(rew) and math.isfinite(cost)


def test_compat_dummy_vector_env_trains_on_user_envs():
    import fsrl_b200.compat
    fsrl_b200.compat.install()
    from tianshou.env import DummyVectorEnv

    from fsrl_b200.envs import HostVectorEnv
    train = DummyVectorEnv([lambda i=i: UserEnv(5, seed=i) for i in range(4)])
    assert isinstance(train, HostVectorEnv) and len(train) == 4
    agent = _policy_for_user("ppo")
    epoch, stat, info = agent.learn(train, DummyVectorEnv([lambda: UserEnv(4, seed=9)]), epoch=1, episode_per_collect=4,
                                    step_per_epoch=200, repeat_per_collect=1, buffer_size=2000, testing_num=1,
                                    batch_size=64, save_ckpt=False, verbose=False, show_progress=False)
    assert epoch == 1
    for k, v in agent.state_dict.items():
        assert _finite(v), k
