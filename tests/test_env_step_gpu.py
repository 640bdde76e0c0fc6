"""The gym protocol of the device envs (DeviceVectorEnv.step / reset(id)) and FastCollector's generic path for
policies the rollout kernel cannot run, against the CPU env twin (oracle/envs_flight.py) and the oracle collector.

Env-range actions come from the Philox uniform stream on the host, and the generic-path policies are exact fp32
functions of the observation, so every comparison is bit for bit."""
import math

import numpy as np
import pytest
import torch

from helpers import buffer_to_numpy, build_ppo

pytestmark = pytest.mark.gpu
TASKS = ["SafetyCarCircle-v0", "SafetyCarRun-v0", "SafetyBallCircle-v0", "SafetyBallRun-v0", "SafetyAntCircle-v0",
         "SafetyPointGoal1Gymnasium-v0", "SafetyAntRun-v0", "SafetyDroneCircle-v0", "SafetyDroneRun-v0"]
DRONES = ["SafetyDroneCircle-v0", "SafetyDroneRun-v0"]
COLS = ("obs", "obs_next", "act", "rew", "cost", "logp", "terminated", "truncated")
STATE = ("env_state", "obs_cur", "env_t", "ep_idx", "act_ctr", "active", "done_now", "ep_rew", "ep_len")


def _venv(task, E, seed=5):
    from fsrl_b200.envs import DeviceVectorEnv
    return DeviceVectorEnv(task, E, device="cuda", seed=seed)


def _twin(venv):
    from oracle.envs_flight import OracleVecEnvExt
    return OracleVecEnvExt(venv.kind, venv.env_num, venv.seed_value)


def _h(t):
    return t.detach().cpu().numpy()


def _actions(ids, t, A, seed=77):
    from oracle.philox import action_uniform
    ids = np.asarray(ids)
    return action_uniform(seed, ids, np.full(len(ids), t, np.uint32), A)


def _check_step(out, ref, what):
    obs, rew, term, trunc, info = out
    oobs, orew, ocost, oterm, otrunc = ref
    assert np.array_equal(_h(obs), oobs), what
    assert np.array_equal(_h(rew), orew) and np.array_equal(_h(info.cost), ocost), what
    assert np.array_equal(_h(term), oterm) and np.array_equal(_h(trunc), otrunc & ~oterm), what
    assert term.dtype == torch.bool and obs.is_cuda


@pytest.mark.parametrize("task", TASKS)
def test_step_matches_twin(task):
    """More than a horizon of step() with all envs, reset(id) of the finished ones in between."""
    E = 16
    venv = _venv(task, E)
    oenv = _twin(venv)
    obs, info = venv.reset()
    assert np.array_equal(_h(obs), oenv.reset()) and len(info) == E
    n_term = 0
    for t in range(venv.max_episode_steps + 20):
        a = _actions(np.arange(E), t, venv.A)
        act = torch.from_numpy(a).cuda() if t % 2 == 0 else a          # device tensor, or an upload
        out = venv.step(act)
        ref = oenv.step(a)
        _check_step(out, ref, t)
        assert np.array_equal(out[4].env_id, np.arange(E))
        oterm, otrunc = ref[3], ref[4]
        n_term += int(oterm.sum())
        done = np.nonzero(oterm | otrunc)[0]
        if len(done):
            robs, rinfo = venv.reset(done)
            assert np.array_equal(_h(robs), oenv.reset(done)) and len(rinfo) == len(done), t
    assert np.array_equal(_h(venv.obs_cur), oenv.observe())
    assert np.array_equal(_h(venv.env_state), oenv.st)
    assert np.array_equal(_h(venv.env_t), oenv.t)
    assert np.array_equal(_h(venv.ep_idx).astype(np.uint32), oenv.ep_idx)
    if task in DRONES:
        assert n_term > 0


@pytest.mark.parametrize("task,E,n", [("SafetyDroneCircle-v0", 40, 5), ("SafetyAntCircle-v0", 1200, 700)])
def test_subset_step_touches_only_listed_envs(task, E, n):
    """700 ids span two launches of at most 512 ids each."""
    venv = _venv(task, E)
    oenv = _twin(venv)
    venv.reset()
    oenv.reset()
    rng = np.random.default_rng(3)
    for t in range(4):
        ids = rng.permutation(E)[:n]
        before = {k: getattr(venv, k).clone() for k in STATE}
        a = _actions(ids, t, venv.A)
        out = venv.step(torch.from_numpy(a).cuda(), ids)
        _check_step(out, oenv.step(a, ids), t)
        assert np.array_equal(out[4].env_id, ids)
        rest = np.setdiff1d(np.arange(E), ids)
        for k in STATE:
            now, old = _h(getattr(venv, k)), _h(before[k])
            if k == "env_state":
                now, old = now[:, rest], old[:, rest]
            else:
                now, old = now[rest], old[rest]
            assert np.array_equal(now, old), (t, k)
        assert np.array_equal(_h(venv.ep_len)[ids], _h(before["ep_len"])[ids] + 1)
        assert np.array_equal(_h(venv.obs_cur)[ids], _h(out[0]))
        robs, _ = venv.reset(ids[:3])
        assert np.array_equal(_h(robs), oenv.reset(ids[:3]))
    assert np.array_equal(_h(venv.env_state), oenv.st)


@pytest.mark.parametrize("task", ["SafetyCarCircle-v0", "SafetyDroneCircle-v0"])
@pytest.mark.parametrize("E,n_episode", [(8, 8), (8, 13)])
def test_fused_collect_continues_after_step(task, E, n_episode):
    """step() / reset(id) leave act_ctr alone, and a random-mode fused collect that follows them stores what the
    oracle collector stores when it continues from the twin's state."""
    from oracle import collector as ocol
    rounds = n_episode // E + 2
    T = 300
    policy, venv, buf, col = build_ppo(task, n_env=E, buffer_size=E * T * rounds)
    assert col.fused
    oenv = _twin(venv)
    oenv.reset()
    ctr0 = _h(venv.act_ctr).copy()
    for t in range(6):
        a = _actions(np.arange(E), t, venv.A)
        _, _, term, trunc, _ = venv.step(a)
        _, _, _, oterm, otrunc = oenv.step(a)
        done = np.nonzero(oterm | otrunc)[0]
        if len(done):
            venv.reset(done)
            oenv.reset(done)
    venv.reset([1, 2])
    oenv.reset([1, 2])
    assert np.array_equal(_h(venv.act_ctr), ctr0)
    assert np.array_equal(_h(venv.env_state), oenv.st)
    stats = col.collect(n_episode=n_episode, random=True)
    obuf = ocol.OracleBuffer(E * T * rounds, E, venv.D, venv.A)
    ctr = ctr0.astype(np.uint32)
    ostats = ocol.collect(oenv, None, n_episode, policy._act_seed, ctr, obuf, mode="random",
                          action_bound=policy.action_bound_method or "none")
    _assert_same_collect(stats, ostats, buf, obuf)
    assert np.array_equal(_h(venv.act_ctr).astype(np.uint32), ctr)


def _assert_same_collect(stats, ostats, buf, obuf):
    for k in ("n/ep", "n/st", "terminated", "truncated", "total_cost", "len"):
        assert stats[k] == ostats[k], k
    assert stats["rew"] == pytest.approx(ostats["rew"], rel=1e-12, abs=1e-12)
    b = buffer_to_numpy(buf)
    assert np.array_equal(b["ptr"], obuf.ptr) and np.array_equal(b["len"], obuf.len)
    for k in COLS:
        assert np.array_equal(b[k], getattr(obuf, k)), k


class HalfObs(torch.nn.Module):
    """A policy without fill_rollout whose action is an exact fp32 function of the observation.  It then
    scribbles over the observations it was given, which must not reach the env state."""

    def __init__(self, A):
        super().__init__()
        self.A = A

    def forward(self, batch, state=None, **kw):
        from fsrl_b200.data import Batch
        act = 0.5 * batch.obs[:, :self.A]
        batch.obs.fill_(float("nan"))
        return Batch(act=act)


@pytest.mark.parametrize("task", ["SafetyDroneCircle-v0", "SafetyCarRun-v0"])
@pytest.mark.parametrize("E,n_episode", [(16, 16), (16, 10), (6, 20)])
def test_generic_collect_matches_oracle_collector(task, E, n_episode):
    """n_episode <= E retires finished envs inline; n_episode > E resets them in the resolve kernel."""
    from fsrl_b200.data import FastCollector, VectorReplayBuffer
    from oracle import collector as ocol
    T = 300
    rounds = n_episode // E + 2
    venv = _venv(task, E, seed=9)
    buf = VectorReplayBuffer(E * T * rounds, E)
    policy = HalfObs(venv.A)
    col = FastCollector(policy, venv, buf)                   # resets every env
    assert col.fused is False
    stats = col.collect(n_episode=n_episode)
    oenv = _twin(venv)
    oenv.reset()
    obuf = ocol.OracleBuffer(E * T * rounds, E, venv.D, venv.A)
    ctr = np.zeros(E, np.uint32)
    actor = lambda obs: 0.5 * obs[:, :venv.A]
    ostats = ocol.collect(oenv, actor, n_episode, 0, ctr, obuf, mode="eval", head="deterministic")
    _assert_same_collect(stats, ostats, buf, obuf)
    assert not _h(venv.act_ctr).any()
    # the collect ends with a reset of every env, as the fused path's does
    assert np.array_equal(_h(venv.ep_idx).astype(np.uint32), oenv.ep_idx)
    assert np.array_equal(_h(venv.obs_cur), oenv.observe())


def _replay_ring(policy, venv, buf):
    """Step the twin env by env with the ring's stored raw actions; every stored column must match.  Returns
    the ring's transitions as rows of (obs, action as the env received it, rew, cost) bytes."""
    b = buffer_to_numpy(buf)
    oenv = _twin(venv)
    oenv.reset()
    rows = []
    for e in range(venv.env_num):
        for t in range(int(b["len"][e])):
            p = e * buf.cap + t
            assert np.array_equal(b["obs"][p], oenv.observe([e])[0]), (e, t)
            a = np.asarray(policy.map_action(b["act"][p][None]), np.float32)
            obs, rew, cost, term, trunc = oenv.step(a, [e])
            assert np.array_equal(b["obs_next"][p], obs[0]) and b["rew"][p] == rew[0] and b["cost"][p] == cost[0]
            assert b["terminated"][p] == term[0] and b["truncated"][p] == (trunc[0] & ~term[0]), (e, t)
            assert b["logp"][p] == 0
            rows.append(np.concatenate([b["obs"][p], a[0], [b["rew"][p], b["cost"][p]]]).astype(np.float32).tobytes())
        last = e * buf.cap + int(b["len"][e]) - 1
        assert b["terminated"][last] or b["truncated"][last]
    return rows


@pytest.mark.parametrize("hidden", [(64, 64, 64), (64, 128)])
def test_builtin_forward_with_a_non_arena_actor_collects(hidden):
    """A BasePolicy subclass that only adds learn(): its actor is a tianshou ActorProb the arena cannot hold
    (three hidden layers, or unequal widths), so forward() runs the module itself and the collect is generic."""
    from fsrl_b200 import envs, nets
    from fsrl_b200.data import Batch, FastCollector, VectorReplayBuffer
    from fsrl_b200.policy.base_policy import BasePolicy

    class Plain(BasePolicy):
        def learn(self, batch, **kw):
            return {}

    task, E = "SafetyCarRun-v0", 6
    env = envs.make(task)
    D, A, T = env.observation_space.shape[0], env.action_space.shape[0], env.spec.max_episode_steps
    torch.manual_seed(1)
    actor = nets.ActorProb(nets.Net(D, hidden_sizes=hidden), A).cuda()
    critic = nets.Critic(nets.Net(D, hidden_sizes=hidden)).cuda()
    policy = Plain(actor, critic, observation_space=env.observation_space, action_space=env.action_space)
    venv = envs.DeviceVectorEnv(task, E, seed=4)
    buf = VectorReplayBuffer(E * T, E)
    col = FastCollector(policy, venv, buf)
    assert col.fused is False
    policy.train()
    stats = col.collect(n_episode=E)
    assert stats["n/ep"] == E and stats["n/st"] == E * T
    _replay_ring(policy, venv, buf)
    # eval: the stored action is the actor's bounded mean of the stored observation
    policy.eval()
    buf.reset()
    col.collect(n_episode=E)
    b = buffer_to_numpy(buf)
    with torch.no_grad():
        (mu, _), _ = actor(torch.from_numpy(b["obs"]).cuda())
        out = policy(Batch(obs=torch.from_numpy(b["obs"]).cuda()))
    np.testing.assert_allclose(_h(out.act), _h(mu), rtol=0, atol=0)
    np.testing.assert_allclose(b["act"], _h(mu), rtol=1e-5, atol=1e-6)


def _deep_policy(env):
    """A BasePolicy with a 3-hidden-layer actor (the arena holds 2 hidden layers only), its own forward,
    process_fn and learn (a Gaussian policy-gradient step and a value regression)."""
    from fsrl_b200.data import Batch
    from fsrl_b200.policy.base_policy import BasePolicy
    nn = torch.nn
    D, A = env.observation_space.shape[0], env.action_space.shape[0]

    def mlp(out):
        return nn.Sequential(nn.Linear(D, 64), nn.ReLU(), nn.Linear(64, 64), nn.ReLU(), nn.Linear(64, 64), nn.ReLU(),
                             nn.Linear(64, out)).cuda()

    class Deep(BasePolicy):
        def __init__(self):
            super().__init__(mlp(A), [mlp(1)], observation_space=env.observation_space, action_space=env.action_space)
            self.log_std = nn.Parameter(torch.full((A,), -0.5, device="cuda"))
            self.optim = torch.optim.Adam(self.parameters(), lr=1e-3)

        def forward(self, batch, state=None, **kw):
            mu = self.actor(batch.obs)
            act = mu + self.log_std.exp() * torch.randn_like(mu) if self.training else mu
            return Batch(act=act)

        def process_fn(self, batch, buffer, indices):
            return buffer[indices]

        def learn(self, batch, batch_size=None, repeat=1, **kw):
            losses = []
            for _ in range(repeat):
                v = self.critics[0](batch.obs).flatten()
                adv = (batch.rew - v).detach()
                dist = torch.distributions.Normal(self.actor(batch.obs), self.log_std.exp())
                loss = -(dist.log_prob(batch.act).sum(-1) * adv).mean() + ((v - batch.rew) ** 2).mean()
                self.optim.zero_grad()
                loss.backward()
                self.optim.step()
                losses.append(loss.item())
            self.logger.store(**{"loss/total": float(np.mean(losses))})

    return Deep()


def test_network_outside_the_arena_collects_and_trains():
    from fsrl_b200 import envs
    from fsrl_b200.data import FastCollector, TrajectoryBuffer, VectorReplayBuffer
    from fsrl_b200.trainer import OnpolicyTrainer
    task, E = "SafetyDroneCircle-v0", 4
    env = envs.make(task)
    T = env.spec.max_episode_steps
    torch.manual_seed(0)
    policy = _deep_policy(env)
    venv = envs.DeviceVectorEnv(task, E, seed=21)
    buf = VectorReplayBuffer(E * T, E)
    tb = TrajectoryBuffer(use_grid_filter=False)
    col = FastCollector(policy, venv, buf, traj_buffer=tb)
    assert col.fused is False
    policy.train()
    stats = col.collect(n_episode=E)
    assert stats["n/ep"] == E
    # the ring replays through the twin, env by env, from the stored raw actions
    rows = _replay_ring(policy, venv, buf)
    # the harvest keeps the ring's episodes (actions as the env received them)
    assert len(tb.buffer) == E
    g = {k: _h(v) for k, v in tb.get_all().items()}
    got = [np.concatenate([g["observations"][i], g["actions"][i], [g["rewards"][i], g["costs"][i]]])
           .astype(np.float32).tobytes() for i in range(len(g["rewards"]))]
    assert sorted(got) == sorted(rows)
    # two short on-policy epochs with the policy's own learn()
    from fsrl_b200.utils.logger import BaseLogger
    logger = BaseLogger()
    policy.logger = logger
    col2 = FastCollector(policy, envs.DeviceVectorEnv(task, E, seed=22), VectorReplayBuffer(E * T, E))
    test_col = FastCollector(policy, envs.DeviceVectorEnv(task, 2, seed=23))
    trainer = OnpolicyTrainer(policy, col2, test_col, max_epoch=2, batch_size=256, step_per_epoch=1,
                              repeat_per_collect=2, episode_per_collect=E, episode_per_test=2, logger=logger,
                              verbose=False, show_progress=False)
    epochs = [(epoch, stats_) for epoch, stats_, _ in trainer]
    assert [e for e, _ in epochs] == [1, 2]
    assert trainer.cum_episode == 2 * E and trainer.env_step == col2.collect_step > 0
    assert test_col.collect_episode == 4
    for _, s in epochs:
        nums = {k: v for k, v in s.items() if isinstance(v, (int, float))}
        assert "loss/total" in nums and "train/reward" in nums and "test/reward" in nums, s
        assert all(math.isfinite(v) for v in nums.values()), s
    assert all(torch.isfinite(p).all() for p in policy.parameters())
