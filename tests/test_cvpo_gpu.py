"""CVPO on the device against the oracle chain (reference -> oracle/cvpo.py -> CUDA):

* the unsquashed conditioned-sigma rollout head (FSRL_HEAD_GAUSS_COND_RAW): stored raw actions and
  log-probs against a float64 evaluation of the actor with the same Philox draws;
* fsrl_cvpo_steps: per-step statistics and final parameters / duals against oracle.offpolicy.nstep_targets +
  oracle.cvpo.cvpo_update fed the same sampled indices and the same Philox draws (next actions of the current
  actor, particles of actor_old), over two collect cycles separated by post_update_fn / pre_update_fn;
* the M-step head gradient against float64 autograd of the oracle's M-step loss;
* examples/train_agent.py --algo cvpo end to end, and a checkpoint round trip."""
import os
import sys

import numpy as np
import pytest
import torch

from test_cvpo_host import cvpo_noise

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEY_ACT = 0x4143544E


def _agent(task="SafetyCarCircle-v0", hidden=64, cond=True, double=False, bounded=True, K=16, est=1, mst=1, seed=3):
    from fsrl_b200 import envs
    from fsrl_b200.agent import CVPOAgent
    env = envs.make(task)
    return CVPOAgent(env, seed=seed, hidden_sizes=(hidden, hidden), sample_act_num=K, estep_iter_num=est,
                     mstep_iter_num=mst, double_critic=double, conditioned_sigma=cond, unbounded=not bounded), env


def _collect(policy, task, n_env, seed=5):
    from fsrl_b200 import envs
    from fsrl_b200.data import FastCollector, VectorReplayBuffer
    venv = envs.DeviceVectorEnv(task, n_env, seed=seed)
    buf = VectorReplayBuffer(n_env * venv.max_episode_steps, n_env)
    col = FastCollector(policy, venv, buf)
    return venv, buf, col


# ---- rollout head --------------------------------------------------------------------------------------------
def _actor64(sd, prefix, D, A, H, cond, bounded, max_action):
    g = lambda k: sd[prefix + k].detach().cpu().double()
    w = [g("preprocess.model.model.0.weight"), g("preprocess.model.model.0.bias"),
         g("preprocess.model.model.2.weight"), g("preprocess.model.model.2.bias"),
         g("mu.model.0.weight"), g("mu.model.0.bias")]

    def f(obs):
        x = torch.relu(torch.as_tensor(obs, dtype=torch.float64) @ w[0].T + w[1])
        x = torch.relu(x @ w[2].T + w[3])
        mu = x @ w[4].T + w[5]
        if bounded:
            mu = max_action * torch.tanh(mu)
        if cond:
            s = (x @ g("sigma.model.0.weight").T + g("sigma.model.0.bias")).clamp(-20, 2).exp()
        else:
            s = g("sigma_param").view(1, -1).exp().expand_as(mu)
        return mu, s
    return f


@pytest.mark.parametrize("task,hidden,bounded", [("SafetyCarCircle-v0", 64, True), ("SafetyCarCircle-v0", 128, False),
                                                 ("SafetyAntCircle-v0", 64, False), ("SafetyAntCircle-v0", 128, True)])
def test_rollout_raw_head_matches_float64(task, hidden, bounded):
    """Train, random and eval collects with the raw head: stored actions and log-probs against float64 with the same
    Philox draws, the sigma clamp hit at both ends, and the stored actions replayed through the CPU env twin."""
    from helpers import buffer_to_numpy
    from oracle.envs import OracleVecEnv
    from oracle.philox import action_noise, action_uniform
    from fsrl_b200 import _lib
    agent, env = _agent(task, hidden=hidden, bounded=bounded)
    pol = agent.policy
    A = env.action_space.shape[0]
    with torch.no_grad():
        # dims 3i: sigma head far above its clamp (sigma = e^2); dims 3i+1: far below it (sigma = e^-20) with a zero
        # mean row, so that act - mu = sigma*eps stays exact in f32 and the log-prob remains well conditioned
        sb, mw, mb = pol.actor.sigma.model[0].bias, pol.actor.mu.model[0].weight, pol.actor.mu.model[0].bias
        for j in range(A):
            if j % 3 == 0:
                sb[j] = 1e3
            elif j % 3 == 1:
                sb[j] = -1e3
                mw[j].zero_()
                mb[j] = 0.0
    r = _lib.Rollout()
    pol.fill_rollout(r)
    assert r.head == _lib.HEAD_GAUSS_COND_RAW
    n_env = 80                                               # several CTAs of the rollout kernel
    venv, buf, col = _collect(pol, task, n_env)
    pol.train()
    col.collect(n_episode=n_env)
    bn = buffer_to_numpy(buf)
    sd = pol.state_dict()
    f = _actor64(sd, "actor.", env.observation_space.shape[0], A, hidden, True, bounded, float(env.action_space.high[0]))
    lens = bn["len"].astype(np.int64)
    T = int(lens.max())
    p_all = np.arange(n_env)[:, None] * buf.cap + np.arange(T)[None, :]
    valid = np.arange(T)[None, :] < lens[:, None]
    rows = p_all[valid]
    mu, s = f(bn["obs"][rows])
    mu, s = mu.numpy(), s.numpy()
    assert (s[:, 0::3] == np.exp(2.0)).all() and (A < 2 or (s[:, 1::3] == np.exp(-20.0)).all())
    eps = action_noise(pol._act_seed, np.repeat(np.arange(n_env), lens), np.concatenate([np.arange(l) for l in lens]), A)
    act64 = mu + s * eps
    got = bn["act"][rows].astype(np.float64)
    tol = 2e-5 * np.abs(act64) + 2e-5 * np.abs(act64).max(axis=0)      # per action dim: the clamped scales differ by e^22
    assert (np.abs(got - act64) <= tol).all(), np.abs(got - act64).max(axis=0)
    z = (got - mu) / s
    lp64 = (-0.5 * z * z - np.log(s) - 0.5 * np.log(2 * np.pi)).sum(1)
    np.testing.assert_allclose(bn["logp"][rows], lp64, rtol=1e-4, atol=1e-3)
    # the stored raw actions drive the CPU twin (clip + affine map of map_action) to the same transitions, bit for bit
    lo, hi = env.action_space.low.astype(np.float32), env.action_space.high.astype(np.float32)
    oenv = OracleVecEnv(venv.kind, n_env, venv.seed_value)
    obs = oenv.reset()
    for t in range(T):
        live = t < lens
        p = np.arange(n_env) * buf.cap + t
        assert np.array_equal(bn["obs"][p][live], obs[live]), t
        a = np.where(live[:, None], np.clip(bn["act"][p], -1, 1), 0).astype(np.float32)
        a = (lo + ((hi - lo) * (a + np.float32(1))) / np.float32(2)).astype(np.float32)
        obs, rew, cost, term, trunc = oenv.step(a)
        assert np.array_equal(bn["rew"][p][live], rew[live]) and np.array_equal(bn["cost"][p][live], cost[live]), t
        assert np.array_equal(bn["obs_next"][p][live], obs[live]), t
    # random mode (action_space.sample() through map_action_inverse): uniform draws, no log-prob, counters continue
    col.reset_buffer()
    col.collect(n_episode=n_env, random=True)
    bn = buffer_to_numpy(buf)
    lr_ = bn["len"].astype(np.int64)
    rows = (np.arange(n_env)[:, None] * buf.cap + np.arange(int(lr_.max()))[None, :])[np.arange(int(lr_.max()))[None, :] < lr_[:, None]]
    ctr = np.concatenate([lens[e] + np.arange(lr_[e]) for e in range(n_env)])
    want = action_uniform(pol._act_seed, np.repeat(np.arange(n_env), lr_), ctr, A)
    assert np.array_equal(bn["act"][rows], want) and not bn["logp"][rows].any()
    # eval mode: act = mu
    pol.eval()
    col.reset_buffer()
    col.collect(n_episode=n_env)
    bn = buffer_to_numpy(buf)
    rows = np.arange(bn["len"][0])
    mu, _ = f(bn["obs"][rows])
    np.testing.assert_allclose(bn["act"][rows], mu.numpy(), rtol=2e-5, atol=2e-5)
    pol.train()


# ---- gradient steps against the oracle ------------------------------------------------------------------------
def _q(sd, prefix, D, H, k=None):
    from oracle import nets as onets
    net = onets.ValueNet(D, [H, H])
    pre = "preprocess" if k is None else f"preprocess{k}"
    last = "last" if k is None else f"last{k}"
    g = lambda key: sd[prefix + key].detach().cpu()
    onets.load_linear(net.body.layers[0], g(pre + ".model.model.0.weight"), g(pre + ".model.model.0.bias"))
    onets.load_linear(net.body.layers[1], g(pre + ".model.model.2.weight"), g(pre + ".model.model.2.bias"))
    onets.load_linear(net.last, g(last + ".model.0.weight"), g(last + ".model.0.bias"))
    return net


def _oracle_nets(sd, D, A, H, cond, bounded, double, max_action):
    from oracle import nets as onets
    mk_a = lambda p: onets.load_from_state_dict(onets.GaussActor(D, A, [H, H], max_action=max_action,
                                                                 unbounded=not bounded, conditioned_sigma=cond), sd, p)
    if double:
        mk_c = lambda p: [[_q(sd, f"{p}{i}.", D + A, H, k) for k in (1, 2)] for i in range(2)]
    else:
        mk_c = lambda p: [_q(sd, f"{p}{i}.", D + A, H) for i in range(2)]
    return mk_a("actor."), mk_a("actor_old."), mk_c("critics."), mk_c("critics_old.")


def _flat(mods):
    out = []
    for m in mods:
        for q in (m if isinstance(m, list) else [m]):
            out += [p.detach().reshape(-1) for p in q.parameters()]
    return torch.cat(out).numpy()


def _q_min(c, obs, act):
    if isinstance(c, list):
        return torch.min(c[0](obs, act), c[1](obs, act))
    return c(obs, act)


CASES = [  # cond, double, bounded, estep_iters, mstep_iters, K, H, task (SafetyAntCircle-v0: A = 8, both Philox chunks)
    (True, False, True, 1, 1, 16, 64, "SafetyCarRun-v0"),
    (True, True, False, 3, 2, 64, 128, "SafetyCarRun-v0"),
    (False, False, False, 3, 1, 16, 128, "SafetyCarRun-v0"),
    (False, True, True, 1, 2, 64, 64, "SafetyCarRun-v0"),
    (True, False, False, 3, 2, 64, 64, "SafetyCarRun-v0"),
    (False, False, True, 1, 1, 16, 128, "SafetyCarRun-v0"),
    (True, True, True, 3, 2, 16, 64, "SafetyAntCircle-v0"),
    (False, False, False, 1, 1, 64, 128, "SafetyAntCircle-v0"),
]


def _adam_state(opt, p):
    st = opt.state[p]
    return float(st["exp_avg"].reshape(-1)[0]), float(st["exp_avg_sq"].reshape(-1)[0]), float(st["step"])


@pytest.mark.parametrize("cond,double,bounded,est,mst,K,H,task", CASES)
def test_cvpo_steps_match_oracle(cond, double, bounded, est, mst, K, H, task):
    from oracle import cvpo as ocvpo, offpolicy as ooff
    from test_offpolicy_gpu import _oracle_buffer
    agent, env = _agent(task, hidden=H, cond=cond, double=double, bounded=bounded, K=K, est=est, mst=mst)
    pol = agent.policy
    venv, buf, col = _collect(pol, task, 4)
    pol.train()
    col.collect(n_episode=4)
    D, A = env.observation_space.shape[0], env.action_space.shape[0]
    sd = pol.state_dict()
    max_action = float(env.action_space.high[0])
    actor, actor_old, crit, crit_old = _oracle_nets(sd, D, A, H, cond, bounded, double, max_action)
    a_opt = torch.optim.Adam(actor.parameters(), lr=5e-4)
    c_opt = torch.optim.Adam([p for c in crit for q in (c if isinstance(c, list) else [c]) for p in q.parameters()], lr=1e-3)
    estep_dual = torch.tensor([1.0, 0.0], requires_grad=True)
    e_opt = torch.optim.Adam([estep_dual], lr=0.02)
    ob = _oracle_buffer(buf)
    gamma, n_step, B, n = pol._gamma, pol._n_step, 64, 4
    thr = pol.qc_thres
    step = 0
    for cycle in range(2):
        pol.pre_update_fn(stats_train={"cost": 0.0})
        mduals = (torch.zeros(1, requires_grad=True), torch.zeros(1, requires_grad=True))
        m_opt = torch.optim.Adam(list(mduals), lr=0.1)
        np.random.seed(11 + cycle)
        idx_all = pol.sample_batch_indices(buf, n, B).cpu().numpy().astype(np.int64)
        ostats = []
        for k in range(n):
            idx = idx_all[k]
            with torch.no_grad():
                _, terminal = ooff.nstep_targets(ob, idx, [np.zeros(B)] * 2, gamma, n_step)
                obs_next = torch.from_numpy(ob.obs_next[terminal])
                mu, sig = actor(obs_next)
                a_next = mu + sig * torch.from_numpy(cvpo_noise(pol._upd_seed, B, A, step, 0))
                tq = [_q_min(crit_old[i], obs_next, a_next).numpy() for i in range(2)]
                obs = torch.from_numpy(ob.obs[idx])
                mu_o, sig_o = actor_old(obs)
                eps = torch.from_numpy(cvpo_noise(pol._upd_seed, K * B, A, step, 1)).view(K, B, A)
                particles = mu_o[None] + sig_o[None] * eps
            rets, _ = ooff.nstep_targets(ob, idx, tq, gamma, n_step)
            ostats.append(ocvpo.cvpo_update(actor, actor_old, crit, crit_old, a_opt, c_opt, estep_dual, e_opt, mduals,
                                            m_opt, obs, torch.from_numpy(ob.act[idx]), torch.from_numpy(rets),
                                            particles, qc_thres=thr, estep_iters=est, mstep_iters=mst, tau=0.05))
            step += 1
        np.random.seed(11 + cycle)
        pol.update_many(n, B, buf)
        st = pol.last_stats
        for key in ostats[0]:
            want = np.array([s[key] for s in ostats])
            np.testing.assert_allclose(np.asarray(st[key]), want, rtol=2e-3, atol=2e-5, err_msg=f"cycle {cycle} {key}")
        # the M-step duals themselves (not only their clipped uses) and their Adam state, before the next cycle's reset
        ms = pol._mstep_state.cpu().numpy()
        for i, p in enumerate(mduals):
            np.testing.assert_allclose(ms[i], float(p.detach()), rtol=1e-3, atol=1e-5, err_msg=f"cycle {cycle} mstep dual {i}")
            m, v, t = _adam_state(m_opt, p)
            np.testing.assert_allclose(ms[2 + i], m, rtol=5e-3, atol=1e-9 + 5e-3 * abs(m), err_msg=f"mstep adam m {i}")
            np.testing.assert_allclose(ms[4 + i], v, rtol=5e-3, atol=1e-12 + 5e-3 * abs(v), err_msg=f"mstep adam v {i}")
            assert ms[6] == t
        pol.post_update_fn(stats_train={"cost": 0.0})
        actor_old.load_state_dict(actor.state_dict())
    np.testing.assert_allclose(pol.estep_dual.cpu().numpy(), estep_dual.detach().numpy(), rtol=1e-4, atol=1e-6)
    es = pol._estep_state.cpu().numpy()
    e_st = e_opt.state[estep_dual]
    np.testing.assert_allclose(es[2:4], e_st["exp_avg"].numpy(), rtol=5e-3, atol=1e-7)
    np.testing.assert_allclose(es[4:6], e_st["exp_avg_sq"].numpy(), rtol=5e-3, atol=1e-10)
    assert es[6] == float(e_st["step"])
    sd2 = pol.state_dict()
    a2, a2o, c2, c2o = _oracle_nets(sd2, D, A, H, cond, bounded, double, max_action)
    assert np.abs(_flat([a2]) - _flat([actor])).max() < 1e-4
    assert np.abs(_flat([a2o]) - _flat([actor_old])).max() < 1e-4
    assert np.abs(_flat(c2) - _flat(crit)).max() < 2e-4
    assert np.abs(_flat(c2o) - _flat(crit_old)).max() < 2e-4


# ---- head gradients against float64 autograd ------------------------------------------------------------------------
@pytest.mark.parametrize("cond,bounded", [(True, True), (False, False)])
def test_mstep_head_gradient_matches_float64_autograd(cond, bounded):
    """One step with mstep_iter_num=1: the M-step kernel's d loss / d head output (left in the actor slot's dout)
    against float64 autograd of the oracle's M-step loss on the same weights, particles and E-step weights."""
    from oracle import cvpo as ocvpo
    task, H, K, B = "SafetyCarRun-v0", 64, 16, 64
    agent, env = _agent(task, hidden=H, cond=cond, bounded=bounded, K=K)
    pol = agent.policy
    if cond:                                  # sigma of dim 0 far past its upper clamp: the gate must zero its gradient
        with torch.no_grad():
            pol.actor.sigma.model[0].bias[0] = 1e3
    venv, buf, col = _collect(pol, task, 4)
    pol.train()
    col.collect(n_episode=4)
    pol.pre_update_fn()
    sd0 = {k: v.clone() for k, v in pol.state_dict().items() if torch.is_tensor(v)}
    np.random.seed(3)
    pol.update_many(1, B, buf)
    torch.cuda.synchronize()
    idx = pol._cw["part_idx"][:B].long()
    w = pol._cw["weights"][:K * B].view(K, B).double().cpu()
    parts = pol._cw["particles"][:K * B].view(K, B, -1).double().cpu()
    mu_old = pol._cw["mu_old"][:B].double().cpu(); std_old = pol._cw["std_old"][:B].double().cpu()
    A = parts.shape[-1]
    eng = pol._eng
    g = pol._groups()
    dout = eng.slot_view(g["actor"][0], "dout")[:B].double().cpu()
    # the actor before its Adam step produced `out`; rebuild it in float64 from the saved weights
    obs = buf.obs[idx].double().cpu()
    gw = lambda k: sd0["actor." + k].double().cpu()
    x = torch.relu(obs @ gw("preprocess.model.model.0.weight").T + gw("preprocess.model.model.0.bias"))
    x = torch.relu(x @ gw("preprocess.model.model.2.weight").T + gw("preprocess.model.model.2.bias"))
    o_mu = (x @ gw("mu.model.0.weight").T + gw("mu.model.0.bias")).requires_grad_(True)
    if cond:
        o_s = (x @ gw("sigma.model.0.weight").T + gw("sigma.model.0.bias")).requires_grad_(True)
        std = o_s.clamp(-20, 2).exp()
    else:
        o_s = gw("sigma_param").view(1, -1).clone().requires_grad_(True)
        std = o_s.exp().expand(B, A)
    mu = pol.actor._max * torch.tanh(o_mu) if bounded else o_mu
    from torch.distributions import Independent, Normal
    d1, d2 = Independent(Normal(mu, std_old), 1), Independent(Normal(mu_old, std), 1)
    lik = d1.expand((K, B)).log_prob(parts) + d2.expand((K, B)).log_prob(parts)
    kl_mu, kl_std = ocvpo.gaussian_kl(mu_old, std_old, mu, std)
    st = pol.last_stats
    loss = -(w * lik).mean() + float(st["mstep/mstep_dual_mu"][0]) * kl_mu + float(st["mstep/mstep_dual_std"][0]) * kl_std
    loss.backward()
    want_mu = o_mu.grad.numpy()
    got_mu = dout[:, :A].numpy()
    scale = np.abs(want_mu).max()
    assert np.abs(got_mu - want_mu).max() <= 1e-3 * scale + 1e-9
    if cond:
        want_s, got_s = o_s.grad.numpy(), dout[:, A:2 * A].numpy()
    else:
        want_s, got_s = o_s.grad.numpy().reshape(-1), dout[:, A:2 * A].numpy().sum(0)
    assert np.abs(got_s - want_s).max() <= 1e-3 * np.abs(want_s).max() + 1e-9


@pytest.mark.parametrize("double,K", [(False, 16), (True, 64)])
def test_estep_dual_gradient_matches_float64_autograd(double, K):
    """First step of a fresh policy (estep_iter_num=1): the dual gradient the E-step kernel fed to Adam (its first
    moment is 0.1 * grad) against float64 autograd of the reference's dual loss (cvpo.py:278-287) on the Q values
    the device computed for the particles, at the initial dual [eta, lambda] = [1, 0]."""
    task, H, B = "SafetyCarRun-v0", 64, 64
    agent, env = _agent(task, hidden=H, double=double, K=K)
    pol = agent.policy
    venv, buf, col = _collect(pol, task, 4)
    pol.train()
    col.collect(n_episode=4)
    pol.pre_update_fn()
    np.random.seed(4)
    pol.update_many(1, B, buf)
    torch.cuda.synchronize()
    g_dev = pol._estep_state[2:4].double().cpu().numpy() / 0.1
    eng, g = pol._eng, pol._groups()
    outs = [eng.slot_view(sl, "out")[:K * B, 0].double().cpu() for sl in g["critics"]]
    per = 2 if double else 1
    q = [torch.min(*outs[per * i:per * i + per]) if double else outs[i] for i in range(2)]
    q = [x.view(K, B).T for x in q]                            # (B, K) like the reference's q_values
    dual = torch.tensor([1.0, 0.0], dtype=torch.float64, requires_grad=True)
    eta = dual[0]
    combined = q[0] - dual[1] * q[1]
    loss = eta * pol._estep_kl + dual[1] * pol.qc_thres[0]
    loss = loss + eta * torch.mean(torch.logsumexp(combined / eta, dim=1) - np.log(K))
    loss.backward()
    want = dual.grad.numpy()
    assert np.abs(g_dev - want).max() <= 1e-4 * np.abs(want).max() + 1e-7, (g_dev, want)
    assert float(pol.last_stats["loss/estep_loss"][0]) == pytest.approx(float(loss), rel=1e-4, abs=1e-6)


# ---- end to end ------------------------------------------------------------------------------------------------------
def test_train_agent_cvpo_and_checkpoint_round_trip(tmp_path):
    import json
    sys.path.insert(0, os.path.join(ROOT, "examples"))
    import train_agent
    argv = ["--algo", "cvpo", "--task", "SafetyBallRun-v0", "--epoch", "2", "--step_per_epoch", "1600",
            "--training_num", "16", "--episode_per_collect", "16", "--testing_num", "2", "--hidden_sizes", "(64,64)",
            "--buffer_size", "6400", "--logdir", str(tmp_path), "--verbose", "False", "--save_interval", "1",
            "--update_per_step", "0.05"]
    epoch, stats, info = train_agent.main(argv)
    assert epoch == 2 and info["train_speed"] > 0
    from fsrl_b200.utils.exp_util import load_config_and_model
    run = [d for d in os.listdir(tmp_path)][0]
    cfg, model = load_config_and_model(os.path.join(tmp_path, run))
    sd = model["model"]
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "cvpo_host_golden.json")))
    want = set(golden["state_dict"]["single"]["keys"])
    assert set(sd) == want, sorted(set(sd) ^ want)
    from fsrl_b200 import envs
    from fsrl_b200.agent import CVPOAgent
    from fsrl_b200.data.batch import Batch
    agent2 = CVPOAgent(envs.make("SafetyBallRun-v0"), seed=99, hidden_sizes=(64, 64))
    agent2.policy.load_state_dict(sd)
    agent3 = CVPOAgent(envs.make("SafetyBallRun-v0"), seed=98, hidden_sizes=(64, 64))
    agent3.policy.load_state_dict(sd)
    for a in (agent2, agent3):
        a.policy.eval()
    obs = torch.randn(32, envs.make("SafetyBallRun-v0").observation_space.shape[0], device="cuda")
    r2 = agent2.policy(Batch(obs=obs)); r3 = agent3.policy(Batch(obs=obs))
    assert torch.equal(r2.act, r3.act) and torch.isfinite(r2.act).all()
    test = envs.DeviceVectorEnv("SafetyBallRun-v0", 2, seed=4)
    e2 = agent2.evaluate(test, eval_episodes=2)
    test = envs.DeviceVectorEnv("SafetyBallRun-v0", 2, seed=4)
    e3 = agent3.evaluate(test, eval_episodes=2)
    assert e2 == e3 and all(np.isfinite(v) for v in e2)
