"""SAC-/DDPG-Lagrangian parity: n-step targets, critic / actor / alpha updates and Polyak sync on
the device (fsrl_offpolicy_steps through the C-ABI) against the torch-CPU restatement of
sac_lag.py:136-269 / ddpg_lag.py:120-223 / base_policy.py:453-512, with identical weights,
identical sampled indices and the same reparameterisation noise (Philox stream replayed by the
oracle).  Tolerances: per-step losses rtol 5e-4 on the first steps; parameters atol 5e-5."""
import numpy as np
import pytest
import torch

from helpers import buffer_to_numpy, synthetic_ring, upd_noise as _upd_noise

pytestmark = pytest.mark.gpu

def _build(algo, task="SafetyCarRun-v0", hidden=(64, 64), n_env=4, seed=10):
    from fsrl_b200 import envs
    from fsrl_b200.agent import DDPGLagAgent, SACLagAgent
    from fsrl_b200.data import FastCollector, VectorReplayBuffer
    env = envs.make(task)
    if algo == "sac":
        agent = SACLagAgent(env, seed=seed, hidden_sizes=hidden, unbounded=True, n_step=2, tau=0.05)
    else:
        agent = DDPGLagAgent(env, seed=seed, hidden_sizes=hidden, n_step=2, tau=0.05, actor_lr=5e-4)
    venv = envs.DeviceVectorEnv(task, n_env, seed=seed + 2)
    buf = VectorReplayBuffer(n_env * env.spec.max_episode_steps, n_env)
    col = FastCollector(agent.policy, venv, buf, exploration_noise=True)
    return agent.policy, venv, buf, col


def _oracle_buffer(buf):
    from oracle.collector import OracleBuffer
    b = buffer_to_numpy(buf)
    ob = OracleBuffer(buf.maxsize, buf.buffer_num, buf.D, buf.A)
    for k in ("obs", "obs_next", "act", "rew", "cost", "terminated", "truncated"):
        setattr(ob, k, b[k])
    ob.ptr = b["ptr"].astype(np.int64); ob.len = b["len"].astype(np.int64)
    return ob


def _load_q(net, sd, prefix, k=None):
    from oracle import nets as onets
    pre = "preprocess" if k is None else f"preprocess{k}"
    last = "last" if k is None else f"last{k}"
    g = lambda key: sd[prefix + key].detach().cpu()
    onets.load_linear(net.body.layers[0], g(pre + ".model.model.0.weight"), g(pre + ".model.model.0.bias"))
    onets.load_linear(net.body.layers[1], g(pre + ".model.model.2.weight"), g(pre + ".model.model.2.bias"))
    onets.load_linear(net.last, g(last + ".model.0.weight"), g(last + ".model.0.bias"))
    return net


def _flat(mods):
    return torch.cat([p.detach().reshape(-1) for m in mods for p in m.parameters()]).numpy()


def test_nstep_prepare_matches_oracle():
    """The n-step walk on a collected ring that never wrapped, and on synthetic rings: full rings wrapped with
    ptr mid-ring, partly filled rings, and terminations and truncations 1 to 8 steps before ptr, up to
    n_step = FSRL_MAX_NSTEP = 8.  n_step = 9 is refused."""
    import ctypes
    from fsrl_b200 import _lib
    from oracle import offpolicy as ooff
    policy, venv, buf, col = _build("ddpg", n_env=3)
    col.collect(n_episode=5)                    # several episodes per env, ring not wrapped
    policy._ensure_engine(256)
    D, A = venv.D, venv.A
    rng = np.random.default_rng(0)
    s = torch.cuda.current_stream().cuda_stream
    rings = [(buf, (1, 2, 3, 5))] + [(synthetic_ring(D, A, 8, 64, layout, seed=k), (1, 2, 5, 8))
                                     for k, layout in enumerate(("wrapped", "partial", "mixed"))]
    for ring, n_steps in rings:
        ob = _oracle_buffer(ring)
        valid = ob.sample_all()
        # every transition within 9 steps of a ring's newest slot, where the walk wraps or stops, plus random ones
        near = np.concatenate([e * ob.cap + (ob.ptr[e] - 1 - np.arange(9)) % ob.cap for e in range(ob.E) if ob.len[e] >= 9])
        idx = np.concatenate([near, rng.choice(valid, 256 - len(near))]).astype(np.int32)
        assert np.isin(idx, valid).all()
        for n_step in n_steps:
            policy._n_step = n_step
            d = policy._descriptor(ring)
            it = torch.as_tensor(idx, device="cuda")
            _lib.check(_lib.lib.fsrl_nstep_prepare(ctypes.byref(d), it.data_ptr(), 256, s))
            torch.cuda.synchronize()
            tq = [rng.standard_normal(256).astype(np.float32) for _ in range(2)]
            rets, terminal = ooff.nstep_targets(ob, idx, tq, policy._gamma, n_step)
            w = policy._w
            assert np.array_equal(w["term_idx"].cpu().numpy()[:256], terminal.astype(np.int32))      # integer-exact
            vm = w["vmask"].cpu().numpy()[:256]; gp = w["gpow"].cpu().numpy()[:256]; part = w["partial"].cpu().numpy()
            assert np.array_equal(vm, (~ob.terminated[terminal]).astype(np.float32))
            for i in range(2):
                got = (tq[i] * vm).astype(np.float64) * gp + part[i * 256:(i + 1) * 256]
                np.testing.assert_allclose(got.astype(np.float32), rets[:, i], rtol=1e-6, atol=1e-6)
        if ring is not buf:
            # the synthetic rings put both kinds of ends inside the 8-step walks
            assert ob.terminated[terminal].any() and (ob.truncated[terminal] & ~ob.terminated[terminal]).any()
    policy._n_step = 9
    d = policy._descriptor(buf)
    with pytest.raises(ValueError, match="n_step 9 out of range"):
        _lib.check(_lib.lib.fsrl_nstep_prepare(ctypes.byref(d), it.data_ptr(), 256, s))


@pytest.mark.parametrize("auto_alpha", [True, False])
def test_sac_steps_match_oracle(auto_alpha):
    from oracle import nets as onets, offpolicy as ooff
    hidden = (64, 64)
    policy, venv, buf, col = _build("sac", hidden=hidden)
    if not auto_alpha:
        policy._is_auto_alpha = False
        policy._alpha0 = 0.2
    col.collect(n_episode=4)
    policy.lag_optims[0].lagrangian = 0.8
    sd = policy.state_dict()
    D, A = venv.D, venv.A
    actor = onets.load_from_state_dict(onets.GaussActor(D, A, list(hidden), unbounded=True, conditioned_sigma=True), sd, "actor.")
    crit = [[_load_q(onets.ValueNet(D + A, list(hidden)), sd, f"critics.{i}.", k) for k in (1, 2)] for i in range(2)]
    crit_old = [[_load_q(onets.ValueNet(D + A, list(hidden)), sd, f"critics_old.{i}.", k) for k in (1, 2)] for i in range(2)]
    a_opt = torch.optim.Adam(actor.parameters(), lr=5e-4)
    c_opt = torch.optim.Adam([p for pair in crit for q in pair for p in q.parameters()], lr=1e-3)
    auto = None
    alpha = 0.2
    if auto_alpha:
        log_alpha = torch.zeros(1, requires_grad=True)
        auto = (-float(A), log_alpha, torch.optim.Adam([log_alpha], lr=3e-4))
        alpha = 1.0
    ob = _oracle_buffer(buf)
    K, B = 6, 128
    np.random.seed(5)
    idx_all = policy.sample_batch_indices(buf, K, B).cpu().numpy()
    ostats = []
    for k in range(K):
        st, alpha = ooff.sac_step(actor, crit, crit_old, a_opt, c_opt, ob, idx_all[k].astype(np.int64),
                                  _upd_noise(policy._upd_seed, B, A, k, 0), _upd_noise(policy._upd_seed, B, A, k, 1),
                                  alpha=alpha, gamma=policy._gamma, n_step=2, tau=0.05, lagrangian=0.8, auto_alpha=auto)
        ostats.append(st)
    np.random.seed(5)
    policy.update_many(K, B, buf)
    st = policy.last_stats
    for key in ("loss/q0", "loss/q1", "loss/actor_rew", "loss/actor_safety", "loss/actor_total"):
        want = np.array([s[key] for s in ostats])
        np.testing.assert_allclose(np.asarray(st[key]), want, rtol=2e-3, atol=2e-5, err_msg=key)
    if auto_alpha:
        np.testing.assert_allclose(st["loss/alpha_value"], [s["loss/alpha_value"] for s in ostats], rtol=1e-4)
    sd2 = policy.state_dict()
    actor2 = onets.load_from_state_dict(onets.GaussActor(D, A, list(hidden), unbounded=True, conditioned_sigma=True), sd2, "actor.")
    assert np.abs(_flat([actor2]) - _flat([actor])).max() < 1e-4
    for i in range(2):
        for k in (1, 2):
            q2 = _load_q(onets.ValueNet(D + A, list(hidden)), sd2, f"critics.{i}.", k)
            assert np.abs(_flat([q2]) - _flat([crit[i][k - 1]])).max() < 2e-4
            q2o = _load_q(onets.ValueNet(D + A, list(hidden)), sd2, f"critics_old.{i}.", k)
            assert np.abs(_flat([q2o]) - _flat([crit_old[i][k - 1]])).max() < 2e-4


def test_ddpg_steps_match_oracle():
    from oracle import nets as onets, offpolicy as ooff
    hidden = (64, 64)
    policy, venv, buf, col = _build("ddpg", hidden=hidden)
    col.collect(n_episode=4)
    policy.lag_optims[0].lagrangian = 0.5
    sd = policy.state_dict()
    D, A = venv.D, venv.A
    mk_actor = lambda pfx: onets.load_from_state_dict(onets.DetActor(D, A, list(hidden)), sd, pfx)
    actor, actor_old = mk_actor("actor."), mk_actor("actor_old.")
    crit = [_load_q(onets.ValueNet(D + A, list(hidden)), sd, f"critics.{i}.") for i in range(2)]
    crit_old = [_load_q(onets.ValueNet(D + A, list(hidden)), sd, f"critics_old.{i}.") for i in range(2)]
    a_opt = torch.optim.Adam(actor.parameters(), lr=5e-4)
    c_opt = torch.optim.Adam([p for q in crit for p in q.parameters()], lr=1e-3)
    ob = _oracle_buffer(buf)
    K, B = 6, 128
    np.random.seed(9)
    idx_all = policy.sample_batch_indices(buf, K, B).cpu().numpy()
    ostats = [ooff.ddpg_step(actor, actor_old, crit, crit_old, a_opt, c_opt, ob, idx_all[k].astype(np.int64),
                             gamma=policy._gamma, n_step=2, tau=0.05, lagrangian=0.5) for k in range(K)]
    np.random.seed(9)
    policy.update_many(K, B, buf)
    st = policy.last_stats
    for key in ("loss/q0", "loss/q1", "loss/actor_rew", "loss/actor_safety", "loss/actor_total"):
        want = np.array([s[key] for s in ostats])
        np.testing.assert_allclose(np.asarray(st[key]), want, rtol=2e-3, atol=2e-5, err_msg=key)
    sd2 = policy.state_dict()
    a2 = onets.load_from_state_dict(onets.DetActor(D, A, list(hidden)), sd2, "actor.")
    a2o = onets.load_from_state_dict(onets.DetActor(D, A, list(hidden)), sd2, "actor_old.")
    assert np.abs(_flat([a2]) - _flat([actor])).max() < 1e-4
    assert np.abs(_flat([a2o]) - _flat([actor_old])).max() < 1e-4
    for i in range(2):
        q2 = _load_q(onets.ValueNet(D + A, list(hidden)), sd2, f"critics.{i}.")
        assert np.abs(_flat([q2]) - _flat([crit[i]])).max() < 2e-4


@pytest.mark.parametrize("algo,head", [("sac", "gauss_cond"), ("ddpg", "deterministic")])
def test_offpolicy_rollout_heads_match_oracle(algo, head):
    from oracle import collector as ocol, nets as onets
    from oracle.envs import OracleVecEnv
    hidden = (64, 64)
    policy, venv, buf, col = _build(algo, hidden=hidden, n_env=5)
    stats = col.collect(n_episode=5)
    sd = policy.state_dict()
    D, A = venv.D, venv.A
    if algo == "sac":
        actor = onets.load_from_state_dict(onets.GaussActor(D, A, list(hidden), unbounded=True, conditioned_sigma=True), sd, "actor.")
    else:
        actor = onets.load_from_state_dict(onets.DetActor(D, A, list(hidden)), sd, "actor.")
    oenv = OracleVecEnv(venv.kind, 5, venv.seed_value); oenv.reset()
    obuf = ocol.OracleBuffer(buf.maxsize, 5, D, A)
    ostats = ocol.collect(oenv, actor, 5, policy._act_seed, np.zeros(5, np.uint32), obuf, head=head,
                          expl_sigma=0.1 if algo == "ddpg" else 0.0)
    b = buffer_to_numpy(buf)
    assert stats["n/st"] == ostats["n/st"] and np.array_equal(b["len"], obuf.len)
    first = np.arange(5) * obuf.cap
    np.testing.assert_allclose(b["act"][first], obuf.act[first], rtol=2e-5, atol=2e-6)
    np.testing.assert_allclose(b["act"], obuf.act, rtol=0, atol=5e-3)
    np.testing.assert_allclose(b["rew"], obuf.rew, rtol=0, atol=5e-3)


def test_compute_nstep_returns_api_matches_oracle():
    """BasePolicy.compute_nstep_returns (base_policy.py:453-512) as a public call: user-supplied target_q_fn,
    batch.rets of shape (B, 1, C) like the reference's (target_q keeps its trailing axis)."""
    from oracle import offpolicy as ooff
    policy, venv, buf, col = _build("ddpg", n_env=3)
    col.collect(n_episode=5)
    ob = _oracle_buffer(buf)
    rng = np.random.default_rng(1)
    idx = rng.choice(ob.sample_all(), 200).astype(np.int64)
    for n_step in (1, 2, 4):
        tq = [rng.standard_normal(200).astype(np.float32) for _ in range(2)]
        seen = {}

        def target_q_fn(buffer, terminal):
            seen["terminal"] = terminal.cpu().numpy().copy()
            return [torch.from_numpy(t).cuda().reshape(-1, 1) for t in tq]

        batch = policy.compute_nstep_returns(None, buf, idx, target_q_fn, n_step)
        rets, terminal = ooff.nstep_targets(ob, idx, tq, policy._gamma, n_step)
        assert np.array_equal(seen["terminal"], terminal.astype(np.int32))
        got = batch.rets.cpu().numpy()
        assert got.shape == (200, 1, 2)
        np.testing.assert_allclose(got[:, 0, :], rets, rtol=1e-6, atol=1e-6)
