"""CPO parity: surrogate / cost gradients, the exact KL Hessian-vector product (R-op kernels vs
autograd double backward), conjugate gradients, the dual case analysis and the line search on
the device against the torch-CPU restatement of cpo.py:123-370.  Gradients, Hessian-vector
products and CG solves are compared with float64 autograd (GRAD_TOL / HVP_TOL / CG_TOL below,
relative to the reference vector); the learn() parity keeps the fp32 oracle: per-step scalars rtol
5e-3 (CG amplifies fp32 noise by the condition number), step size / optim_case exact."""
import ctypes

import numpy as np
import pytest
import torch

from helpers import buffer_to_numpy, cg64, cg_stop_tol

pytestmark = pytest.mark.gpu


def _build(task="SafetyCarCircle-v0", hidden=(64, 64), n_env=4, seed=10, **kw):
    from fsrl_b200 import envs
    from fsrl_b200.agent import CPOAgent
    from fsrl_b200.data import FastCollector, VectorReplayBuffer
    env = envs.make(task)
    agent = CPOAgent(env, seed=seed, hidden_sizes=hidden, **kw)
    venv = envs.DeviceVectorEnv(task, n_env, seed=seed + 2)
    buf = VectorReplayBuffer(n_env * env.spec.max_episode_steps, n_env)
    col = FastCollector(agent.policy, venv, buf, exploration_noise=True)
    return agent.policy, venv, buf, col


def _oracle(policy, hidden):
    from oracle import nets as onets
    sd = policy.state_dict()
    D, A = policy.arena.slots[0].D, policy.arena.slots[0].out
    actor = onets.load_from_state_dict(onets.GaussActor(D, A, list(hidden)), sd, "actor.")
    critics = [onets.load_from_state_dict(onets.ValueNet(D, list(hidden)), sd, f"critics.{i}.") for i in range(2)]
    return actor, critics


def _oracle_vec(actor):
    """oracle parameter vector in torch's parameters() order (body, mu, sigma_param)"""
    return torch.cat([p.detach().reshape(-1) for p in actor.parameters()]).numpy()


def _to_arena_order(vec, D, H, A):
    """torch order [sigma_param?]: GaussActor registers body.layers.{0,1}, mu, then sigma_param ->
    W1[H,D] b1 W2[H,H] b2 W3[A,H] b3 sigma[A]  -> arena: W1t[D,H] b1 W2t b2 W3t[H,A] b3 sigma"""
    o = 0
    def take(n):
        nonlocal o
        v = vec[o:o + n]; o += n
        return v
    # parameters() order of oracle.nets.GaussActor: sigma_param first? resolve by construction
    raise NotImplementedError


def _arena_to_torch_order(actor, v, D, H, A):
    """arena-layout vector -> list of tensors shaped like actor.parameters()"""
    o = 0
    w1t = v[o:o + D * H].reshape(D, H); o += D * H
    b1 = v[o:o + H]; o += H
    w2t = v[o:o + H * H].reshape(H, H); o += H * H
    b2 = v[o:o + H]; o += H
    w3t = v[o:o + H * A].reshape(H, A); o += H * A
    b3 = v[o:o + A]; o += A
    sg = v[o:o + A]
    named = {"body.layers.0.weight": w1t.T, "body.layers.0.bias": b1, "body.layers.1.weight": w2t.T,
             "body.layers.1.bias": b2, "mu.weight": w3t.T, "mu.bias": b3, "sigma_param": sg.reshape(A, 1)}
    return np.concatenate([np.ascontiguousarray(named[n]).reshape(-1) for n, _ in actor.named_parameters()])


def _torch_to_arena_order(actor, v, D, H, A):
    out = {}
    o = 0
    for n, p in actor.named_parameters():
        k = p.numel()
        out[n] = v[o:o + k].reshape(tuple(p.shape)); o += k
    return np.concatenate([out["body.layers.0.weight"].T.reshape(-1), out["body.layers.0.bias"],
                           out["body.layers.1.weight"].T.reshape(-1), out["body.layers.1.bias"],
                           out["mu.weight"].T.reshape(-1), out["mu.bias"], out["sigma_param"].reshape(-1)])


def _prepare(hidden=(64, 64), task="SafetyCarCircle-v0", n_env=4):
    from oracle import cpo as ocpo
    policy, venv, buf, col = _build(task, hidden=hidden, n_env=n_env, max_backtracks=10, optim_critic_iters=3)
    stats = col.collect(n_episode=n_env)
    policy.pre_update_fn(stats_train=stats)
    actor, critics = _oracle(policy, hidden)
    idx = buf.sample_indices(0)
    batch = policy.process_fn(None, buf, idx)
    b = buffer_to_numpy(buf)
    sel = idx.cpu().numpy()
    ob = {k: b[k][sel] for k in ("obs", "obs_next", "act", "rew", "cost", "terminated", "truncated")}
    ob = ocpo.process(actor, critics, ob, 0.99, 0.95)
    # process_fn parity, then hand the oracle the device's numbers for everything downstream
    np.testing.assert_allclose(batch.advs.cpu().numpy(), ob["advs"], rtol=2e-3, atol=2e-4)
    np.testing.assert_allclose(batch.mean_old.cpu().numpy(), ob["mean_old"], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(batch.std_old.cpu().numpy(), ob["std_old"], rtol=1e-6)
    ob["advs"] = batch.advs.cpu().numpy().copy(); ob["rets"] = batch.rets.cpu().numpy().copy()
    ob["logp_old"] = batch.logp_old.cpu().numpy().copy(); ob["mean_old"] = batch.mean_old.cpu().numpy().copy()
    ob["std_old"] = batch.std_old.cpu().numpy().copy()
    return policy, batch, ob, actor, critics, stats


# float64 oracle bounds (|err| / max|ref| for vectors); the observed errors are printed
GRAD_TOL = 5e-5      # theta = theta_old: observed <= 2e-6
# theta moved: the surrogate gradients are means of ratio-weighted terms that largely cancel, and the
# device sums up to 4096 rows per thread in fp32 (observed 3.7e-4 at 2x512 on 4800 rows, <= 2e-6 at 2x64
# and 2x128); the engine tests bound those sums by their terms' magnitudes
GRAD_TOL_MOVED = 5e-4
HVP_TOL = 1e-4
CG_TOL = 2e-4        # iterate 4 or so, where the early exit is tested
CG10_TOL = 2e-2      # iterate 10: fp32 CG loses conjugacy as |r| falls by ~300 x (observed 7e-3 at 2x128)

HVP_CASES = [
    # the first two keep their ids: 2x64, ~1200 rows, the whole batch in order
    pytest.param(False, (64, 64), 4, False, id="False"),
    pytest.param(True, (64, 64), 4, False, id="True"),
    pytest.param(False, (64, 64), 16, True, id="h64-16env-perm"),
    pytest.param(False, (128, 128), 16, True, id="h128-16env-perm"),
    pytest.param(True, (128, 128), 16, False, id="moved-h128-16env"),
    pytest.param(False, (512, 512), 4, True, id="h512-perm"),
    pytest.param(True, (512, 512), 16, True, id="moved-h512-16env-perm"),
]


def _rows(n_all, gathered, seed=5):
    """rows of the minibatch and its device perm: all rows in order, or a shuffled minibatch as learn()
    gathers it (the whole permuted batch above 4096 rows, else the first two thirds of it)"""
    if not gathered:
        return np.arange(n_all), None
    rows = np.random.default_rng(seed).permutation(n_all)
    if n_all <= 4096:
        rows = rows[:2 * n_all // 3]
    return rows, torch.as_tensor(rows.astype(np.int32), device="cuda")


def _kl64(actor, ob, rows):
    from torch.distributions import Independent, Normal, kl_divergence
    t = lambda k: torch.from_numpy(np.ascontiguousarray(ob[k][rows])).double()
    mu, sigma = actor(t("obs"))
    return kl_divergence(Independent(Normal(t("mean_old"), t("std_old")), 1), Independent(Normal(mu, sigma), 1)).mean()


@pytest.mark.parametrize("moved,hidden,n_env,gathered", HVP_CASES)
def test_gradients_and_hvp_match_autograd(moved, hidden, n_env, gathered):
    """Head gradients, wgrad_to and the exact KL Hessian-vector product against float64 autograd
    (double backward).  moved=True perturbs theta away from theta_old so the exact Hessian !=
    Gauss-Newton; n_env=16 collects ~4800 rows, above the 4096 rows where wgrad splits them;
    gathered reads a shuffled minibatch through perm."""
    from fsrl_b200 import _lib
    from torch.distributions import Independent, Normal
    from oracle import cpo as ocpo
    policy, batch, ob, actor, critics, stats = _prepare(hidden, n_env=n_env)
    a = policy.arena.slots[0]
    D, H, A, P = a.D, a.H, a.out, a.size
    if moved:
        g = torch.Generator().manual_seed(1)
        delta = 0.05 * (64 / H) ** 0.5 * torch.randn(P, generator=g)     # the same relative move at every width
        policy.arena.theta[a.offset:a.offset + P] += delta.cuda()
        ocpo._set_flat(actor, torch.from_numpy(_arena_to_torch_order(actor, policy.arena.theta[a.offset:a.offset + P].cpu().numpy(), D, H, A)))
    actor.double()
    n_all = batch.n
    assert n_all > 4096 or n_env == 4
    rows, perm = _rows(n_all, gathered)
    n = len(rows)
    eng = policy._ensure_engine(n_all)
    eng.sync_mirror([a])
    d = policy._descriptor(batch, perm, n)
    inp = eng.make_input(batch.obs, perm)
    eng.forward([a], inp, n, save=True)
    # ---- float64 oracle scalars / gradients ------------------------------------------------------
    t = lambda k: torch.from_numpy(np.ascontiguousarray(ob[k][rows])).double()
    obs, act = t("obs"), t("act")
    mu, sigma = actor(obs)
    dist = Independent(Normal(mu, sigma), 1)
    logp = dist.log_prob(act)
    ratio = torch.exp(logp - t("logp_old"))
    objective = torch.mean(ratio * t("advs")[:, 0])
    cost_s = torch.mean(ratio * t("advs")[:, 1])
    kl = _kl64(actor, ob, rows)
    g_ref = ocpo._flat_grad(objective, actor, retain_graph=True).numpy()
    b_ref = ocpo._flat_grad(-cost_s, actor, retain_graph=True).numpy()
    flat_kl = ocpo._flat_grad(kl, actor, create_graph=True)
    e, nl = eng.engine(), eng.netlist([a])
    s = torch.cuda.current_stream().cuda_stream
    errs = {}
    for mode, ref, val in ((1, g_ref, objective.item()), (2, b_ref, cost_s.item())):
        policy._head(d, mode)
        sm = policy._sums.cpu().numpy()
        assert abs(sm[mode - 1] / n - val) <= 5e-5 * max(1, abs(val))
        eng.backward([a], n)
        out = policy._vec["g"]
        _lib.check(_lib.lib.fsrl_engine_wgrad_to(ctypes.byref(e), ctypes.byref(nl), ctypes.byref(inp), n, out.data_ptr(), s))
        got = _arena_to_torch_order(actor, out.cpu().numpy(), D, H, A)
        errs[f"grad{mode}"] = np.abs(got - ref).max() / np.abs(ref).max()
    policy._head(d, 3)
    assert abs(policy._sums.cpu().numpy()[2] / n - kl.item()) <= 1e-5 + 1e-4 * abs(kl.item())
    eng.backward([a], n)
    # ---- Hessian-vector products ---------------------------------------------------------------------
    gen = torch.Generator().manual_seed(3)
    vs, hvs = [], []
    for trial in range(3):
        v_t = torch.randn(P, generator=gen).double()          # the device gets the same fp32 values
        hv_ref = (ocpo._flat_grad(torch.dot(flat_kl, v_t), actor, retain_graph=True) + 0.1 * v_t).numpy()
        v_arena = torch.from_numpy(_torch_to_arena_order(actor, v_t.float().numpy(), D, H, A)).cuda()
        hv = policy._vec["hv"]
        policy._hvp(d, v_arena, hv)
        got = _arena_to_torch_order(actor, hv.cpu().numpy(), D, H, A).astype(np.float64)
        errs[f"hv{trial}"] = np.abs(got - hv_ref).max() / np.abs(hv_ref).max()
        vs.append(v_t.numpy()); hvs.append(got)
    # reference-free properties of the device products: symmetry u.Hv = v.Hu, and at theta = theta_old
    # (Fisher information + damping) v.Hv >= damping |v|^2
    nrm = np.linalg.norm
    for i, j in ((0, 1), (1, 2)):
        scale = nrm(vs[i]) * nrm(hvs[j]) + nrm(vs[j]) * nrm(hvs[i])
        errs[f"sym{i}{j}"] = abs(vs[i] @ hvs[j] - vs[j] @ hvs[i]) / scale
    psd = min((v @ hv - 0.1 * v @ v) / (nrm(v) * nrm(hv)) for v, hv in zip(vs, hvs))
    print(f"\nhvp moved={moved} hidden={hidden} rows={n} gathered={gathered}: " +
          " ".join(f"{k}={v:.2e}" for k, v in errs.items()) + f" min (vHv - 0.1|v|^2)/(|v||Hv|)={psd:.2e} "
          f"(bounds grad {GRAD_TOL_MOVED if moved else GRAD_TOL:g}, hv / sym {HVP_TOL:g})")
    grad_tol = GRAD_TOL_MOVED if moved else GRAD_TOL
    for k, v in errs.items():
        assert v <= (grad_tol if k.startswith("grad") else HVP_TOL), (k, v)
    if not moved:
        assert psd >= -HVP_TOL, psd


@pytest.mark.parametrize("early", [False, True], ids=["10-iterations", "early-exit"])
def test_cg_solve_matches_float64_cg(early):
    """fsrl_cg_solve at 2x128 on a shuffled batch above 4096 rows against float64 CG driven by the float64
    autograd Hessian-vector product, for all 10 iterations and with a residual_tol that must stop it after
    the same iteration as the float64 run."""
    from fsrl_b200 import _lib
    from oracle import cpo as ocpo
    policy, batch, ob, actor, critics, stats = _prepare((128, 128), n_env=16)
    a = policy.arena.slots[0]
    D, H, A = a.D, a.H, a.out
    n = batch.n
    assert n > 4096
    rows, perm = _rows(n, True, seed=7)
    eng = policy._ensure_engine(n)
    eng.sync_mirror([a])
    d = policy._descriptor(batch, perm, n)
    inp = eng.make_input(batch.obs, perm)
    e, nl, s = eng.engine(), eng.netlist([a]), torch.cuda.current_stream().cuda_stream
    # the device state learn() solves in: g = grad objective, then the kl head gradient's backward cache
    eng.forward([a], inp, n, save=True)
    policy._head(d, 1)
    eng.backward([a], n)
    g = policy._vec["g"]
    _lib.check(_lib.lib.fsrl_engine_wgrad_to(ctypes.byref(e), ctypes.byref(nl), ctypes.byref(inp), n, g.data_ptr(), s))
    policy._head(d, 3)
    eng.backward([a], n)
    actor.double()
    flat_kl = ocpo._flat_grad(_kl64(actor, ob, rows), actor, create_graph=True)
    mvp = lambda v: ocpo._flat_grad(flat_kl @ v, actor, retain_graph=True) + 0.1 * v
    rhs = torch.from_numpy(_arena_to_torch_order(actor, g.cpu().numpy(), D, H, A)).double()
    x_full, res = cg64(mvp, rhs, nsteps=10, tol=0.0)
    tol, x_ref, sep = 0.0, x_full, 0.0
    if early:
        k, tol = cg_stop_tol(res)
        assert min(res[:k]) / res[k] > 1.5, res       # room for the device's fp32 residuals on both sides
        x_ref, res_stop = cg64(mvp, rhs, nsteps=10, tol=tol)
        assert len(res_stop) == k + 1
        sep = float((x_ref - x_full).norm() / x_full.norm())
        assert sep > 20 * CG_TOL, sep                    # stopping at k + 1 is visible at the tolerance
    out = policy._vec["Hinv_g"]
    policy._cg(d, g, out, nsteps=10, residual_tol=tol)
    got = torch.from_numpy(_arena_to_torch_order(actor, out.cpu().numpy(), D, H, A)).double()
    err = float((got - x_ref).norm() / x_ref.norm())
    done = float(policy._cg_state[4].item())
    bound = CG_TOL if early else CG10_TOL
    print(f"\ncg early={early} rows={n} tol={tol:.3e} residuals={[f'{r:.2e}' for r in res]}: "
          f"|x - x_ref|/|x_ref| = {err:.2e} (bound {bound:g}), stopped vs 10 iterations {sep:.2e}")
    assert done == (1.0 if early else 0.0)
    assert err <= bound


@pytest.mark.parametrize("cost_limit", [1000.0, 0.0])
def test_cpo_learn_matches_oracle(cost_limit):
    from oracle import cpo as ocpo
    policy, batch, ob, actor, critics, stats = _prepare()
    policy._cost_limit = cost_limit
    opt = torch.optim.Adam([p for c in critics for p in c.parameters()], lr=1e-3)
    np.random.seed(11)
    ostats = ocpo.learn(actor, critics, opt, ob, 99999, 2, stats["cost"], cost_limit, optim_critic_iters=3,
                        max_backtracks=10)
    np.random.seed(11)
    policy.learn(batch, batch_size=99999, repeat=2)
    st = policy.last_stats
    for k in range(2):
        assert st["loss/optim_case"][k] == ostats[k]["loss/optim_case"]
        assert abs(st["loss/step_size"][k] - ostats[k]["loss/step_size"]) < 1e-9
    for key in ("loss/kl", "loss/rew_loss", "loss/cost_loss", "loss/optim_C", "loss/optim_Q", "loss/optim_lam",
                "loss/vf0", "loss/vf1", "loss/entropy"):
        want = np.array([s[key] for s in ostats]); got = np.array(st[key])
        np.testing.assert_allclose(got[:1], want[:1], rtol=5e-3, atol=1e-5, err_msg=key)
        # the second trust-region step starts from slightly different weights (CG amplifies fp32
        # noise by the condition number of H): looser, but still the same case / step size
        np.testing.assert_allclose(got, want, rtol=0.15, atol=1e-3, err_msg=key)
    # parameters after two trust-region steps
    a = policy.arena.slots[0]
    got = _arena_to_torch_order(actor, policy.arena.theta[a.offset:a.offset + a.size].cpu().numpy(), a.D, a.H, a.out)
    want = _oracle_vec(actor)
    # two unit-norm trust-region steps (the step direction is L2-normalised, cpo.py:310)
    assert np.abs(got - want).max() < 1e-2
