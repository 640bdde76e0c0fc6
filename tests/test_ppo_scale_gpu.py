"""PPO-Lagrangian parity at the BENCHMARKED shapes (BASELINE.json c2: 2048 envs x 300 steps, 2x256 MLP,
batch 256; c5: 2x512 MLP) through the production path: gather, per-minibatch advantage statistics and the
minibatch update chain that bench.py times.

Reference arithmetic: /root/reference/fsrl/policy/ppo_lag.py:173-257 restated by oracle/ppo.py (pinned on the
reference's own PPOLagrangian.learn, tests/test_oracle_golden.py).  Three kinds of evidence:

1. the first minibatch steps of a c2-shaped epoch against the fp32 oracle at the tight tolerance of the small
   tests (rtol 3e-4), and the parameters after a complete 8-step epoch at atol 2e-5;
2. un-clipped gradients of one minibatch per parameter group against an fp64 autograd reference, H = 256 and
   H = 512, printed next to the fp32 oracle's own error (the device's 3xTF32 arithmetic is ~8x coarser: asserted
   bound 2e-5 relative per group; typical 5e-7 .. 2e-6 against 1e-7 .. 6e-7 for fp32 autograd);
3. whole trajectories (62 steps, H = 512) against the fp64 twin of the oracle: at every step the device must be
   as close to exact arithmetic as the fp32 oracle is (envelope of the fp32-vs-fp64 deviation), which replaces
   the hand-picked loose bound the 512-wide case used to carry."""
import copy

import numpy as np
import pytest
import torch

from helpers import build_ppo, oracle_nets

pytestmark = pytest.mark.gpu

KEYS = ("loss/actor_rew", "loss/actor_safety", "loss/vf0", "loss/vf1", "loss/kl", "loss/total", "loss/grad_norm")


def _collect(task, hidden, n_env, lag, max_grad_norm=0.5):
    policy, venv, buf, col = build_ppo(task, hidden=hidden, n_env=n_env, max_grad_norm=max_grad_norm)
    col.collect(n_episode=n_env)
    policy.lag_optims[0].lagrangian = lag
    actor, critics = oracle_nets(policy, hidden)
    idx = buf.sample_indices(0)
    batch = policy.process_fn(None, buf, idx)
    g = lambda t: t.detach().cpu().numpy().copy()
    ob = dict(obs=g(batch.obs), act=g(batch.act), advs=g(batch.advs), rets=g(batch.rets), values=g(batch.values),
              logp_old=g(batch.logp_old))
    return policy, batch, ob, actor, critics


def _sub_batch(policy, batch, n):
    """The first n rows of a processed batch as a batch of its own (contiguous copies)."""
    from fsrl_b200.policy.base_policy import DeviceBatch
    b = DeviceBatch()
    b.n = n
    b.obs, b.act, b.logp_old = batch.obs[:n].contiguous(), batch.act[:n].contiguous(), batch.logp_old[:n].contiguous()
    b.v, b.adv, b.ret = batch.v[:, :n].contiguous(), batch.adv[:, :n].contiguous(), batch.ret[:, :n].contiguous()
    b.values, b.rets, b.advs = b.v.t(), b.ret.t(), b.adv.t()
    return b


def _adam(actor, critics, lr=5e-4):
    return torch.optim.Adam([p for m in [actor] + critics for p in m.parameters()], lr=lr)


def _params(nets):
    out = []
    for m in nets:
        for l in m.body.layers:
            out += [l.weight.detach().reshape(-1), l.bias.detach().reshape(-1)]
        head = m.mu if hasattr(m, "mu") else m.last
        out += [head.weight.detach().reshape(-1), head.bias.detach().reshape(-1)]
        if hasattr(m, "sigma_param"):
            out.append(m.sigma_param.detach().reshape(-1))
    return torch.cat(out).double().numpy()


def _product_params(policy):
    from test_ppo_gpu import _product_params as pp
    return pp(policy).astype(np.float64)


def _assert_params_within_fp32_noise(policy, nets32, actor, critics, osub, lag, seed, bs=256, lr=5e-4):
    """Parameters after a short epoch, next to the fp64 twin of the oracle.  The device GEMMs are 3xTF32: every fp32
    operand is split into two tf32 halves and a_lo*b_lo is dropped, i.e. ~2^-21 relative error per product against 2^-24
    for an fp32 FMA chain.  Losses and gradient norms do not see the difference (asserted at rtol 3e-4 by the callers), but
    Adam's normalisation m / (sqrt(v) + eps) turns absolute gradient noise of ~1e-9 on elements whose gradient nearly
    cancels (|g| ~ eps = 1e-8) into parameter steps of a sizeable fraction of lr.  Hence the statement that is asserted:
    all but a 1e-3 share of the elements agree with exact arithmetic to 2e-5, and no element is off by more than half
    the distance Adam can move it (lr per step).  The fp32 oracle's own distance is printed beside the device's."""
    from oracle import ppo as oppo
    a64, c64 = copy.deepcopy(actor).double(), [m.double() for m in copy.deepcopy(critics)]
    o64 = {k: v.astype(np.float64) for k, v in osub.items()}
    np.random.seed(seed)
    n_steps = len(oppo.learn(a64, c64, _adam(a64, c64, lr), o64, bs, 1, lag, max_grad_norm=0.5, target_kl=1e9))
    p64, p32, pdev = _params([a64] + c64), _params(nets32), _product_params(policy)
    e32, edev = np.abs(p32 - p64), np.abs(pdev - p64)
    print("\nmax |param - fp64| after %d steps: device %.3e, fp32 oracle %.3e; share of elements off by > 2e-5: device %.2e, "
          "oracle %.2e; median |param - fp64|: device %.2e, oracle %.2e"
          % (n_steps, edev.max(), e32.max(), (edev > 2e-5).mean(), (e32 > 2e-5).mean(), np.median(edev), np.median(e32)))
    assert (edev > 2e-5).mean() <= 1e-3, (edev > 2e-5).mean()
    assert edev.max() <= 0.5 * lr * n_steps, edev.max()
    assert np.median(edev) <= 1e-7, np.median(edev)


def test_c2_shape_first_steps_and_epoch_parameters():
    """c2: SafetyCarCircle-v0, 2048 envs x 300 steps = 614 400 rows, 2x256 MLP, batch 256, grad clip 0.5."""
    from oracle import ppo as oppo
    lag = 0.3
    policy, batch, ob, actor, critics = _collect("SafetyCarCircle-v0", (256, 256), 2048, lag)
    assert batch.n == 2048 * 300
    # (a) first 8 of the 2 400 minibatch steps of one repeat
    a1, c1 = copy.deepcopy(actor), copy.deepcopy(critics)
    np.random.seed(77)
    ostats = oppo.learn(a1, c1, _adam(a1, c1), ob, 256, 1, lag, max_grad_norm=0.5, target_kl=1e9, max_steps=8)
    sd0 = copy.deepcopy(policy.state_dict())
    np.random.seed(77)
    policy._target_kl = 1e9
    policy.learn(batch, batch_size=256, repeat=1)
    st = policy.last_stats
    assert len(st["loss/kl"]) == 2400
    for key in KEYS:
        want = np.array([s[key] for s in ostats])
        np.testing.assert_allclose(np.asarray(st[key])[:8], want, rtol=3e-4, atol=3e-6, err_msg=key)
    assert np.isfinite(_product_params(policy)).all()
    # (b) a complete epoch of 8 minibatches at the same widths: parameters after the 8 Adam steps
    policy.load_state_dict(sd0)
    policy.optim.m.zero_(); policy.optim.v.zero_(); policy.optim.step_count = 0
    n = 8 * 256
    sub = _sub_batch(policy, batch, n)
    osub = {k: v[:n].copy() for k, v in ob.items()}
    a2, c2 = copy.deepcopy(actor), copy.deepcopy(critics)
    np.random.seed(78)
    ostats = oppo.learn(a2, c2, _adam(a2, c2), osub, 256, 1, lag, max_grad_norm=0.5, target_kl=1e9)
    np.random.seed(78)
    policy.learn(sub, batch_size=256, repeat=1)
    st = policy.last_stats
    for key in KEYS:
        want = np.array([s[key] for s in ostats])
        np.testing.assert_allclose(np.asarray(st[key]), want, rtol=3e-4, atol=3e-6, err_msg=key)
    _assert_params_within_fp32_noise(policy, [a2] + c2, actor, critics, osub, lag, 78)


def test_persistent_path_small_epoch_matches_oracle():
    """64 envs x 300 steps = 75 minibatches of 256 rows through the persistent wgmma launch
    (csrc/ppo_persist.cu): the gate must select it, and the first 8 steps / the parameters after a complete
    8-step epoch must match the fp32 oracle like the three-launch chain does."""
    import ctypes
    from fsrl_b200 import _lib
    from oracle import ppo as oppo
    lag = 0.3
    policy, batch, ob, actor, critics = _collect("SafetyCarCircle-v0", (256, 256), 64, lag)
    policy._ensure_update_state(256, batch.n, 1)
    u = policy._descriptor(batch, torch.zeros(batch.n, dtype=torch.int32, device="cuda"))
    assert _lib.lib.fsrl_ppo_persist_active(ctypes.byref(u), batch.n, 256) == 1
    sd0 = copy.deepcopy(policy.state_dict())
    a1, c1 = copy.deepcopy(actor), copy.deepcopy(critics)
    np.random.seed(31)
    ostats = oppo.learn(a1, c1, _adam(a1, c1), ob, 256, 1, lag, max_grad_norm=0.5, target_kl=1e9, max_steps=8)
    np.random.seed(31)
    policy._target_kl = 1e9
    policy.learn(batch, batch_size=256, repeat=1)
    st = policy.last_stats
    assert len(st["loss/kl"]) == 75
    for key in KEYS:
        want = np.array([s[key] for s in ostats])
        np.testing.assert_allclose(np.asarray(st[key])[:8], want, rtol=3e-4, atol=3e-6, err_msg=key)
    policy.load_state_dict(sd0)
    policy.optim.m.zero_(); policy.optim.v.zero_(); policy.optim.step_count = 0
    n = 8 * 256
    sub = _sub_batch(policy, batch, n)
    osub = {k: v[:n].copy() for k, v in ob.items()}
    a2, c2 = copy.deepcopy(actor), copy.deepcopy(critics)
    np.random.seed(32)
    oppo.learn(a2, c2, _adam(a2, c2), osub, 256, 1, lag, max_grad_norm=0.5, target_kl=1e9)
    np.random.seed(32)
    policy.learn(sub, batch_size=256, repeat=1)
    _assert_params_within_fp32_noise(policy, [a2] + c2, actor, critics, osub, lag, 32)


def _group_names(policy):
    names = []
    for i in range(1 + policy.critics_num):
        p = "actor" if i == 0 else "critic%d" % (i - 1)
        names += [p + ".W1", p + ".b1", p + ".W2", p + ".b2", p + ".W3", p + ".b3"]
        if i == 0:
            names.append(p + ".log_sigma")
    return names


def _device_gradients(policy, batch, n):
    """Un-clipped gradient of ONE minibatch (the whole batch of n rows), read back from Adam's first moment:
    from zero state m = (1 - beta1) * g.  Returned in the oracle's parameter order, one array per group."""
    policy._ensure_update_state(n, n, 1)
    policy.optim.m.zero_(); policy.optim.v.zero_(); policy.optim.step_count = 0
    policy._target_kl = 1e9
    policy.learn(batch, batch_size=n, repeat=1)
    m = policy.optim.m.detach().cpu().double().numpy() / (1.0 - policy.optim.param_groups[0]["betas"][0])
    out = []
    for s in policy.arena.slots:
        w1, b1, w2, b2, w3, b3, ex = s.offsets()
        D, H, o = s.D, s.H, s.out
        out += [m[w1:w1 + D * H].reshape(D, H).T.reshape(-1), m[b1:b1 + H], m[w2:w2 + H * H].reshape(H, H).T.reshape(-1),
                m[b2:b2 + H], m[w3:w3 + H * o].reshape(H, o).T.reshape(-1), m[b3:b3 + o]]
        if s.n_extra:
            out.append(m[ex:ex + s.n_extra])
    return out


@pytest.mark.parametrize("hidden,task,lag", [((256, 256), "SafetyCarCircle-v0", 0.3),
                                             ((512, 512), "SafetyAntCircle-v0", 0.8),
                                             ((512, 512), "SafetyPointGoal1Gymnasium-v0", 0.4)])
def test_gradients_against_fp64_autograd(hidden, task, lag):
    """dW1, db1, dW2, db2, dW3, db3 (+ d log sigma) of every network for one 256-row minibatch: the device
    (3xTF32 tensor-core GEMMs, fp32 accumulation) vs fp64 autograd, next to the fp32 oracle vs fp64."""
    from oracle import ppo as oppo
    policy, batch, ob, actor, critics = _collect(task, hidden, 4, lag, max_grad_norm=None)
    n = 256
    sub = _sub_batch(policy, batch, n)
    osub = {k: v[:n].copy() for k, v in ob.items()}
    g32, g64 = [], []
    a, c = copy.deepcopy(actor), copy.deepcopy(critics)
    np.random.seed(5)
    oppo.learn(a, c, _adam(a, c), osub, n, 1, lag, max_grad_norm=None, target_kl=1e9, grads_out=g32)
    a, c = copy.deepcopy(actor).double(), [m.double() for m in copy.deepcopy(critics)]
    o64 = {k: v.astype(np.float64) for k, v in osub.items()}
    np.random.seed(5)
    oppo.learn(a, c, _adam(a, c), o64, n, 1, lag, max_grad_norm=None, target_kl=1e9, grads_out=g64)
    np.random.seed(5)
    gdev = _device_gradients(policy, sub, n)
    names = _group_names(policy)

    def in_group_order(grads, nets):
        # oracle gradients come in parameters() order (a module's own Parameters -- log sigma -- before its children's)
        table = {"body.layers.0.weight": 0, "body.layers.0.bias": 1, "body.layers.1.weight": 2, "body.layers.1.bias": 3,
                 "mu.weight": 4, "mu.bias": 5, "last.weight": 4, "last.bias": 5, "sigma_param": 6}
        out, k = [], 0
        for m in nets:
            named = [n for n, _ in m.named_parameters()]
            slots = {table[n]: grads[k + i] for i, n in enumerate(named)}
            out += [slots[j] for j in sorted(slots)]
            k += len(named)
        return out

    g32, g64 = in_group_order(g32, [actor] + critics), in_group_order(g64, [actor] + critics)
    assert len(gdev) == len(g32) == len(g64) == len(names)
    rows = []
    for name, d, f, x in zip(names, gdev, g32, g64):
        x = x.reshape(-1).numpy(); f = f.reshape(-1).double().numpy()
        scale = np.linalg.norm(x) + 1e-30
        e_dev, e_32 = np.linalg.norm(d - x) / scale, np.linalg.norm(f - x) / scale
        rows.append((name, e_dev, e_32))
    print("\n%-18s %12s %12s" % ("group", "device/fp64", "fp32/fp64"))
    for r in rows:
        print("%-18s %12.3e %12.3e" % r)
    for name, e_dev, e_32 in rows:
        # The fp32 autograd reference sits near 1e-7 from fp64 (printed above).  The persistent wgmma launch (H = 256
        # case; 3xTF32 with the cross terms in their own accumulator, DESIGN.md 3a) and the three-launch chain (H = 512
        # cases, mma.sync 3xTF32, one accumulator) stay a few times above it; the chain reaches 1e-5 where the value loss
        # gradient 2 (v - ret) cancels (|v - ret| << |v| amplifies the forward error of v into every group of that critic
        # alike).  A wrong term in a kernel shows up at 1e-2 and above.
        assert e_dev <= (3e-6 if hidden == (256, 256) else 2e-5), (name, e_dev, e_32)


@pytest.mark.parametrize("hidden,task,lag", [((512, 512), "SafetyPointGoal1Gymnasium-v0", 0.4),
                                             ((256, 256), "SafetyCarCircle-v0", 0.0)])
def test_trajectory_stays_within_fp32_envelope_of_fp64(hidden, task, lag):
    """62 optimiser steps (4 envs, batch 64: the case whose tolerance had been loosened for H = 512).  Two fp32
    implementations of the same update drift apart through rounding alone; the fp64 twin of the oracle measures
    that drift.  env32[t] = max_{s<=t} |oracle32[s] - oracle64[s]|; the device must satisfy
    |device[t] - oracle64[t]| <= 16 * env32[t] + 3e-4 |oracle64[t]| + 3e-6 at EVERY step and for every logged key
    (the device's 3xTF32 products are ~8x coarser than an fp32 FMA chain, DESIGN.md 3a; 16 leaves a factor 2), and the final
    parameters obey the same rule."""
    from oracle import ppo as oppo
    policy, batch, ob, actor, critics = _collect(task, hidden, 4, lag)
    bs = 64
    a32, c32 = copy.deepcopy(actor), copy.deepcopy(critics)
    np.random.seed(123)
    s32 = oppo.learn(a32, c32, _adam(a32, c32), ob, bs, 1, lag, max_grad_norm=0.5, target_kl=1e9)
    a64, c64 = copy.deepcopy(actor).double(), [m.double() for m in copy.deepcopy(critics)]
    o64 = {k: v.astype(np.float64) for k, v in ob.items()}
    np.random.seed(123)
    s64 = oppo.learn(a64, c64, _adam(a64, c64), o64, bs, 1, lag, max_grad_norm=0.5, target_kl=1e9)
    np.random.seed(123)
    policy._target_kl = 1e9
    policy.learn(batch, batch_size=bs, repeat=1)
    st = policy.last_stats
    keys = [k for k in KEYS if k != "loss/actor_safety" or lag > 0]
    for key in keys:
        w64 = np.array([s[key] for s in s64]); w32 = np.array([s[key] for s in s32]); got = np.asarray(st[key], dtype=np.float64)
        assert len(got) == len(w64)
        env = np.maximum.accumulate(np.abs(w32 - w64))
        bound = 16.0 * env + 3e-4 * np.abs(w64) + 3e-6
        bad = np.abs(got - w64) > bound
        assert not bad.any(), (key, np.nonzero(bad)[0][:5], np.abs(got - w64)[bad][:5], bound[bad][:5])
    p64, p32, pdev = _params([a64] + c64), _params([a32] + c32), _product_params(policy)
    e32, edev = np.abs(p32 - p64).max(), np.abs(pdev - p64).max()
    print("\nmax |param - fp64|: device %.3e, fp32 oracle %.3e" % (edev, e32))
    assert edev <= 16.0 * e32 + 2e-6, (edev, e32)
