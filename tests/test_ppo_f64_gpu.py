"""The PPO-Lagrangian update on the device, stage by stage, against float64 (the stage functions of tests/ppo64.py,
which tests/test_ppo_f64_host.py ties to the oracle's autograd).

The three-launch chain (csrc/ppo.cu) keeps one minibatch's activations in the policy's scratch: per net
h1 | h2 | dz1 | dz2 as [bmax][H], then dout as [bmax][16]; scratch row i is row perm[mb_off + i] of the batch.
Each stage is fed what the device left from the stage before it, so that an error points at one kernel:

  moments   ppo_adv_stats_kernel: mean and 1 / std of every advantage column of the minibatch, (0, 1) without
            advantage normalisation
  forward   ppo_fwd_kernel: h1, h2 with the device's ReLU masks
  head      ppo_bwd_kernel's loss gradient: dout at the head outputs recomputed from the device's h2
  backward  ppo_bwd_kernel: dz2 from the device's dout, dz1 from the device's dz2
  wgrad     ppo_wgrad(_adam)_kernel: every parameter group as a contraction of the device's x, h1, h2, dz1, dz2, dout,
            read back from Adam's moments; the global norm and the clip scale
  adam      theta and the second moment against helpers.adam64 fed the device's own gradient
  stats     loss/actor_rew, actor_safety, kl, vf_i, entropy and total against float64 sums

The persistent launch (csrc/ppo_persist.cu) writes no scratch: its gradient, statistics and Adam step are checked
against the float64 update of the whole minibatch.  With Adam's betas at 0 the first moment after any step is that
step's (clipped) gradient and v = m^2, so theta before the last step follows from theta, m and v after it.

Every bound is a tolerance times a measured scale: the same expression evaluated on the magnitudes of its terms.
The synthetic batches put the ratio exp(logp - logp_old) on both sides of the clip range and of the dual clip, and the
stored values on both sides of the value clip, each a clear margin away from the kink; the head stage asserts that
margin before it compares.  The last row of every minibatch carries a large advantage, so that a dropped, doubled or
misplaced row moves the weight gradient far past its bound."""
import copy
import ctypes
import math

import numpy as np
import pytest
import torch

import ppo64
from helpers import adam64, synthetic_ring

pytestmark = pytest.mark.gpu

FLT_MIN = float(np.finfo(np.float32).tiny)
LR = 5e-4
# Bounds: about 10x the worst value observed over all cases on an H100 80GB HBM3 (700 W power limit), given in each
# comment; every case prints its errors.
MOM_TOL = 1e-6       # advantage mean (relative to mean |adv|) and 1 / std (relative): 1.0e-7
FWD_TOL = 7e-6       # h1, h2 against float64 with device masks, relative to the magnitude chain: 6.5e-7
DOUT_TOL = 3e-5      # head dout, relative to the element's magnitude: 2.4e-6
BWD_TOL = 3e-5       # dz2, dz1 from the device's dout / dz2, relative to the magnitude of the product: 3.2e-6
GRAD_TOL = 9e-6      # weight gradients from the device's activations, relative to |X|^T |G|: 8.6e-7
NORM_TOL = 6e-6      # loss/grad_norm, relative to the norm of |X|^T |G| (chain) or to itself (persistent): 6.2e-7
STAT_TOL = 8e-6      # statistics, relative to the sum of the magnitudes of their terms: 7.8e-7
PGRAD_TOL = 3e-6     # persistent launch: max |g - g64| / max |X|^T |G| per parameter group, natural masks: 2.2e-7
ULP_TOL = 32.0       # Adam's theta and v in fp32 ulps of their scale: 3.2
GAE_TOL = 5e-7       # recomputed advantages / returns, relative to the largest value, return and reward: 4.5e-8
KINK = 1e-3          # the float64 ratio / value offset is at least this far from every kink it can meet


class _BoxEnv:
    """The two spaces an agent reads: a user env with Box(-high, high) actions."""

    def __init__(self, D, A, high):
        from fsrl_b200.spaces import Box
        self.observation_space = Box(-np.inf, np.inf, (D,), np.float32)
        self.action_space = Box(-high, high, (A,), np.float32)


def _policy(D, A, H, C=2, high=1.0, bounded=True, lag=0.7, betas=None, persist=False, seed=3, **kw):
    if C == 2:
        from fsrl_b200.agent import PPOLagAgent
        p = PPOLagAgent(_BoxEnv(D, A, high), seed=seed, hidden_sizes=(H, H), unbounded=not bounded, lr=LR,
                        **kw).policy
        if p.lag_optims:
            p.lag_optims[0].lagrangian = lag
    else:
        from torch.distributions import Independent, Normal
        from fsrl_b200 import nets
        from fsrl_b200.agent.ppo_lag_agent import init_actor_critic
        from fsrl_b200.optim import FusedAdam
        from fsrl_b200.policy import PPOLagrangian
        torch.manual_seed(seed)
        env = _BoxEnv(D, A, high)
        actor = nets.ActorProb(nets.Net(D, hidden_sizes=(H, H)), A, max_action=high, unbounded=not bounded)
        critics = [nets.Critic(nets.Net(D, hidden_sizes=(H, H)))]
        torch.nn.init.constant_(actor.sigma_param, -0.5)
        init_actor_critic(actor, critics)
        actor.device = "cuda"
        p = PPOLagrangian(actor, critics, FusedAdam(lr=LR), lambda *l: Independent(Normal(*l), 1),
                          observation_space=env.observation_space, action_space=env.action_space, **kw)
        p.arena
    if betas is not None:
        from fsrl_b200.optim import FusedAdam
        p.optim = FusedAdam(lr=LR, betas=betas)
    p._persist_off = not persist
    p._target_kl = 1e9
    assert p.actor._max == high and p.actor._unbounded == (not bounded)
    return p


def _opts(p):
    use_saf = p.use_lagrangian and p.critics_num > 1
    return ppo64.Opts(A=p.arena.slots[0].out, C=p.critics_num, max_action=float(p.actor._max),
                      bounded=not p.actor._unbounded, eps_clip=p._eps_clip, dual_clip=float(p._dual_clip or 0.0),
                      vf_coef=p._weight_vf, value_clip=p._value_clip, norm_adv=p._norm_adv, use_saf=use_saf,
                      lag=p.lagrangians()[0] if use_saf else 0.0,
                      resc=p.rescaling_factor() if p.use_lagrangian else 1.0)


def _d(t):
    return t.detach().double()


def _split(p, vec):
    """a flat arena vector as one dict per net in the layout of ppo64"""
    out = []
    for s in p.arena.slots:
        w1, b1, w2, b2, w3, b3, ex = s.offsets()
        P = dict(w1=vec[w1:b1].view(s.D, s.H), b1=vec[b1:w2], w2=vec[w2:b2].view(s.H, s.H), b2=vec[b2:w3],
                 w3=vec[w3:b3].view(s.H, s.out), b3=vec[b3:ex])
        if s.n_extra:
            P["ls"] = vec[ex:ex + s.n_extra]
        out.append(P)
    return out


# ratio bands clear of 1 +- eps_clip (0.2) and of the dual clip (1.5); value offsets clear of +- eps_clip
RATIO_BANDS = ((0.35, 0.75), (0.83, 1.17), (1.25, 1.42), (1.58, 2.4))
VOFF_BANDS = ((0.0, 0.15), (0.25, 0.6))


def _bands(bands, n, g):
    k = torch.randint(0, len(bands), (n,), generator=g, device="cuda")
    lo = torch.tensor([b[0] for b in bands], device="cuda", dtype=torch.float64)[k]
    hi = torch.tensor([b[1] for b in bands], device="cuda", dtype=torch.float64)[k]
    return lo + (hi - lo) * torch.rand(n, generator=g, device="cuda", dtype=torch.float64)


def _batch(p, n, seed, trap_rows=()):
    """A DeviceBatch of n synthetic rows at the policy's current parameters: actions drawn from the policy, logp_old
    set so that the ratios fall in RATIO_BANDS, stored values VOFF_BANDS away from the critics, and advantages of
    40 / -30 on the batch rows trap_rows."""
    from fsrl_b200.policy.base_policy import DeviceBatch
    s0 = p.arena.slots[0]
    D, A, C = s0.D, s0.out, p.critics_num
    o = _opts(p)
    g = torch.Generator(device="cuda").manual_seed(seed)
    obs = torch.randn(n, D, generator=g, device="cuda")
    nets = _split(p, _d(p.arena.theta))
    outs = [ppo64.forward(P, _d(obs))[4] for P in nets]
    mu = o.max_action * torch.tanh(outs[0]) if o.bounded else outs[0]
    ls = nets[0]["ls"]
    act = (mu + ls.exp() * torch.randn(n, A, generator=g, device="cuda", dtype=torch.float64)).float()
    logp = (-0.5 * ((_d(act) - mu) / ls.exp()) ** 2 - ls - ppo64.LOG_SQRT_2PI).sum(1)
    sign = lambda: torch.randint(0, 2, (C, n), generator=g, device="cuda").double() * 2 - 1
    v = torch.stack([q[:, 0] for q in outs[1:]])
    b = DeviceBatch()
    b.n = n
    b.obs, b.act = obs.contiguous(), act.contiguous()
    b.logp_old = (logp - _bands(RATIO_BANDS, n, g).log()).float().contiguous()
    b.v = (v + sign() * _bands(VOFF_BANDS, C * n, g).view(C, n)).float().contiguous()
    b.ret = (v + torch.randn(C, n, generator=g, device="cuda", dtype=torch.float64)).float().contiguous()
    b.adv = (1.5 * torch.randn(C, n, generator=g, device="cuda") + 0.2).contiguous()
    for r in trap_rows:
        b.adv[0, r] = 40.0
        if C > 1:
            b.adv[1, r] = -30.0
    b.values, b.rets, b.advs = b.v.t(), b.ret.t(), b.adv.t()
    return b


def _learn(p, batch, bs, seed, repeat=1):
    np.random.seed(seed)
    p.learn(batch, batch_size=bs, repeat=repeat)
    return {k: np.asarray(v, dtype=np.float64) for k, v in p.last_stats.items()}


def _perm(seed, n):
    return torch.from_numpy(np.random.RandomState(seed).permutation(n)).cuda()


def _scratch(p, net, B):
    """h1, h2, dz1, dz2 [B][H] and dout [B][16] of the chain's last minibatch, in float64"""
    H, bmax = p.arena.slots[0].H, p._bmax
    base = net * bmax * (4 * H + 16)
    sc = p._scratch
    blk = [_d(sc[base + k * bmax * H:base + (k + 1) * bmax * H].view(bmax, H)[:B]) for k in range(4)]
    return blk + [_d(sc[base + 4 * bmax * H:base + 4 * bmax * H + bmax * 16].view(bmax, 16)[:B])]


def _grad_beta0(p):
    """the last step's gradient under betas (0, 0): |g| = sqrt(v) (v = fl(g^2), exact to half an ulp of g), sign of m"""
    m, v = _d(p.optim.m), _d(p.optim.v)
    return torch.where(v > 0, torch.copysign(v.sqrt(), m), m)


def _theta_before_beta0(p):
    """theta before the last Adam step of a run with betas (0, 0): theta_t = theta_{t-1} - lr m / (sqrt(v) + eps)"""
    m, v = _d(p.optim.m), _d(p.optim.v)
    return _d(p.arena.theta) + LR * m / (v.sqrt() + p.optim.param_groups[0]["eps"])


def _rows(batch, idx):
    return ppo64.Rows(act=_d(batch.act[idx]), lpo=_d(batch.logp_old[idx]), adv=_d(batch.adv[:, idx]),
                      ret=_d(batch.ret[:, idx]), values=_d(batch.v[:, idx]))


def _err(got, ref, scale, floor=0.0):
    got, ref, scale = (torch.as_tensor(v, dtype=torch.float64, device="cuda") for v in (got, ref, scale))
    tiny = torch.finfo(torch.float64).tiny
    return float((torch.clamp((got - ref).abs() - floor, min=0.0) / torch.clamp(scale, min=tiny)).max())


def _kinks(o, stats, R, v_dev):
    """the float64 distance of every row from the kinks of the loss, relative"""
    ratio, ar = stats["ratio"], stats["ar"]
    d = torch.minimum((ratio - (1 - o.eps_clip)).abs(), (ratio - (1 + o.eps_clip)).abs())
    if o.dual_clip:
        d = torch.where(ar < 0, torch.minimum(d, (ratio - o.dual_clip).abs()), d)
    out = float(d.min())
    if o.value_clip:
        for i, v in enumerate(v_dev):
            off = v - R.values[i]
            out = min(out, float(torch.minimum((off - o.eps_clip).abs(), (off + o.eps_clip).abs()).min()))
    return out


def _stat_errs(o, stats, st, row, errs):
    keys = ["actor_rew", "kl", "entropy", "total"] + ["vf%d" % i for i in range(o.C)] + \
        (["actor_safety"] if o.use_saf else [])
    for k in keys:
        errs["stat." + k] = abs(float(st["loss/" + k][row]) - stats[k]) / max(stats["s_" + k], FLT_MIN)


def _check_chain(p, batch, theta, idx, mb, g_dev, st, row, clip=None):
    """stages moments .. wgrad and the statistics of the chain's last minibatch (batch rows idx, minibatch mb of the
    repeat, parameters theta before its step); g_dev = the device's gradient of that step"""
    o = _opts(p)
    B, C = len(idx), o.C
    nets = _split(p, theta)
    x, R = _d(batch.obs[idx]), _rows(batch, idx)
    errs = {}
    # moments
    ms = _d(p._mb_stats[4 * mb:4 * mb + 4].view(2, 2))[:C]
    mean64, rstd64 = ppo64.adv_stats(R.adv, o.norm_adv)
    if o.norm_adv:
        for c in range(C):
            errs["mom.mean%d" % c] = float((ms[c, 0] - mean64[c]).abs() / R.adv[c].abs().mean())
            errs["mom.rstd%d" % c] = float((ms[c, 1] - rstd64[c]).abs() / rstd64[c])
    else:
        assert torch.equal(ms, torch.tensor([[0.0, 1.0]] * C, dtype=torch.float64, device="cuda"))
    mean_d, rstd_d = ms[:, 0], ms[:, 1]
    # forward, and the head outputs recomputed from the device's h2
    saved = [_scratch(p, i, B) for i in range(len(nets))]
    outs = []
    for i, P in enumerate(nets):
        h1, h2 = saved[i][0], saved[i][1]
        masks = ((h1 > 0).double(), (h2 > 0).double())
        _, _, h1r, h2r, _ = ppo64.forward(P, x, masks)
        h1m, h2m, _ = ppo64.forward_mag(P, x, masks)
        errs["fwd.h1.%d" % i] = _err(h1, h1r, h1m)
        errs["fwd.h2.%d" % i] = _err(h2, h2r, h2m)
        outs.append(h2 @ P["w3"] + P["b3"])
    # head
    douts, dmags, stats = ppo64.head(o, outs, nets[0]["ls"], R, mean_d, rstd_d)
    margin = _kinks(o, stats, R, [q[:, 0] for q in outs[1:]])
    assert margin > KINK, margin
    A = o.A
    for i in range(len(nets)):
        dd, w = saved[i][4], (2 * A if i == 0 else 1)
        assert (dd[:, w:] == 0).all()
        errs["head.%d" % i] = _err(dd[:, :w], douts[i], dmags[i], FLT_MIN)
    # backward and weight gradients
    gd = _split(p, g_dev)
    gref, gmag = [], []
    for i, P in enumerate(nets):
        h1, h2, dz1, dz2, dout = saved[i]
        nout, n_extra = (A, A) if i == 0 else (1, 0)
        dz2r, dz2m = ppo64.backward_dz2(P, dout, nout, h2)
        dz1r, dz1m = ppo64.backward_dz1(P, dz2, h1)
        errs["bwd.dz2.%d" % i] = _err(dz2, dz2r, dz2m, FLT_MIN)
        errs["bwd.dz1.%d" % i] = _err(dz1, dz1r, dz1m, FLT_MIN)
        gref.append(ppo64.wgrad(x, h1, h2, dz1, dz2, dout, nout, n_extra))
        gmag.append(ppo64.wgrad_mag(x, h1, h2, dz1, dz2, dout, nout, n_extra))
    gn = math.sqrt(sum(float((g ** 2).sum()) for G in gref for g in G.values()))
    gn_mag = math.sqrt(sum(float((g ** 2).sum()) for G in gmag for g in G.values()))
    scale = 1.0
    if clip:
        scale = min(clip / (gn + 1e-6), 1.0)
        assert scale < 0.9, scale                       # the clip bites
    errs["norm"] = abs(float(st["loss/grad_norm"][row]) - gn) / gn_mag
    for i in range(len(nets)):
        for k in gref[i]:
            errs["wgrad.%d.%s" % (i, k)] = _err(gd[i][k], scale * gref[i][k], scale * gmag[i][k], B * FLT_MIN)
    _stat_errs(o, stats, st, row, errs)
    return errs, margin


TOLS = {"mom": MOM_TOL, "fwd": FWD_TOL, "head": DOUT_TOL, "bwd": BWD_TOL, "wgrad": GRAD_TOL, "norm": NORM_TOL,
        "stat": STAT_TOL, "pgrad": PGRAD_TOL, "adam": ULP_TOL}


def _report(label, errs):
    bounds = {k: TOLS[k.split(".")[0]] for k in errs}
    worst = {}
    for k, v in errs.items():
        st = k.split(".")[0]
        worst[st] = max(worst.get(st, 0.0), v)
    print(f"\n{label}: " + " ".join(f"{k}={v:.2e}/{TOLS[k]:.0e}" for k, v in worst.items()), end="")
    bad = {k: v for k, v in errs.items() if not v <= bounds[k]}
    assert not bad, bad


def _ulps(got, want, scale):
    sp = torch.from_numpy(np.spacing(scale.abs().float().cpu().numpy())).double().cuda()
    return float(((got - want).abs() / sp).max())


# ---- 1. the chain, one minibatch per case ----------------------------------------------------------------------
# id: (H, n, batch_size, A, D, policy options); n in [bs, 2 bs) is one minibatch (merged when n > bs).  The tile rows
# MlpTile<H>::R are 64 / 32 / 16 / 16; the weight-gradient roles stream 128-row chunks.
CHAIN = {
    "h64-n2": (64, 2, 2, 2, 8, {}),
    "h64-n3": (64, 3, 2, 3, 5, {}),
    "h64-n63": (64, 63, 32, 1, 1, {}),
    "h64-n64": (64, 64, 64, 2, 34, {}),
    "h64-n65": (64, 65, 33, 8, 79, {}),
    "h128-n31": (128, 31, 16, 2, 8, {}),
    "h128-n32": (128, 32, 32, 3, 76, {}),
    "h128-n33": (128, 33, 17, 8, 5, {}),
    "h128-n127-D80": (128, 127, 64, 2, 80, {}),
    "h128-n128": (128, 128, 128, 1, 34, {}),
    "h128-n129": (128, 129, 65, 2, 8, dict(max_grad_norm=0.02)),
    "h256-n15": (256, 15, 8, 2, 8, {}),
    "h256-n16": (256, 16, 16, 8, 1, {}),
    "h256-n17": (256, 17, 9, 3, 34, {}),
    "h256-n255": (256, 255, 128, 2, 79, dict(max_grad_norm=0.02)),
    "h512-n15": (512, 15, 8, 2, 8, {}),
    "h512-n16-D80": (512, 16, 16, 2, 80, {}),
    "h512-n17": (512, 17, 9, 1, 5, {}),
    "h512-n4500": (512, 4500, 2251, 2, 60, {}),
    "max2.5": (64, 200, 101, 3, 11, dict(high=2.5)),
    "unbounded": (128, 200, 101, 2, 11, dict(bounded=False)),
    "one-critic": (64, 200, 101, 2, 11, dict(C=1)),
    "no-lagrangian": (128, 200, 101, 2, 11, dict(use_lagrangian=False)),
    "no-rescaling": (64, 200, 101, 2, 11, dict(rescaling=False)),
    "no-adv-norm": (64, 200, 101, 2, 11, dict(advantage_normalization=False)),
    "vclip-dclip": (128, 200, 101, 3, 11, dict(value_clip=True, dual_clip=1.5, reward_normalization=True)),
    "lag0": (64, 200, 101, 2, 11, dict(lag=0.0)),
    "adam-t10001": (64, 200, 101, 2, 11, {}),
}


@pytest.mark.parametrize("name", list(CHAIN))
def test_chain_stages(name):
    H, n, bs, A, D, kw = CHAIN[name]
    clip = kw.get("max_grad_norm")
    p = _policy(D, A, H, **kw)
    seed = 11 + n + A + D
    perm = _perm(seed, n)
    batch = _batch(p, n, seed, trap_rows=[int(perm[n - 1])])
    theta0 = _d(p.arena.theta).clone()
    p._ensure_update_state(bs, n, 1)
    t0, m0, v0 = 0, torch.zeros_like(theta0), torch.zeros_like(theta0)
    if name == "adam-t10001":                      # a late step: both bias corrections near 1
        t0 = 10000
        p.optim.step_count = t0
    p.arena.grad.zero_()
    st = _learn(p, batch, bs, seed)
    assert len(st["loss/kl"]) == 1
    # the fused weight-gradient + Adam launch (H <= 256) keeps the gradient on chip; H = 512 takes the unfused one
    assert bool((p.arena.grad == 0).all()) == (H <= 256)
    b1, b2 = p.optim.param_groups[0]["betas"]
    w1 = float(np.float32(1.0 - b1))
    g_dev = m0 + (_d(p.optim.m) - m0) / w1
    errs, margin = _check_chain(p, batch, theta0, perm, 0, g_dev, st, 0, clip)
    # Adam from the device's own (clipped) gradient
    pr, _, vr = adam64(theta0, g_dev, m0, v0, t0 + 1, LR, (b1, b2), p.optim.param_groups[0]["eps"])
    errs["adam.theta"] = _ulps(_d(p.arena.theta), pr, pr.abs() + LR)
    errs["adam.v"] = _ulps(_d(p.optim.v), vr, vr)
    _report(f"chain {name} H={H} n={n} bs={bs} A={A} D={D} (kink margin {margin:.2e})", errs)


# ---- 2. steps after the first, and the merged tail ------------------------------------------------------------
@pytest.mark.parametrize("H,n,bs", [(64, 300, 128), (128, 256, 64)], ids=["tail-n300-bs128", "h128-4steps"])
def test_chain_last_step_at_recovered_parameters(H, n, bs):
    """Adam with betas (0, 0): the scratch holds the last minibatch, theta before its step is recovered from theta,
    m and v, and that minibatch (the merged 172-row tail, or the 4th of 4) is checked stage by stage."""
    A, D = 2, 8
    p = _policy(D, A, H, betas=(0.0, 0.0))
    seed = 23 + n
    perm = _perm(seed, n)
    n_mb = n // bs
    off = (n_mb - 1) * bs
    batch = _batch(p, n, seed, trap_rows=[int(perm[n - 1]), int(perm[off])])
    st = _learn(p, batch, bs, seed)
    assert len(st["loss/kl"]) == n_mb
    errs, margin = _check_chain(p, batch, _theta_before_beta0(p), perm[off:], n_mb - 1, _grad_beta0(p), st, n_mb - 1)
    _report(f"chain step {n_mb} of {n_mb} H={H} n={n} bs={bs} rows {off}..{n - 1} (kink margin {margin:.2e})", errs)


# ---- 3. the persistent launch across its gate ------------------------------------------------------------------
PERSIST = {
    "one-critic": (2, 8, dict(C=1, max_grad_norm=0.02)),
    "A1-D1": (1, 1, dict(max_grad_norm=0.02)),
    "A8-D3-unbounded": (8, 3, dict(bounded=False, max_grad_norm=0.02)),
    "A2-D40-max2": (2, 40, dict(high=2.0, max_grad_norm=0.02)),
    "no-grad-clip": (3, 8, dict(max_grad_norm=None)),
    "vclip-dclip": (2, 8, dict(value_clip=True, dual_clip=1.5, reward_normalization=True, max_grad_norm=0.02)),
    "no-adv-norm": (2, 8, dict(advantage_normalization=False, max_grad_norm=0.02)),
}


def _check_persist(p, batch, theta, idx, g_dev, st, row):
    o = _opts(p)
    x, R = _d(batch.obs[idx]), _rows(batch, idx)
    stats, gref, gmag = ppo64.gradients(o, _split(p, theta), x, R)
    clip = p._grad_norm
    gn = math.sqrt(sum(float((g ** 2).sum()) for G in gref for g in G.values()))
    scale = min(clip / (gn + 1e-6), 1.0) if clip else 1.0
    if clip:
        assert scale < 0.9, scale
    errs = {"norm": abs(float(st["loss/grad_norm"][row]) - gn) / gn}
    gd = _split(p, g_dev)
    for i in range(len(gref)):
        for k in gref[i]:
            errs["pgrad.%d.%s" % (i, k)] = float((gd[i][k] - scale * gref[i][k]).abs().max() /
                                                 (scale * gmag[i][k].max()))
    _stat_errs(o, stats, st, row, errs)
    return errs


@pytest.mark.parametrize("name", list(PERSIST))
def test_persistent_launch(name):
    """One 256-row step, then a 4-step launch whose last step is checked at the recovered parameters."""
    from fsrl_b200 import _lib
    A, D, kw = PERSIST[name]
    H, bs = 256, 256
    p = _policy(D, A, H, betas=(0.0, 0.0), persist=True, **kw)
    for n in (256, 1024):
        seed = 31 + n + A + D
        perm = _perm(seed, n)
        batch = _batch(p, n, seed, trap_rows=[int(perm[n - 1])])
        p._ensure_update_state(bs, n, 1)
        u = p._descriptor(batch, torch.zeros(n, dtype=torch.int32, device="cuda"))
        assert _lib.lib.fsrl_ppo_persist_active(ctypes.byref(u), n, bs) == 1
        theta0 = _d(p.arena.theta).clone()
        st = _learn(p, batch, bs, seed)
        k = n // bs
        assert len(st["loss/kl"]) == k
        theta = theta0 if k == 1 else _theta_before_beta0(p)
        g_dev = _grad_beta0(p)
        errs = _check_persist(p, batch, theta, perm[(k - 1) * bs:], g_dev, st, k - 1)
        if k == 1:                 # Adam with betas (0, 0) from the device's own gradient
            pr, _, vr = adam64(theta0, g_dev, 0 * g_dev, 0 * g_dev, p.optim.step_count, LR, (0.0, 0.0))
            errs["adam.theta"] = _ulps(_d(p.arena.theta), pr, pr.abs() + LR)
            errs["adam.v"] = _ulps(_d(p.optim.v), vr, vr)
        _report(f"persistent {name} A={A} D={D} step {k} of {k}", errs)


# ---- 4. recompute_advantage ------------------------------------------------------------------------------------
def _gae64(p, batch, buf, idx, theta):
    """advantages and returns [C][N] of a float64 critic pass through the oracle's dual GAE"""
    from oracle import returns
    nets = _split(p, theta)[1:]
    v = torch.stack([ppo64.forward(P, _d(batch.obs))[4][:, 0] for P in nets]).cpu().numpy()
    vn = torch.stack([ppo64.forward(P, _d(batch.obs_next))[4][:, 0] for P in nets]).cpu().numpy()
    unf = torch.isin(idx, buf.unfinished_index()).cpu().numpy()
    c = lambda t: t.detach().cpu().numpy()
    _, rets, advs = returns.dual_gae(v, vn, c(batch.rew), c(batch.cost), c(batch.terminated).astype(bool),
                                     c(batch.truncated).astype(bool), unf, p._gamma, p._lambda)
    return torch.from_numpy(np.ascontiguousarray(advs.T)).double().cuda(), \
        torch.from_numpy(np.ascontiguousarray(rets.T)).double().cuda()


def test_recompute_advantage():
    """repeat = 2 with recompute_advantage: the second repeat's advantages and returns are a float64 GAE over the
    critics as they stand after the first repeat, and the NumPy stream is consumed as without recompute."""
    D, A, H, bs, seed = 8, 2, 64, 128, 7
    p = _policy(D, A, H, recompute_advantage=True)
    buf = synthetic_ring(D, A, 8, 64, "wrapped", seed=seed)
    buf.logp.copy_(-2.0 + 0.3 * torch.randn(buf.logp.shape, device="cuda"))
    idx = buf.sample_indices(0)
    batch = p.process_fn(None, buf, idx)
    sd0 = copy.deepcopy(p.state_dict())
    theta0 = _d(p.arena.theta).clone()
    a0, r0 = _gae64(p, batch, buf, idx, theta0)
    scale = lambda a, r: float(a.abs().max() + r.abs().max() + _d(batch.rew).abs().max() + 1.0)
    errs = {"gae.check0": max(_err(batch.adv, a0, scale(a0, r0)), _err(batch.ret, r0, scale(a0, r0)))}
    # the first repeat alone: the critics the second repeat must use
    adv_first = batch.adv.clone()
    _learn(p, batch, bs, seed, repeat=1)
    theta1 = _d(p.arena.theta).clone()
    a1, r1 = _gae64(p, batch, buf, idx, theta1)
    # again from the start, both repeats
    p.load_state_dict(sd0)
    p.optim.m.zero_(); p.optim.v.zero_(); p.optim.step_count = 0
    p._mirror_dirty = True
    batch = p.process_fn(None, buf, idx)
    assert torch.equal(batch.adv, adv_first)
    _learn(p, batch, bs, seed, repeat=2)
    state = np.random.get_state()
    np.random.seed(seed)
    np.random.permutation(batch.n); np.random.permutation(batch.n)
    want = np.random.get_state()
    assert state[0] == want[0] and np.array_equal(state[1], want[1]) and state[2:] == want[2:]
    errs["gae.adv"] = _err(batch.adv, a1, scale(a1, r1))
    errs["gae.ret"] = _err(batch.ret, r1, scale(a1, r1))
    moved = float((a1 - a0).abs().max()) / scale(a1, r1)
    print(f"\nrecompute: advantages moved by {moved:.2e} of their scale over the first repeat; "
          + " ".join(f"{k}={v:.2e}/{GAE_TOL:.0e}" for k, v in errs.items()), end="")
    assert moved > 100 * GAE_TOL, moved
    assert all(v <= GAE_TOL for v in errs.values()), errs


# ---- 5. the widest input -----------------------------------------------------------------------------------------
def test_observation_wider_than_the_engine_is_refused():
    from fsrl_b200 import _lib
    D = int(_lib.lib.fsrl_engine_dx_ld()) + 1
    with pytest.raises(ValueError, match="observation width %d" % D):
        p = _policy(D, 2, 64)
        _learn(p, _batch(p, 64, 1), 64, 1)
