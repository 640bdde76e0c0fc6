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

Long launches (thousands of steps, on both paths) run at lr = 0, which keeps theta fixed, so that every step is the
float64 update of its own minibatch at theta0 (section 6).

Every bound is a tolerance times a measured scale: the same expression evaluated on the magnitudes of its terms.
The synthetic batches put the ratio exp(logp - logp_old) on both sides of the clip range and of the dual clip, and the
stored values on both sides of the value clip, each a clear margin away from the kink; the head stage asserts that
margin before it compares.  The last row of every minibatch carries a large advantage, so that a dropped, doubled or
misplaced row moves the weight gradient far past its bound."""
import copy
import ctypes
import math
import time

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
NORM_TOL = 6e-6      # loss/grad_norm, relative to the norm of |X|^T |G| (chain) or to itself (persistent): 6.2e-7,
                     # 1.3e-6 over the 16384 steps of the long launch at D = 40
STAT_TOL = 8e-6      # statistics, relative to the sum of the magnitudes of their terms: 7.8e-7
PGRAD_TOL = 3e-6     # persistent launch: max |g - g64| / max |X|^T |G| per parameter group, natural masks: 2.2e-7
ULP_TOL = 32.0       # Adam's theta and v in fp32 ulps of their scale: 3.2
GAE_TOL = 5e-7       # recomputed advantages / returns, relative to the largest value, return and reward: 4.5e-8
KINK = 1e-3          # the float64 ratio / value offset is at least this far from every kink it can meet
M_TOL = 6e-7         # long launches: Adam's m, relative to the recurrence run on the per-group gradient scales: 6.3e-8
V_TOL = 9e-7         # long launches: Adam's v, likewise on the squared scales: 9.4e-8


class _BoxEnv:
    """The two spaces an agent reads: a user env with Box(-high, high) actions."""

    def __init__(self, D, A, high):
        from fsrl_b200.spaces import Box
        self.observation_space = Box(-np.inf, np.inf, (D,), np.float32)
        self.action_space = Box(-high, high, (A,), np.float32)


def _policy(D, A, H, C=2, high=1.0, bounded=True, lag=0.7, betas=None, lr=LR, persist=False, seed=3, **kw):
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
    if betas is not None or lr != LR:
        from fsrl_b200.optim import FusedAdam
        p.optim = FusedAdam(lr=lr, betas=betas or p.optim.param_groups[0]["betas"])
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


ROW_CHUNK = 1 << 17     # rows per float64 pass over a whole batch


def _relu_clearance(nets, x):
    """per row, the least |z| / (its magnitude chain) over the layer-1 and layer-2 pre-activations of every net"""
    out = []
    for xc in x.split(ROW_CHUNK):
        c = torch.full(xc.shape[:1], math.inf, dtype=torch.float64, device="cuda")
        for P in nets:
            z1, z2, _, _, _ = ppo64.forward(P, xc)
            one = torch.ones_like(z1)
            m1 = ppo64.forward_mag(P, xc, (one, one))[0]
            m2 = ppo64.forward_mag(P, xc, ((z1 > 0).double(), one))[1]
            c = torch.minimum(c, torch.minimum((z1.abs() / m1).amin(1), (z2.abs() / m2).amin(1)))
        out.append(c)
    return torch.cat(out)


def _batch(p, n, seed, trap_rows=(), relu_margin=0.0):
    """A DeviceBatch of n synthetic rows at the policy's current parameters: actions drawn from the policy, logp_old
    set so that the ratios fall in RATIO_BANDS, stored values VOFF_BANDS away from the critics, and advantages of
    40 / -30 on the batch rows trap_rows.  With relu_margin, the observations of every row with a hidden
    pre-activation closer to zero than relu_margin (_relu_clearance) are redrawn until none is; b.redrawn counts
    those rows and b.clearance is the least clearance left."""
    from fsrl_b200.policy.base_policy import DeviceBatch
    s0 = p.arena.slots[0]
    D, A, C = s0.D, s0.out, p.critics_num
    o = _opts(p)
    g = torch.Generator(device="cuda").manual_seed(seed)
    obs = torch.randn(n, D, generator=g, device="cuda")
    nets = _split(p, _d(p.arena.theta))
    redrawn = torch.zeros(n, dtype=torch.bool, device="cuda")
    while relu_margin:
        clearance = _relu_clearance(nets, _d(obs))
        bad = clearance < relu_margin
        if not bad.any():
            break
        redrawn |= bad
        obs[bad] = torch.randn(int(bad.sum()), D, generator=g, device="cuda")
    outs = [torch.cat([ppo64.forward(P, xc)[4] for xc in _d(obs).split(ROW_CHUNK)]) for P in nets]
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
    b.redrawn = int(redrawn.sum())
    if relu_margin:
        b.clearance = float(clearance.min())
    return b


def _learn(p, batch, bs, seed, repeat=1):
    np.random.seed(seed)
    p.learn(batch, batch_size=bs, repeat=repeat)
    return {k: np.asarray(v, dtype=np.float64) for k, v in p.last_stats.items()}


def _perms(seed, n, repeat):
    """the minibatch permutations of the first `repeat` repeats of a learn after np.random.seed(seed)"""
    rs = np.random.RandomState(seed)
    return [torch.from_numpy(rs.permutation(n)).cuda() for _ in range(repeat)]


def _perm(seed, n):
    return _perms(seed, n, 1)[0]


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
    """the batch rows idx [B], or M minibatches of them [M][B], in the layout of ppo64.Rows"""
    cols = lambda t: _d(t[:, idx]).movedim(0, -2)
    return ppo64.Rows(act=_d(batch.act[idx]), lpo=_d(batch.logp_old[idx]), adv=cols(batch.adv), ret=cols(batch.ret),
                      values=cols(batch.v))


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
            off = v - R.values[..., i, :]
            out = min(out, float(torch.minimum((off - o.eps_clip).abs(), (off + o.eps_clip).abs()).min()))
    return out


def _stat_errs(o, stats, st, row, errs):
    """the logged statistics of step row (or of the steps row of [M] minibatch statistics); keeps the worst"""
    keys = ["actor_rew", "kl", "entropy", "total"] + ["vf%d" % i for i in range(o.C)] + \
        (["actor_safety"] if o.use_saf else [])
    f64 = lambda v: torch.as_tensor(v, dtype=torch.float64, device="cuda")
    for k in keys:
        e = float(((f64(st["loss/" + k][row]) - f64(stats[k])).abs() / f64(stats["s_" + k]).clamp(min=FLT_MIN)).max())
        errs["stat." + k] = max(errs.get("stat." + k, 0.0), e)


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
        "stat": STAT_TOL, "pgrad": PGRAD_TOL, "adam": ULP_TOL, "adam_m": M_TOL, "adam_v": V_TOL}


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


def _persistent(p, batch, n, bs):
    """whether a learn of n rows in minibatches of bs takes the persistent launch"""
    from fsrl_b200 import _lib
    p._ensure_update_state(bs, n, 1)
    u = p._descriptor(batch, torch.zeros(batch.n, dtype=torch.int32, device="cuda"))
    return _lib.lib.fsrl_ppo_persist_active(ctypes.byref(u), n, bs) == 1


@pytest.mark.parametrize("name", list(PERSIST))
def test_persistent_launch(name):
    """One 256-row step, then a 4-step launch whose last step is checked at the recovered parameters."""
    A, D, kw = PERSIST[name]
    H, bs = 256, 256
    p = _policy(D, A, H, betas=(0.0, 0.0), persist=True, **kw)
    for n in (256, 1024):
        seed = 31 + n + A + D
        perm = _perm(seed, n)
        batch = _batch(p, n, seed, trap_rows=[int(perm[n - 1])])
        assert _persistent(p, batch, n, bs)
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


# ---- 6. long launches ------------------------------------------------------------------------------------------
# At lr = 0 theta stays theta0 bit for bit while every step still runs its whole Adam path (the step is -(0 / bc1)
# times the moment ratio), so step k of repeat r is the float64 update of the rows perm_r[256 k : 256 (k + 1)] at
# theta0.  Each step's statistics are checked against their own float64 values, and Adam's m and v after the learn
# against the float64 recurrence over every step's clipped gradient (v remembers about the last 1000 steps): every
# gradient element of every step, every minibatch index, statistics slot and operand image of the launch is tied to a
# check.  The rows keep every hidden pre-activation of every net RELU_MARGIN clear of zero at theta0, so the float64
# ReLU masks are the device's at every step; the ratios and value offsets stay KINK clear of the loss's kinks.
MAX_MB = 16384       # minibatches of one persistent launch (pp::MAX_MB in csrc/ppo_persist.cu)
RELU_MARGIN = 1e-5   # least |z| / magnitude chain of a hidden pre-activation: over 10x the forward error (6.5e-7)
# name: (D, A, H, n, repeat, persistent, policy options); batch_size 256, max_grad_norm 0.5
LONG = {
    "c2": (8, 2, 256, 2048 * 300, 4, True, {}),
    "c2-chain": (8, 2, 256, 2048 * 300, 4, False, {}),
    "c5-chain": (34, 8, 512, 1024 * 500, 1, False, {}),
    "gate-top": (40, 8, 256, MAX_MB * 256, 1, True, {}),
    "one-critic": (8, 3, 256, 64 * 256, 2, True, dict(C=1, bounded=False, value_clip=True, dual_clip=1.5,
                                                     reward_normalization=True)),
}


def _check_long(p, batch, theta0, perms, st):
    """every step of a learn at lr = 0 that started from zero Adam moments, against float64: each step's statistics
    and gradient norm, and m, v after the last step against the recurrence over every step's clipped gradient.
    A group's m (v) is measured against the same recurrence run on the group's gradient scale (squared)."""
    o = _opts(p)
    nets = _split(p, theta0)
    b1, b2 = p.optim.param_groups[0]["betas"]
    bs, H = 256, p.arena.slots[0].H
    n_mb = batch.n // bs
    T = len(perms) * n_mb
    assert len(st["loss/kl"]) == T
    f64 = lambda v: torch.as_tensor(v, dtype=torch.float64, device="cuda")
    m64 = [{k: torch.zeros_like(v) for k, v in P.items()} for P in nets]
    v64 = [{k: torch.zeros_like(v) for k, v in P.items()} for P in nets]
    mmag = [dict.fromkeys(P, 0.0) for P in nets]
    vmag = [dict.fromkeys(P, 0.0) for P in nets]
    errs, margin, clip = {"norm": 0.0}, math.inf, p._grad_norm
    chunk = 65536 // H                                 # minibatches per float64 evaluation
    for r, perm in enumerate(perms):
        for k0 in range(0, n_mb, chunk):
            M = min(chunk, n_mb - k0)
            idx = perm[k0 * bs:(k0 + M) * bs].view(M, bs)
            steps = r * n_mb + k0 + np.arange(M)
            R = _rows(batch, idx)
            stats, gref, gmag = ppo64.gradients(o, nets, _d(batch.obs[idx]), R)
            margin = min(margin, _kinks(o, stats, R, stats["v"]))
            gn = sum((g ** 2).flatten(1).sum(1) for G in gref for g in G.values()).sqrt()
            scale = (clip / (gn + 1e-6)).clamp(max=1.0) if clip else torch.ones_like(gn)
            errs["norm"] = max(errs["norm"], float(((f64(st["loss/grad_norm"][steps]) - gn).abs() / gn).max()))
            _stat_errs(o, stats, st, steps, errs)
            j = f64(steps)
            w1, w2 = (1 - b1) * b1 ** (T - 1 - j), (1 - b2) * b2 ** (T - 1 - j)
            for i, G in enumerate(gref):
                for key, g in G.items():
                    sg = scale.view(-1, *[1] * (g.dim() - 1)) * g
                    smax = scale * gmag[i][key].flatten(1).amax(1)
                    m64[i][key] += torch.tensordot(w1, sg, dims=1)
                    v64[i][key] += torch.tensordot(w2, sg * sg, dims=1)
                    mmag[i][key] += float((w1 * smax).sum())
                    vmag[i][key] += float((w2 * smax ** 2).sum())
    md, vd = _split(p, _d(p.optim.m)), _split(p, _d(p.optim.v))
    for i in range(len(nets)):
        for key in nets[i]:
            errs["adam_m.%d.%s" % (i, key)] = float((md[i][key] - m64[i][key]).abs().max()) / mmag[i][key]
            errs["adam_v.%d.%s" % (i, key)] = float((vd[i][key] - v64[i][key]).abs().max()) / vmag[i][key]
    return errs, margin


@pytest.mark.parametrize("name", list(LONG))
def test_long_launch_every_step(name):
    """Every step of a long learn at lr = 0 against float64; on the c2 shape, Adam's step at t = 4 x 2400 + 1."""
    D, A, H, n, repeat, persist, kw = LONG[name]
    bs, seed = 256, 41
    t_start = time.perf_counter()
    p = _policy(D, A, H, lr=0.0, betas=(0.9, 0.999), persist=persist, max_grad_norm=0.5, **kw)
    batch = _batch(p, n, seed, relu_margin=RELU_MARGIN)
    assert batch.clearance >= RELU_MARGIN
    theta0 = p.arena.theta.detach().clone()
    assert _persistent(p, batch, n, bs) == persist
    st = _learn(p, batch, bs, seed, repeat)
    assert torch.equal(p.arena.theta, theta0)               # lr = 0: the parameters never move
    assert p.optim.step_count == repeat * (n // bs)
    errs, margin = _check_long(p, batch, _d(theta0), _perms(seed, n, repeat), st)
    assert margin > KINK, margin
    if name.startswith("c2"):
        # one more 256-row learn at lr 5e-4: Adam at a large t, from the device's own m and v
        p.optim.param_groups[0]["lr"] = LR
        one = _batch(p, bs, seed + 1)
        assert _persistent(p, one, bs, bs) == persist
        t = p.optim.step_count + 1
        _learn(p, one, bs, seed)
        assert p.optim.step_count == t
        b1, b2 = p.optim.param_groups[0]["betas"]
        m, v = _d(p.optim.m), _d(p.optim.v)
        pr = _d(theta0) - LR / (1 - b1 ** t) * m / (v.sqrt() / math.sqrt(1 - b2 ** t) + p.optim.param_groups[0]["eps"])
        errs["adam.theta"] = _ulps(_d(p.arena.theta), pr, pr.abs() + LR)
    T = repeat * (n // bs)
    _report(f"long {name} {'persistent' if persist else 'chain'} D={D} A={A} H={H} n={n} repeat={repeat}: {T} steps, "
            f"{batch.redrawn} rows redrawn for the ReLU margin (clearance {batch.clearance:.1e}), kink margin "
            f"{margin:.2e}, {time.perf_counter() - t_start:.1f} s", errs)


def test_persistent_launch_is_deterministic():
    """A c2-shaped learn (4 repeats of 2400 steps, lr 5e-4, betas (0.9, 0.999)) twice from the same state: theta, m
    and v bit for bit, so that every step read the parameters the step before it published; the statistics, summed
    with atomics, to a relative 1e-6 of each statistic's largest value."""
    n, bs, seed = 2048 * 300, 256, 43
    p = _policy(8, 2, 256, betas=(0.9, 0.999), persist=True, max_grad_norm=0.5)
    batch = _batch(p, n, seed)
    assert _persistent(p, batch, n, bs)
    start = [t.detach().clone() for t in (p.arena.theta, p.optim.m, p.optim.v)]
    runs = []
    for _ in range(2):
        for t, s in zip((p.arena.theta, p.optim.m, p.optim.v), start):
            t.data.copy_(s)
        p.optim.step_count = 0
        p._mirror_dirty = True
        st = _learn(p, batch, bs, seed, repeat=4)
        runs.append(([t.detach().clone() for t in (p.arena.theta, p.optim.m, p.optim.v)], st))
    (s0, st0), (s1, st1) = runs
    assert len(st0["loss/kl"]) == 4 * n // bs
    assert float((s0[0] - start[0]).abs().max()) > 100 * LR        # the parameters moved
    for name, a, b in zip(("theta", "m", "v"), s0, s1):
        assert torch.equal(a, b), (name, float((a - b).abs().max()))
    worst = max(float(np.abs(st0[k] - st1[k]).max() / max(np.abs(st0[k]).max(), FLT_MIN)) for k in st0)
    print(f"\ndeterminism: theta, m, v bit-identical; statistics {worst:.1e}/1e-06", end="")
    assert worst <= 1e-6


# (D, A, H, C, n, batch_size, persistent)
GATE = {
    "c2": (8, 2, 256, 2, 2048 * 300, 256, True),
    "top": (40, 8, 256, 2, MAX_MB * 256, 256, True),
    "one-critic": (8, 3, 256, 1, 64 * 256, 256, True),
    "max-mb+1": (40, 8, 256, 2, (MAX_MB + 1) * 256, 256, False),
    "merged-tail": (8, 2, 256, 2, 2048 * 300 + 128, 256, False),
    "bs128": (8, 2, 256, 2, 2048 * 300, 128, False),
    "bs512": (8, 2, 256, 2, 2048 * 300, 512, False),
    "h128": (8, 2, 128, 2, 2048 * 300, 256, False),
    "h512": (8, 2, 512, 2, 2048 * 300, 256, False),
    "D41": (41, 2, 256, 2, 2048 * 300, 256, False),
}


@pytest.mark.parametrize("name", list(GATE))
def test_persistent_gate(name):
    """which learns the persistent launch takes, the rest going to the chain"""
    D, A, H, C, n, bs, want = GATE[name]
    p = _policy(D, A, H, C=C, persist=True)
    assert _persistent(p, _batch(p, 256, 1), n, bs) == want
