"""CPO, TRPO-Lagrangian and FOCOPS on the device, stage by stage, against float64.

Each stage is fed what the device left from the stage before it, so that an error points at one kernel:

  process_fn  fsrl_standardize, and mean_old / std_old against a float64 actor with the device's parameters
  forward     h1, h2 and the head output z of the engine's saved forward pass
  heads       fsrl_cpo_head modes 0-3 and fsrl_focops_head evaluated at the device's fp32 z: the batch sums and
              every row's 2A dout columns
  wgrad       fsrl_engine_wgrad_to of the objective, the -cost surrogate and the KL, backpropagated in float64
              from the device's dout
  HVP         fsrl_cpo_hvp against float64 double backward of the mean KL, plus u.Hv = v.Hu and, at
              theta = theta_old, v.Hv >= damping |v|^2
  CG          fsrl_cg_solve against float64 CG driven by the float64 Hessian-vector product
  CPO         the dual case analysis and the line search, fed the device's g, b, H^-1 g, H^-1 b and step
  TRPO        flat gradient, step size, line search and its exhaustion path
  FOCOPS      per-minibatch advantages, the masked head, the clipped gradient and the Adam step
  critic      fsrl_mse_head + wgrad + Adam with the L2 term

The float64 networks take their ReLU masks from the device's saved h1 / h2: a unit whose pre-activation is within
fp32 rounding of zero may switch on one side only (see tests/test_offpolicy_f64_gpu.py).  Every bound is a
tolerance tau times a measured scale, the sum of the magnitudes of the terms that make up the value (for a weight
gradient |X|^T |G| with G propagated in magnitudes), so it holds unchanged from 2 rows to c3's 148 019-row chunk,
where wgrad adds 4096-row fp32 partials with atomics.  A discrete decision (optim_case, a line-search step, the
FOCOPS indicator, the CG exit) is compared only after asserting that its float64 value is clearly away from the
threshold.  Above 4096 rows the atomics' order varies, so nothing here asserts bit-equal reruns."""
import ctypes
import math

import numpy as np
import pytest
import torch

from helpers import adam64, cg64, cg_stop_tol, synthetic_ring

pytestmark = pytest.mark.gpu

F32_EPS = float(np.finfo(np.float32).eps)
LOG_SQRT_2PI = 0.5 * math.log(2.0 * math.pi)
DAMP = 0.1
SPLIT = 4096                 # rows per wgrad CTA at most (csrc/engine.cu eng_wgrad_roles)
C3_D = 60                    # SafetyPointGoal1Gymnasium-v0: D = 60, A = 2

# Bounds: about 10x the worst value observed over all cases on an H100 80GB HBM3 (700 W power limit), given in
# each comment; every case prints its errors.
STD_TOL = 6e-7       # fsrl_standardize, |got - ref| / (1 + max|x| / std): 5.7e-8 (n = 2 048 000)
OLD_TOL = 5e-7       # mean_old / std_old against the float64 actor, relative to the magnitude chain: 4.3e-8
FWD_TOL = 8e-6       # h1, h2, z against float64 with device masks, relative to the magnitude chain: 7.7e-7
SUM_TOL = 3e-7       # head sums, relative to sum |terms|: 2.4e-8
DOUT_TOL = 2e-6      # head dout, relative to the element's magnitude: 3.4e-7
GRAD_TOL = 1e-5      # wgrad, relative to |X|^T |G|: 3.8e-6 on a moved A = 6 batch whose saturated rows
                     # carry fp32-denormal ratios, <= 1.1e-6 on every other case
HVP_TOL = 3e-6       # Hessian-vector product, relative to the magnitude R-op: 2.3e-7
SYM_TOL = 4e-7       # |u.Hv - v.Hu| / (|u||Hv| + |v||Hu|): 3.3e-8
CG_TOL = 1e-4        # |x - x64| / |x64|: 7.2e-6 at A = 8 (10 iterations and the early exit)
CG10_C3_TOL = 0.25   # ... after 10 iterations on c3's 148 019 rows, where fp32 CG loses conjugacy: 2.5e-2
ULP_TOL = 32.0       # Adam / axpy results in fp32 ulps of their operands' scale: 5.4 (critic Adam)
DUAL_TOL = 1e-4      # lambda, nu, q, r, s, shs, the step direction and the TRPO step size, relative: 1.6e-6 (s)
MARGIN = 100.0       # a decision's float64 value is at least MARGIN x its error bound away from the threshold
FLT_MIN = float(np.finfo(np.float32).tiny)   # below it fp32 keeps denormal ulps only: a floor on every bound


class _BoxEnv:
    """The two spaces an agent reads: a user env with Box(-high, high) actions."""

    def __init__(self, D, A, high):
        from fsrl_b200.spaces import Box
        self.observation_space = Box(-np.inf, np.inf, (D,), np.float32)
        self.action_space = Box(-high, high, (A,), np.float32)


def _policy(algo, D, A, high=1.0, H=64, bounded=True, seed=3, **kw):
    from fsrl_b200.agent import CPOAgent, FOCOPSAgent, TRPOLagAgent
    cls = {"cpo": CPOAgent, "trpo": TRPOLagAgent, "focops": FOCOPSAgent}[algo]
    p = cls(_BoxEnv(D, A, high), seed=seed, hidden_sizes=(H, H), unbounded=not bounded, **kw).policy
    assert p.actor._max == high and p.actor._unbounded == (not bounded)
    return p


def _d(t):
    return t.detach().double()


def _batch(p, n_all, seed, saturate=False, adv_c_zero=False):
    """A processed batch from the policy's own process_fn over a synthetic ring of n_all rows; then a sampled
    action act = mean_old + std_old * eps with its logp_old, and standard-normal advantages.  saturate scales every
    7th observation by 40, so that the bounded mean's tanh saturates there."""
    D, A = p.arena.slots[0].D, p.arena.slots[0].out
    n_env = 8
    buf = synthetic_ring(D, A, n_env, -(-n_all // n_env), "wrapped", seed=seed, max_action=p.actor._max)
    if saturate:
        buf.obs[::7] *= 40.0
    batch = p.process_fn(None, buf, buf.sample_indices(0))
    if hasattr(p, "_refresh_old_dist"):
        p._refresh_old_dist(batch)
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = batch.n
    mo, so = _d(batch.mean_old), _d(batch.std_old)
    eps = torch.randn(n, A, generator=g, device="cuda", dtype=torch.float64)
    act = mo + so * eps
    batch.act = act.float().contiguous()
    lp = (-0.5 * ((_d(batch.act) - mo) / so) ** 2 - so.log() - LOG_SQRT_2PI).sum(1)
    batch.logp_old = lp.float().contiguous()
    adv = torch.randn(2, n, generator=g, device="cuda")
    if adv_c_zero:
        adv[1] = 0.0
    batch.adv = adv.contiguous()
    batch.advs = batch.adv.t()
    batch.eps = eps
    return batch, buf


def _perm(n_all, n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randperm(n_all, generator=g)[:n].to(torch.int32).cuda()


def _split_rows(n):
    """(first, last) minibatch row of the second wgrad split, or None below the split"""
    nsplit = -(-n // SPLIT)
    if nsplit < 2:
        return None
    per = -(-(-(-n // nsplit)) // 32) * 32
    return per, min(2 * per, n) - 1


def _traps(batch, perm, n):
    """advantages ~1000x the typical size on the minibatch's last row and on the first and last row of one wgrad
    split: a dropped, doubled or misplaced row then moves the gradient far past its bound"""
    rows = [n - 1]
    sp = _split_rows(n)
    if sp is not None:
        rows += list(sp)
    r = perm[torch.tensor(rows, device="cuda")].long()
    sign = torch.tensor([1.0, -1.0, 1.0][:len(rows)], device="cuda")
    batch.adv[0, r] = 1e3 * sign
    batch.adv[1, r] = -7e2 * sign
    return rows


def _move(p, seed, size=0.05):
    """theta away from theta_old: the same relative move at every width; log sigma moves too"""
    a = p.arena.slots[0]
    g = torch.Generator().manual_seed(seed)
    delta = size * (64 / a.H) ** 0.5 * torch.randn(a.size, generator=g)
    p.arena.theta[a.offset:a.offset + a.size] += delta.cuda()


# ---- float64 networks and heads -------------------------------------------------------------------------------
def _parts(s, th):
    w1, b1, w2, b2, w3, b3, ex = (o - s.offset for o in s.offsets())
    return dict(w1=th[w1:b1].view(s.D, s.H), b1=th[b1:w2], w2=th[w2:b2].view(s.H, s.H), b2=th[b2:w3],
                w3=th[w3:b3].view(s.H, s.out), b3=th[b3:ex], ls=th[ex:ex + s.n_extra])


def _mlp64(s, th, x, masks=None):
    t = _parts(s, th)
    act = (lambda z, k: z * masks[k]) if masks is not None else (lambda z, k: torch.relu(z))
    h1 = act(x @ t["w1"] + t["b1"], 0)
    h2 = act(h1 @ t["w2"] + t["b2"], 1)
    return h1, h2, h2 @ t["w3"] + t["b3"]


def _mag_chain(s, th, x, masks):
    t = {k: v.abs() for k, v in _parts(s, th).items()}
    h1 = (x.abs() @ t["w1"] + t["b1"]) * masks[0]
    h2 = (h1 @ t["w2"] + t["b2"]) * masks[1]
    return h1, h2, h2 @ t["w3"] + t["b3"]


class _Sq:
    """the squash mu(z) of the policy and the magnitudes of its rounding: 1 - t^2 is two terms of size ~1"""

    def __init__(self, p):
        self.bounded, self.m = not p.actor._unbounded, float(p.actor._max)

    def mu(self, z):
        return self.m * torch.tanh(z) if self.bounded else z

    def mup_mag(self, z):
        return self.m * (1 + torch.tanh(z) ** 2) if self.bounded else torch.ones_like(z)

    def mupp_mag(self, z):
        t = torch.tanh(z).abs()
        return 2 * self.m * t * (1 + t * t) if self.bounded else torch.zeros_like(z)


class _Rows:
    """the minibatch's rows of a batch in float64"""

    def __init__(self, batch, perm, n):
        idx = perm.long() if perm is not None else torch.arange(n, device="cuda")
        self.idx = idx
        self.x = _d(batch.obs[idx])
        self.act = _d(batch.act[idx])
        self.mo, self.so = _d(batch.mean_old[idx]), _d(batch.std_old[idx])
        self.lpo = _d(batch.logp_old[idx])
        self.ar, self.ac = _d(batch.adv[0][idx]), _d(batch.adv[1][idx])


def _cpo_head64(sq, z, ls, R, mode):
    """float64 head at z [n, A]: (sum objective, sum cost ratio, sum kl), their sum-|terms| scales, and for mode 1-3
    the d/dz, d/dlog-sigma columns of the mean by autograd with the magnitude of every element"""
    n = z.shape[0]
    z = z.clone().requires_grad_(True)
    lsr = ls.view(1, -1).expand_as(z).clone().requires_grad_(True)
    mu, sg = sq.mu(z), lsr.exp()
    zz = (R.act - mu) / sg
    lp_terms = -0.5 * zz ** 2 - lsr - LOG_SQRT_2PI
    ratio = torch.exp(lp_terms.sum(1) - R.lpo)
    s_lp = (0.5 * zz ** 2 + lsr.abs() + LOG_SQRT_2PI).sum(1) + R.lpo.abs()       # condition of exp(logp - logp_old)
    vr, t1 = (R.so / sg) ** 2, ((R.mo - mu) / sg) ** 2
    kl = 0.5 * (vr + t1 - 1 - vr.log())
    sums = [(ratio * R.ar).sum(), (ratio * R.ac).sum(), kl.sum()]
    scl = [((ratio * R.ar).abs() * (1 + s_lp)).sum(), ((ratio * R.ac).abs() * (1 + s_lp)).sum(),
           (0.5 * (vr + t1 + 1 + vr.log().abs())).sum()]
    out = [float(v) for v in sums], [float(v) for v in scl]
    if mode == 0:
        return out + (None, None)
    f = {1: (ratio * R.ar).mean(), 2: -(ratio * R.ac).mean(), 3: kl.sum(1).mean()}[mode]
    gz, gl = torch.autograd.grad(f, (z, lsr))
    with torch.no_grad():
        mup, sgd = sq.mup_mag(z), sg.detach()
        if mode in (1, 2):
            a = R.ar if mode == 1 else R.ac
            glm = ((ratio * a).abs() * (1 + s_lp) / n).view(-1, 1)
            mz = glm * (R.act.abs() + mu.abs()) / sgd ** 2 * mup
            ml = glm * (zz ** 2 + 1)
        else:
            dm = mu.abs() + R.mo.abs()
            mz = dm / sgd ** 2 / n * mup
            ml = (1 + (R.so ** 2 + dm ** 2) / sgd ** 2) / n
    return out + (torch.cat([gz, gl], 1), torch.cat([mz, ml], 1))


def _grad_scale(s, th, x, masks, dout_mag):
    """|X|^T |G| of every block of wgrad, G propagated back from |dout| through |W| with the device masks"""
    t = {k: v.abs() for k, v in _parts(s, th).items()}
    A = s.out
    h1m, h2m, _ = _mag_chain(s, th, x, masks)
    g3 = dout_mag[:, :A]
    dz2 = (g3 @ t["w3"].t()) * masks[1]
    dz1 = (dz2 @ t["w2"].t()) * masks[0]
    parts = [x.abs().t() @ dz1, dz1.sum(0), h1m.t() @ dz2, dz2.sum(0), h2m.t() @ g3, g3.sum(0)]
    if s.n_extra:
        parts.append(dout_mag[:, A:A + s.n_extra].sum(0))
    return torch.cat([q.reshape(-1) for q in parts])


def _wgrad_ref(s, th, x, masks, dout):
    """float64 autograd of the weight gradient, backpropagated from the device's dout"""
    A = s.out
    thg = th.clone().requires_grad_(True)
    _, _, z = _mlp64(s, thg, x, masks)
    (gth,) = torch.autograd.grad(z, thg, grad_outputs=dout[:, :A])
    if s.n_extra:
        gth = gth.clone()
        gth[-s.n_extra:] = dout[:, A:A + s.n_extra].sum(0)
    return gth


def _err(got, ref, scale, floor=0.0):
    """max |got - ref| / scale, after forgiving `floor`: a ratio exp(logp - logp_old) that underflows into fp32's
    denormals (a saturated row after the move) keeps only absolute precision, so the product terms it enters may
    each be off by FLT_MIN"""
    got, ref, scale = (torch.as_tensor(v, dtype=torch.float64, device="cuda") for v in (got, ref, scale))
    tiny = torch.finfo(torch.float64).tiny
    return float((torch.clamp((got - ref).abs() - floor, min=0.0) / torch.clamp(scale, min=tiny)).max())


def _kl_mean64(s, sq, R, masks):
    def f(th):
        _, _, z = _mlp64(s, th, R.x, masks)
        mu, sg = sq.mu(z[:, :s.out]), _parts(s, th)["ls"].exp()
        vr, t1 = (R.so / sg) ** 2, ((R.mo - mu) / sg) ** 2
        return (0.5 * (vr + t1 - 1 - vr.log())).sum(1).mean()
    return f


def _hvp64(f, th):
    """v -> H v + damping v, float64 double backward of f at th"""
    thg = th.clone().requires_grad_(True)
    (gk,) = torch.autograd.grad(f(thg), thg, create_graph=True)
    return lambda v: torch.autograd.grad(gk @ v, thg, retain_graph=True)[0] + DAMP * v


def _hvp_scale(s, sq, th, v, R, masks, z):
    """the R-op of csrc/cpo.cu with every product taken in magnitudes: the sum of |terms| of each element of Hv"""
    n, A = R.x.shape[0], s.out
    T = {k: q.abs() for k, q in _parts(s, th).items()}
    V = {k: q.abs() for k, q in _parts(s, v).items()}
    x = R.x.abs()
    h1, h2, _ = _mag_chain(s, th, R.x, masks)
    Rh1 = (x @ V["w1"] + V["b1"]) * masks[0]
    Rh2 = (Rh1 @ T["w2"] + h1 @ V["w2"] + V["b2"]) * masks[1]
    Rz = Rh2 @ T["w3"] + h2 @ V["w3"] + V["b3"]
    mu, mup, mupp = sq.mu(z).abs(), sq.mup_mag(z), sq.mupp_mag(z)
    is2 = torch.exp(-2 * _parts(s, th)["ls"])
    vs = V["ls"]
    dm = mu + R.mo.abs()
    kmu = dm * is2 / n
    e = kmu * mup
    Re = (mup * Rz * is2 / n + 2 * kmu * vs) * mup + kmu * mupp * Rz
    Res = (2 * dm * mup * Rz * is2 + 2 * (R.so ** 2 + dm ** 2) * is2 * vs) / n
    da2 = (e @ T["w3"].t()) * masks[1]
    Rda2 = (Re @ T["w3"].t() + e @ V["w3"].t()) * masks[1]
    Rda1 = (Rda2 @ T["w2"].t() + da2 @ V["w2"].t()) * masks[0]
    parts = [x.t() @ Rda1, Rda1.sum(0), Rh1.t() @ da2 + h1.t() @ Rda2, Rda2.sum(0), Rh2.t() @ e + h2.t() @ Re,
             Re.sum(0), Res.sum(0)]
    return torch.cat([q.reshape(-1) for q in parts]) + DAMP * v.abs()


# ---- the device side ------------------------------------------------------------------------------------------
class _Dev:
    """engine, descriptor and input of one minibatch of the policy's actor"""

    def __init__(self, p, batch, perm, n):
        from fsrl_b200 import _lib
        self.lib = _lib
        self.p, self.n = p, n
        self.a = p.arena.slots[0]
        self.eng = p._ensure_engine(n)
        self.eng.sync_mirror([self.a])
        self.d = p._descriptor(batch, perm, n)
        self.inp = self.eng.make_input(batch.obs, perm)
        self.s = torch.cuda.current_stream().cuda_stream

    def theta(self):
        a = self.a
        return self.p.arena.theta[a.offset:a.offset + a.size]

    def view(self, what, slot=None):
        return self.eng.slot_view(slot or self.a, what)[:self.n]

    def forward(self):
        self.eng.forward([self.a], self.inp, self.n, save=True)
        return (_d(self.view("h1")) > 0).double(), (_d(self.view("h2")) > 0).double()

    def head(self, mode):
        self.p._head(self.d, mode)
        return self.p._sums.cpu().numpy().copy()

    def wgrad_to(self, dst):
        e, nl = self.eng.engine(), self.eng.netlist([self.a])
        self.eng.backward([self.a], self.n)
        self.lib.check(self.lib.lib.fsrl_engine_wgrad_to(ctypes.byref(e), ctypes.byref(nl), ctypes.byref(self.inp),
                                                         self.n, dst.data_ptr(), self.s))


def _report(label, errs, bounds):
    print(f"\n{label}: " + " ".join(f"{k}={v:.2e}/{bounds[k]:.0e}" for k, v in errs.items()))
    bad = {k: v for k, v in errs.items() if not v <= bounds[k]}
    assert not bad, bad


# ---- 1. process_fn ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [2, 1023, 1025, 2_048_000])
def test_standardize(n):
    from fsrl_b200 import _lib
    g = torch.Generator(device="cuda").manual_seed(n)
    x = 5.0 + 2.0 * torch.randn(n, generator=g, device="cuda")
    x64 = _d(x)
    ref = (x64 - x64.mean()) / x64.std()
    _lib.check(_lib.lib.fsrl_standardize(x.data_ptr(), n, torch.cuda.current_stream().cuda_stream))
    std = float(x64.std())
    err = float((_d(x) - ref).abs().max()) / (1 + float(x64.abs().max()) / std)
    _report(f"standardize n={n}", {"std": err}, {"std": STD_TOL})


@pytest.mark.parametrize("algo,high,bounded", [("cpo", 1.0, True), ("cpo", 2.0, True), ("cpo", 1.0, False),
                                               ("trpo", 2.0, True), ("focops", 2.0, False)])
def test_process_fn_old_distribution(algo, high, bounded):
    D, A = 11, 3
    p = _policy(algo, D, A, high, H=128, bounded=bounded)
    batch, _ = _batch(p, 3000, seed=2, saturate=bounded)
    s = p.arena.slots[0]
    th = _d(p.arena.theta[s.offset:s.offset + s.size])
    x = _d(batch.obs)
    h1, h2, z = _mlp64(s, th, x)
    masks = ((h1 > 0).double(), (h2 > 0).double())
    _, _, zm = _mag_chain(s, th, x, masks)
    sq = _Sq(p)
    mu = sq.mu(z)
    errs = {"mean_old": _err(batch.mean_old, mu, zm * sq.mup_mag(z)),
            "std_old": _err(batch.std_old, _parts(s, th)["ls"].exp().expand_as(mu), _parts(s, th)["ls"].exp())}
    _report(f"process_fn {algo} high={high} bounded={bounded}", errs, {"mean_old": OLD_TOL, "std_old": OLD_TOL})


# ---- 2-4. heads, flat gradients, Hessian-vector products: the case matrix ------------------------------------
SQUASH = {"b1": (1.0, True), "b2": (2.0, True), "unb": (1.0, False)}
NS = [2, 255, 257, 4096, 4097, 3 * 4096 + 1]


def _matrix():
    cases, k = [], 0
    for A in (2, 3, 4, 6, 8):
        for sq in ("b1", "b2", "unb"):
            for moved in (False, True):
                H, n = (64, 128, 256, 512)[k % 4], NS[k % 6]
                cases.append(pytest.param(A, sq, moved, H, n, 5 + 3 * A, id=f"A{A}-{sq}-{'moved' if moved else 'old'}-h{H}-n{n}"))
                k += 1
    cases.append(pytest.param(2, "b1", False, 128, 99_999, C3_D, id="c3-n99999-old"))
    cases.append(pytest.param(2, "b1", True, 128, 148_019, C3_D, id="c3-n148019-moved"))
    return cases


def _core(A, sq_name, moved, H, n, D, seed=1):
    high, bounded = SQUASH[sq_name]
    p = _policy("cpo", D, A, high, H=H, bounded=bounded, seed=seed)
    n_all = max(n + n // 8, 64)
    batch, _ = _batch(p, n_all, seed=seed + A, saturate=bounded)
    perm = _perm(batch.n, n, seed)
    rows = _traps(batch, perm, n)
    if moved:
        _move(p, seed + 7)
    dv = _Dev(p, batch, perm, n)
    s, sq, R = dv.a, _Sq(p), _Rows(batch, perm, n)
    th = _d(dv.theta())
    ls = _parts(s, th)["ls"]
    masks = dv.forward()
    errs = {}
    # forward
    h1, h2, z64 = _mlp64(s, th, R.x, masks)
    h1m, h2m, zm = _mag_chain(s, th, R.x, masks)
    errs["fwd.h1"] = _err(dv.view("h1"), h1, h1m)
    errs["fwd.h2"] = _err(dv.view("h2"), h2, h2m)
    errs["fwd.z"] = _err(dv.view("out")[:, :A], z64, zm)
    z = _d(dv.view("out")[:, :A])              # the heads are evaluated at the device's z
    sat = int((z.abs() > 9).sum()) if bounded else 0
    # heads and flat gradients
    sm = dv.head(0)
    ref, scl, _, _ = _cpo_head64(sq, z, ls, R, 0)
    for k in range(3):
        errs[f"sum0.{k}"] = abs(sm[k] - ref[k]) / scl[k]
    vec = p._vec["g"]
    for mode in (1, 2, 3):
        sm = dv.head(mode)
        ref, scl, dref, dmag = _cpo_head64(sq, z, ls, R, mode)
        for k in range(3):
            errs[f"sum{mode}.{k}"] = abs(sm[k] - ref[k]) / scl[k]
        dout = _d(dv.view("dout"))
        assert (dout[:, 2 * A:] == 0).all()
        errs[f"dout{mode}"] = _err(dout[:, :2 * A], dref, dmag, FLT_MIN)
        dv.wgrad_to(vec)
        gref = _wgrad_ref(s, th, R.x, masks, dout)
        errs[f"grad{mode}"] = _err(vec, gref, _grad_scale(s, th, R.x, masks, dout.abs()), n * FLT_MIN * (1 + float(R.x.abs().max())))
    # Hessian-vector products: the P-slot now holds the kl head's dout and backward, as learn() leaves it
    f = _kl_mean64(s, sq, R, masks)
    mvp = _hvp64(f, th)
    g = torch.Generator(device="cuda").manual_seed(seed + 11)
    vs, hvs = [], []
    for t in range(2):
        v = torch.randn(s.size, generator=g, device="cuda", dtype=torch.float64).float()
        hv = p._vec["hv"]
        p._hvp(dv.d, v, hv)
        v64, got = _d(v), _d(hv).clone()
        errs[f"hvp{t}"] = _err(got, mvp(v64), _hvp_scale(s, sq, th, v64, R, masks, z))
        vs.append(v64); hvs.append(got)
    nrm = torch.linalg.norm
    errs["sym"] = float((vs[0] @ hvs[1] - vs[1] @ hvs[0]).abs() / (nrm(vs[0]) * nrm(hvs[1]) + nrm(vs[1]) * nrm(hvs[0])))
    psd = min(float((v @ hv - DAMP * v @ v) / (nrm(v) * nrm(hv))) for v, hv in zip(vs, hvs))
    bounds = {k: {"fwd": FWD_TOL, "sum": SUM_TOL, "dou": DOUT_TOL, "gra": GRAD_TOL, "hvp": HVP_TOL,
                  "sym": SYM_TOL}[k[:3]] for k in errs}
    print(f"\n[min (vHv - damping |v|^2) / (|v||Hv|) = {psd:.2e}, saturated |z| > 9: {sat}, trap rows {rows}]", end="")
    _report(f"core A={A} {sq_name} moved={moved} H={H} n={n} D={D}", errs, bounds)
    if not moved:
        assert psd >= -HVP_TOL, psd


@pytest.mark.parametrize("A,sq,moved,H,n,D", _matrix())
def test_heads_gradients_hvp(A, sq, moved, H, n, D):
    _core(A, sq, moved, H, n, D)


# ---- 5. conjugate gradients ------------------------------------------------------------------------------------
@pytest.mark.parametrize("A,sq,H,n,D,early", [(8, "unb", 128, 5000, 21, False), (8, "unb", 128, 5000, 21, True),
                                              (2, "b1", 128, 148_019, C3_D, False)],
                         ids=["A8-unbounded-10", "A8-unbounded-early", "c3-n148019-10"])
def test_cg_solve(A, sq, H, n, D, early):
    high, bounded = SQUASH[sq]
    p = _policy("cpo", D, A, high, H=H, bounded=bounded)
    batch, _ = _batch(p, n + n // 8, seed=4)        # no 40x observations: they inflate the condition number of H
    perm = _perm(batch.n, n, 5)
    dv = _Dev(p, batch, perm, n)
    s, sq_, R = dv.a, _Sq(p), _Rows(batch, perm, n)
    masks = dv.forward()
    dv.head(1)
    gvec = p._vec["g"]
    dv.wgrad_to(gvec)
    dv.head(3)
    dv.eng.backward([s], n)
    th = _d(dv.theta())
    mvp = _hvp64(_kl_mean64(s, sq_, R, masks), th)
    rhs = _d(gvec)
    x_full, res = cg64(mvp, rhs, nsteps=10, tol=0.0)
    tol, x_ref, sep = 0.0, x_full, 0.0
    if early:
        k, tol = cg_stop_tol(res)
        assert min(res[:k]) / res[k] > 1.5, res
        x_ref, res_stop = cg64(mvp, rhs, nsteps=10, tol=tol)
        assert len(res_stop) == k + 1
        sep = float((x_ref - x_full).norm() / x_full.norm())
        assert sep > 20 * CG_TOL, sep
    out = p._vec["Hinv_g"]
    p._cg(dv.d, gvec, out, nsteps=10, residual_tol=tol)
    err = float((_d(out) - x_ref).norm() / x_ref.norm())
    print(f"\n[residuals {[f'{r:.2e}' for r in res]}, stopped vs 10 iterations {sep:.2e}]", end="")
    _report(f"cg A={A} {sq} n={n} early={early}", {"cg": err}, {"cg": CG10_C3_TOL if n > 100_000 else CG_TOL})
    assert float(p._cg_state[4].item()) == (1.0 if early else 0.0)


def _ulps(got, want, scale):
    sp = torch.from_numpy(np.spacing(scale.abs().float().cpu().numpy())).double().cuda()
    return float(((got - want).abs() / sp).max())


def _decide(conds):
    """one tried line-search step: conds = [(value, scale)], accepted when every value is positive.  The float64
    outcome must be clear: every value of an accepted step, and at least one of a rejected step, lies MARGIN x its
    error bound away from zero."""
    room = [abs(v) > MARGIN * SUM_TOL * sc for v, sc in conds]
    if all(v > 0 for v, _ in conds):
        assert all(room), conds
        return True
    assert any(v < 0 and r for (v, _), r in zip(conds, room)), conds
    return False


# ---- 6. CPO dual case analysis and line search -----------------------------------------------------------------
def _cpo_dual64(q, r, s, c, delta):
    """policy/cpo.py's case analysis restated in float64 (reference cpo.py:257-304); returns case, lam, nu and the
    margin of the lambda_a / lambda_b choice (None outside cases 1 and 2)"""
    EPS = 1e-8
    A_, B_ = q - r * r / s, 2 * delta - c * c / s
    case = 3 if (c < 0 and B_ < 0) else 2 if (c < 0 and B_ >= 0) else 1 if (c >= 0 and B_ >= 0) else 0
    margin = None
    if case in (3, 4):
        lam, nu = math.sqrt(q / (2 * delta)), 0.0
    elif case in (1, 2):
        LA, LB = [0, r / c], [r / c, np.inf]
        LA, LB = (LA, LB) if c < 0 else (LB, LA)
        proj = lambda x, L: max(L[0], min(L[1], x))
        lam_a, lam_b = proj(math.sqrt(A_ / B_), LA), proj(math.sqrt(q / (2 * delta)), LB)
        fa = -0.5 * (A_ / (lam_a + EPS) + B_ * lam_a) - r * c / (s + EPS)
        fb = -0.5 * (q / (lam_b + EPS) + 2 * delta * lam_b)
        lam = lam_a if fa >= fb else lam_b
        margin = abs(fa - fb) / (abs(fa) + abs(fb))
        nu = max(0.0, lam * c - r) / (s + EPS)
    else:
        lam, nu = 0.0, math.sqrt(2 * delta / (s + EPS))
    return case, lam, nu, margin, A_, B_


def _terms64(s, sq, th, R, ave_cost, mean_adv_c):
    """objective, cost surrogate and kl at th in float64 (plain ReLU), with the sum-|terms| scales of each"""
    _, _, z = _mlp64(s, th, R.x)
    ls = _parts(s, th)["ls"]
    (o, c, k), (so, sc, sk), _, _ = _cpo_head64(sq, z[:, :s.out], ls, R, 0)
    n = R.x.shape[0]
    return dict(obj=o / n, cost=ave_cost + c / n - mean_adv_c, kl=k / n, s_obj=so / n, s_cost=sc / n, s_kl=sk / n)


@pytest.mark.parametrize("case", [0, 1, 2, 3, 4])
def test_cpo_decision_and_line_search(case):
    A, D, n = 3, 13, 3000
    p = _policy("cpo", D, A, 2.0, H=64, bounded=True, target_kl=0.05)
    batch, _ = _batch(p, 3500, seed=6, saturate=True, adv_c_zero=(case == 4))
    p._ave_cost_return = 5.0
    perm = _perm(batch.n, n, 6)
    dv = _Dev(p, batch, perm, n)
    s, sq, R = dv.a, _Sq(p), _Rows(batch, perm, n)
    theta_start = dv.theta().clone()
    delta = p._delta
    # first pass: s and the cost surrogate, then theta back where it was
    p._cost_limit = 1e6
    st0 = p.policy_loss(batch, perm, n)
    dv.theta().copy_(theta_start)
    dv.eng.sync_mirror([s])
    S0, cs0 = st0["loss/optim_S"], st0["loss/cost_loss"]
    c_target = {2: -0.5, 1: 0.5, 3: -2.0, 0: 2.0, 4: -1.0}[case]
    c_target *= math.sqrt(2 * delta * S0) if case != 4 else 1.0
    p._cost_limit = cs0 - c_target
    masks = dv.forward()
    th0 = _d(dv.theta())
    st = p.policy_loss(batch, perm, n)
    v = {k: _d(t).clone() for k, t in p._vec.items()}
    theta1 = _d(dv.theta())
    assert torch.equal(v["theta0"], th0)
    mean_adv_c = float(R.ac.mean())
    t0 = _terms64(s, sq, th0, R, p._ave_cost_return, mean_adv_c)
    c64 = t0["cost"] - p._cost_limit
    errs = {"cost_loss": abs(st["loss/cost_loss"] - t0["cost"]) / (t0["s_cost"] + p._ave_cost_return + abs(mean_adv_c)),
            "rew_loss": abs(st["loss/rew_loss"] - t0["obj"]) / t0["s_obj"]}
    mvp = _hvp64(_kl_mean64(s, sq, R, masks), th0)
    hg = mvp(v["Hinv_g"])
    q64 = float(hg @ v["Hinv_g"])
    if case == 4:
        assert float(v["b"] @ v["b"]) == 0.0 and c64 < 0
        case64, lam64, nu64, lam_margin, A64, B64 = 4, math.sqrt(q64 / (2 * delta)), 0.0, None, 0.0, 0.0
    else:
        hb = mvp(v["Hinv_b"])
        r64, s64 = float(hg @ v["Hinv_b"]), float(hb @ v["Hinv_b"])
        errs["q"] = abs(st["loss/optim_Q"] - q64) / abs(q64)
        errs["r"] = abs(st["loss/optim_R"] - r64) / math.sqrt(abs(q64 * s64))
        errs["s"] = abs(st["loss/optim_S"] - s64) / abs(s64)
        case64, lam64, nu64, lam_margin, A64, B64 = _cpo_dual64(q64, r64, s64, c64, delta)
        # the decision's inputs are far from its thresholds: c at +-0.5 or +-2 sqrt(2 delta s), so |B| >= 1.5 delta
        assert abs(c64) >= 0.4 * math.sqrt(2 * delta * s64) and abs(B64) >= delta, (c64, B64)
        if lam_margin is not None:
            assert lam_margin > MARGIN * DUAL_TOL, lam_margin
    assert st["loss/optim_case"] == case64 == case, (st["loss/optim_case"], case64)
    errs["lam"] = abs(st["loss/optim_lam"] - lam64) / max(abs(lam64), 1e-30)
    if case in (1, 2):
        errs["nu"] = abs(st["loss/optim_nu"] - nu64) / ((abs(lam64 * c64) + abs(r64)) / s64)
    else:
        errs["nu"] = abs(st["loss/optim_nu"] - nu64) / max(abs(nu64), 1e-30) if nu64 else abs(st["loss/optim_nu"])
    # the normalised step from the device's H^-1 g, H^-1 b and the float64 lambda, nu
    EPS = 1e-8
    step64 = (v["Hinv_g"] + nu64 * v["Hinv_b"]) / (lam64 + EPS) if case > 0 else nu64 * v["Hinv_b"]
    step64 = step64 / step64.norm()
    errs["step"] = float((v["step"] - step64).norm())
    # the line search, at every beta the device tried, fed the device's step vector
    beta_dev = st["loss/step_size"]
    k_dev = int(round(math.log(beta_dev) / math.log(p._backtrack_coeff)))
    assert abs(beta_dev - p._backtrack_coeff ** k_dev) < 1e-12
    exhausted = k_dev == p._max_backtracks
    accepted = None
    obj0, cost0, cval = st["loss/rew_loss"], st["loss/cost_loss"], st["loss/optim_C"]
    for k in range(min(k_dev + 1, p._max_backtracks)):
        beta = p._backtrack_coeff ** k
        tk = _terms64(s, sq, th0 + beta * v["step"], R, p._ave_cost_return, mean_adv_c)
        conds = [(delta - tk["kl"], tk["s_kl"]), (max(-cval, 0) - (tk["cost"] - cost0), tk["s_cost"] + t0["s_cost"])]
        if case > 1:
            conds.append((tk["obj"] - obj0, tk["s_obj"] + t0["s_obj"]))
        if _decide(conds):
            accepted = k
            break
    assert accepted == (None if exhausted else k_dev), (accepted, k_dev)
    beta_last = beta_dev if not exhausted else p._backtrack_coeff ** (p._max_backtracks - 1)
    want = v["theta0"] + beta_last * v["step"]
    errs["theta"] = _ulps(theta1, want, v["theta0"].abs() + (beta_last * v["step"]).abs())
    bounds = {k: ULP_TOL if k == "theta" else (SUM_TOL if k.endswith("_loss") else DUAL_TOL) for k in errs}
    _report(f"cpo case {case} (c={c64:.3e} B={B64:.3e}) beta={beta_dev:.3f} accepted={accepted}", errs, bounds)


# ---- 7. TRPO-Lagrangian ----------------------------------------------------------------------------------------
def _trpo_run(p, batch, n_all, seed):
    """learn() on one whole-batch minibatch, with the masks and theta its step starts from"""
    s = p.arena.slots[0]
    np.random.seed(seed)
    perm = torch.as_tensor(np.random.permutation(n_all).astype(np.int32), device="cuda")
    dv = _Dev(p, batch, perm, n_all)
    p._refresh_old_dist(batch)
    masks = dv.forward()
    th0 = _d(dv.theta())
    np.random.seed(seed)
    p.learn(batch, batch_size=n_all, repeat=1)
    torch.cuda.synchronize()
    v = {k: _d(t).clone() for k, t in p._vec.items()}
    st = {k: vv[0] for k, vv in p.last_stats.items()}
    return dv, perm, masks, th0, v, st, s


@pytest.mark.parametrize("opt", ["lagrangian", "no-lagrangian", "exhaustion"])
def test_trpo_step(opt):
    A, D, n_all = 2, 9, 3000
    kw = dict(optim_critic_iters=1)
    if opt == "no-lagrangian":
        kw["use_lagrangian"] = False
    if opt == "exhaustion":
        kw.update(use_lagrangian=False, target_kl=1.0, max_backtracks=2)
    p = _policy("trpo", D, A, 1.0, H=64, bounded=True, **kw)
    s = p.arena.slots[0]
    if opt == "exhaustion":
        # every mean starts deep in tanh's saturation (z ~ 3, mu' ~ 0.01): the Fisher matrix sees a small curvature
        # there, the step it allows carries z into the linear range, and the true KL outgrows the quadratic model
        _, _, _, _, w3, b3, ex = s.offsets()
        p.arena.theta[w3:b3] *= 0.01
        p.arena.theta[b3:ex] = 3.0
    batch, _ = _batch(p, n_all, seed=8)
    if opt == "exhaustion":
        batch.adv[0] = -batch.eps[:, 0].float()                 # the objective pushes the first mean down
        batch.adv[1] = 0.0
    if p.lag_optims:
        p.lag_optims[0].lagrangian = 0.5
    lag = p.lagrangians()[0] if p.use_lagrangian else 0.0
    resc = p.rescaling_factor() if p.use_lagrangian else 1.0
    dv, perm, masks, th0, v, st, s = _trpo_run(p, batch, n_all, seed=9)
    sq, R = _Sq(p), _Rows(batch, perm, n_all)
    theta1 = _d(dv.theta())
    assert torch.equal(v["theta0"], th0)
    errs = {}
    # flat = -resc (g + lambda b), from the device's g and b
    want = -resc * (v["g"] + lag * v["b"])
    sp = torch.from_numpy(np.spacing((resc * (v["g"].abs() + lag * v["b"].abs())).float().cpu().numpy())).double().cuda()
    errs["flat"] = float(((v["step"] - want).abs() / sp).max())
    sd = v["Hinv_g"]
    mvp = _hvp64(_kl_mean64(s, sq, R, masks), th0)
    shs64 = float(sd @ mvp(sd))
    errs["shs"] = abs(float(sd @ v["hv"]) - shs64) / shs64
    ss0 = math.sqrt(2 * p._delta / shs64)
    # the line search in float64 at every step the device tried
    def loss_of(t):
        return resc * (-t["obj"] + lag * (t["cost"]))

    ratio_terms = lambda th: _terms64(s, sq, th, R, 0.0, 0.0)
    t0 = ratio_terms(th0)
    loss0 = loss_of(t0)
    errs["actor_total"] = abs(st["loss/actor_total"] - loss0) / (resc * (t0["s_obj"] + lag * t0["s_cost"]))
    accepted, tried = None, p._max_backtracks
    ss_dev = st["loss/step_size"]
    if ss_dev > 0:
        tried = int(round(math.log(ss_dev / ss0) / math.log(p._backtrack_coeff))) + 1
        errs["step_size"] = abs(ss_dev / (ss0 * p._backtrack_coeff ** (tried - 1)) - 1)
    for k in range(tried):
        tk = ratio_terms(th0 + ss0 * p._backtrack_coeff ** k * sd)
        conds = [(p._delta - tk["kl"], tk["s_kl"]),
                 (loss0 - loss_of(tk), resc * (tk["s_obj"] + t0["s_obj"] + lag * (tk["s_cost"] + t0["s_cost"])))]
        if _decide(conds):
            accepted = k
            break
    if opt == "exhaustion":
        assert ss_dev == 0.0 and accepted is None
        assert not torch.equal(theta1, th0)             # the last tried parameters stay
    else:
        assert accepted == tried - 1, (accepted, tried)
    if ss_dev > 0:          # the device's own step size: the update is one fp32 axpy
        errs["theta"] = _ulps(theta1, th0 + ss_dev * sd, th0.abs() + (ss_dev * sd).abs())
    else:                   # the last tried step, from the float64 step size: within its DUAL_TOL
        step = ss0 * p._backtrack_coeff ** (tried - 1) * sd
        sp = torch.from_numpy(np.spacing((th0.abs() + step.abs()).float().cpu().numpy())).double().cuda()
        errs["theta_last"] = _err(theta1, th0 + step, step.abs(), ULP_TOL * sp)
    bounds = {"flat": ULP_TOL, "shs": DUAL_TOL, "actor_total": SUM_TOL, "step_size": DUAL_TOL, "theta": ULP_TOL,
              "theta_last": DUAL_TOL}
    _report(f"trpo {opt} lag={lag} tried={tried} step_size={ss_dev:.4e}", errs, bounds)


# ---- 8. FOCOPS actor step --------------------------------------------------------------------------------------
def _focops_head64(sq, z, ls, R, adv_r, adv_c, inv_lam, nu, eta):
    n = z.shape[0]
    z = z.clone().requires_grad_(True)
    lsr = ls.view(1, -1).expand_as(z).clone().requires_grad_(True)
    mu, sg = sq.mu(z), lsr.exp()
    zz = (R.act - mu) / sg
    lp_terms = -0.5 * zz ** 2 - lsr - LOG_SQRT_2PI
    ratio = torch.exp(lp_terms.sum(1) - R.lpo)
    s_lp = (0.5 * zz ** 2 + lsr.abs() + LOG_SQRT_2PI).sum(1) + R.lpo.abs()
    vr, t1 = (sg / R.so) ** 2, ((mu - R.mo) / R.so) ** 2
    kl_t = 0.5 * (vr + t1 - 1 - vr.log())
    kl = kl_t.sum(1)
    kl_s = (0.5 * (vr + t1 + 1 + vr.log().abs())).sum(1)
    adv = adv_r - nu * adv_c
    keep = (kl <= eta).double().detach() if eta is not None else torch.ones_like(kl)
    L = (kl - inv_lam * ratio * adv) * keep
    gz, gl = torch.autograd.grad(L.mean(), (z, lsr))
    with torch.no_grad():
        gr = (inv_lam * (adv_r.abs() + abs(nu) * adv_c.abs()) * ratio * (1 + s_lp)).view(-1, 1)
        mup, k = sq.mup_mag(z), keep.view(-1, 1) / n
        mz = k * ((mu.abs() + R.mo.abs()) / R.so ** 2 + gr * (R.act.abs() + mu.abs()) / sg ** 2) * mup
        ml = k * (vr + 1 + gr * (zz ** 2 + 1))
    sums = [float(L.sum()), float(kl.sum()), float(keep.sum())]
    scl = [float(((kl_s + (inv_lam * ratio * adv).abs() * (1 + s_lp)) * keep).sum()), float(kl_s.sum()), 1.0]
    return kl.detach(), kl_s.detach(), sums, scl, torch.cat([gz, gl], 1), torch.cat([mz, ml], 1)


@pytest.mark.parametrize("A,high,bounded,H,tem_lambda,clip,grown", [
    (2, 1.0, True, 64, 0.1, True, False), (3, 2.0, True, 128, 0.95, True, False),
    (8, 1.0, False, 256, 0.1, True, False), (2, 1.0, False, 64, 50.0, False, False), (2, 1.0, True, 64, 0.1, True, True)],
    ids=["A2-b1-clip", "A3-b2-clip", "A8-unbounded-clip", "A2-unbounded-noclip", "A2-b1-clip-grown"])
def test_focops_step(A, high, bounded, H, tem_lambda, clip, grown):
    """the merged last chunk of Batch.split(4000, merge_last=True) over 10 000 rows: 6000 rows, above one wgrad split.
    tem_lambda sets the weight of the advantage term, and with it whether max_grad_norm = 0.5 clips.  grown: the
    warm-up step runs on a 3000-row engine, which the checked step's 6000 rows grow; Adam continues its moments"""
    D, n_all, n = 7 + A, 10_000, 6000
    p = _policy("focops", D, A, high, H=H, bounded=bounded, tem_lambda=tem_lambda, nu=0.3, auto_nu=False,
                max_grad_norm=0.5)
    batch, _ = _batch(p, n_all, seed=10 + A, saturate=bounded)
    perm = _perm(batch.n, n, 12)
    p._eta = 1e9
    n_warm = n // 2 if grown else n
    p._ensure_engine(n_warm)
    p.policy_loss(batch, perm[:n_warm], n_warm)  # warm-up: Adam moments away from zero
    eng_warm = p._eng
    dv = _Dev(p, batch, perm, n)
    assert (dv.eng is not eng_warm) == grown
    s, sq, R = dv.a, _Sq(p), _Rows(batch, perm, n)
    _move(p, 13, 0.05 if clip else 0.03)        # and theta well away from theta_old, so the per-row KLs spread
    dv.eng.sync_mirror([s])
    masks = dv.forward()
    z = _d(dv.view("out")[:, :A])
    th0 = _d(dv.theta())
    ls = _parts(s, th0)["ls"]
    # eta in the widest gap of the sorted float64 per-row KLs around the median
    kl, kl_s, _, _, _, _ = _focops_head64(sq, z, ls, R, R.ar, R.ac, 1 / tem_lambda, p._nu, None)
    ks, order = torch.sort(kl)
    lo, hi = int(0.3 * n), int(0.7 * n)
    gaps = ks[lo + 1:hi + 1] - ks[lo:hi]
    j = int(torch.argmax(gaps)) + lo
    eta = float(0.5 * (ks[j] + ks[j + 1]))
    gap = float(ks[j + 1] - ks[j])
    # a row's fp32 KL is a handful of operations off by an ulp each: MARGIN ulps of its term sum clear it
    assert gap / 2 > MARGIN * F32_EPS * float(kl_s[order[j:j + 2]].max()), (gap, kl_s[order[j:j + 2]])
    p._eta = eta
    sl = slice(s.offset, s.offset + s.size)
    m0, v0, t0 = _d(eng_warm.adam_m[sl]).clone(), _d(eng_warm.adam_v[sl]).clone(), p._actor_t   # the warm-up's moments
    st = p.policy_loss(batch, perm, n)
    errs = {}
    # per-minibatch normalised advantages (unbiased std)
    an = {}
    for c, a in ((0, R.ar), (1, R.ac)):
        an[c] = (a - a.mean()) / a.std()
        errs[f"adv{c}"] = _err(p._adv_n[c][perm.long()], an[c], 1 + a.abs().max() / a.std())
    kl, kl_s, sums, scl, dref, dmag = _focops_head64(sq, z, ls, R, an[0], an[1], 1 / tem_lambda, p._nu, eta)
    got = p._sums.cpu().numpy()
    assert got[2] == sums[2] == j + 1
    errs["loss"] = abs(got[0] - sums[0]) / scl[0]
    errs["kl"] = abs(got[1] - sums[1]) / scl[1]
    errs["stat"] = max(abs(st["loss/actor_loss"] - sums[0] / n) / (scl[0] / n), abs(st["loss/kl"] - sums[1] / n) / (scl[1] / n))
    dout = _d(dv.view("dout"))
    assert (dout[:, 2 * A:] == 0).all()
    errs["dout"] = _err(dout[:, :2 * A], dref, dmag, FLT_MIN)
    grad = _d(p.arena.grad[sl])
    gref = _wgrad_ref(s, th0, R.x, masks, dout)
    errs["grad"] = _err(grad, gref, _grad_scale(s, th0, R.x, masks, dout.abs()), n * FLT_MIN * (1 + float(R.x.abs().max())))
    nsq = float(p._norm_sq.item())
    nsq64 = float(grad @ grad)
    errs["norm"] = abs(nsq - nsq64) / nsq64
    # clipping or not, decided with room to spare; Adam is then fed the device's gradient and norm
    assert (math.sqrt(nsq64) > 0.5 * 1.1) if clip else (math.sqrt(nsq64) < 0.5 / 1.1), nsq64
    f32 = np.float32
    scale = float(min(f32(0.5) / (np.sqrt(f32(nsq)) + f32(1e-6)), f32(1.0)))
    gc = grad * scale
    g = p.actor_optim.param_groups[0]
    ref, m, vv = adam64(th0, gc, m0, v0, t0 + 1, g["lr"], betas=g["betas"], eps=g["eps"])
    th1 = _d(dv.theta())
    errs["adam"] = max(_ulps(th1, ref, ref.abs() + g["lr"]), _ulps(_d(dv.eng.adam_m[sl]), m, m0.abs() + gc.abs()),
                       _ulps(_d(dv.eng.adam_v[sl]), vv, v0 + gc * gc))
    bounds = {"adv0": STD_TOL, "adv1": STD_TOL, "loss": SUM_TOL, "kl": SUM_TOL, "stat": SUM_TOL, "dout": DOUT_TOL,
              "grad": GRAD_TOL, "norm": SUM_TOL, "adam": ULP_TOL}
    _report(f"focops A={A} high={high} bounded={bounded} H={H} grown={grown} eta={eta:.3e} kept={j + 1}/{n} "
            f"|g|={math.sqrt(nsq64):.3f}", errs, bounds)


# ---- 9. critic step --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("algo,l2,grown", [("cpo", 1e-3, False), ("focops", 1e-3, False), ("trpo", 0.0, False),
                                           ("trpo", 0.0, True)],
                         ids=["cpo-0.001", "focops-0.001", "trpo-0.0", "trpo-0.0-grown"])
def test_critic_step(algo, l2, grown):
    """grown: the warm-up step runs on a 2000-row engine and the checked step on a 5000-row one, as learn() grows
    the engine for a collect larger than all before it; Adam continues the warm-up's moments"""
    D, A, n_all, n = 12, 2, 6000, 5000
    p = _policy(algo, D, A, H=128)
    assert p._l2_reg == l2
    batch, _ = _batch(p, n_all, seed=14)
    perm = _perm(batch.n, n, 15)
    n_warm = 2000 if grown else n
    p._ensure_engine(n_warm)
    p.critics_loss(batch, perm[:n_warm], n_warm)         # warm-up: Adam moments away from zero
    eng = p._eng
    th0, m0, v0 = _d(p.arena.theta).clone(), _d(eng.adam_m).clone(), _d(eng.adam_v).clone()
    p._ensure_engine(n)
    assert (p._eng is not eng) == grown
    eng = p._eng
    crit = p.arena.slots[1:3]
    t0 = p._critic_t
    st = p.critics_loss(batch, perm, n)
    torch.cuda.synchronize()
    th1, m1, v1, grad = _d(p.arena.theta), _d(eng.adam_m), _d(eng.adam_v), _d(p.arena.grad)
    x = _d(batch.obs[perm.long()])
    g = p.optim.param_groups[0]
    errs = {}
    for i, s in enumerate(crit):
        sl = slice(s.offset, s.offset + s.size)
        masks = ((_d(eng.slot_view(s, "h1")[:n]) > 0).double(), (_d(eng.slot_view(s, "h2")[:n]) > 0).double())
        th = th0[sl].clone().requires_grad_(True)
        _, _, out = _mlp64(s, th, x, masks)
        _, _, om = _mag_chain(s, th0[sl], x, masks)
        ret = _d(batch.ret[i][perm.long()])
        td = out[:, 0] - ret
        mse = (td ** 2).mean()
        (gref,) = torch.autograd.grad(mse, th)
        dmag = (2 * (om[:, 0] + ret.abs()) / n).view(-1, 1)
        errs[f"grad{i}"] = _err(grad[sl], gref, _grad_scale(s, th0[sl], x, masks, dmag))
        l2term = l2 * float(th0[sl] @ th0[sl])
        errs[f"vf{i}"] = abs(st[f"loss/vf{i}"] - (float(mse) + l2term)) / (float(((om[:, 0] + ret.abs()) ** 2).mean()) + l2term)
        ref, m, v = adam64(th0[sl], grad[sl], m0[sl], v0[sl], t0 + 1, g["lr"], betas=g["betas"], eps=g["eps"],
                           weight_decay=2 * l2)
        gd = grad[sl] + 2 * l2 * th0[sl]
        errs[f"adam{i}"] = max(_ulps(th1[sl], ref, ref.abs() + g["lr"]), _ulps(m1[sl], m, m0[sl].abs() + gd.abs()),
                               _ulps(v1[sl], v, v0[sl] + gd * gd))
    bounds = {k: {"gra": GRAD_TOL, "vf": SUM_TOL, "ada": ULP_TOL}[k[:3] if k[:2] != "vf" else "vf"] for k in errs}
    _report(f"critic {algo} l2={l2} n={n} grown={grown}", errs, bounds)
