"""SAC- and DDPG-Lagrangian gradient steps (fsrl_offpolicy_steps) one step at a time against float64
autograd.  After ``update_many(1, B, buf)`` the device still holds what that step computed: the
critic-loss gradient in the critic slots of ``arena.grad`` and the actor-loss gradient in the actor
slot (Adam reads ``grad`` without clearing it, and the actor loss's backward through the critics
computes input gradients only), the n-step / target / sample work arrays in ``policy._w``, the
actor-phase head gradients in the engine's ``dout`` scratch and ``[log alpha, m, v, t]`` in
``policy._alpha_state``.  Each stage is checked against its own float64 value, fed the device's
output of the stage before it, so that an error points at the kernel that made it:

  target   the n-step walk, the target-side sample (Philox stream 0) and the n-step target
  critic   d/dtheta of sum_i sum_j mean((q_ij - target_i)^2) at the pre-step critics
  actor    the actor-side sample (stream 1), d loss / d Q and d/dtheta_actor of
           resc * (mean(alpha * logp - min(Q00, Q01)) + lambda * mean(min(Q10, Q11))) at the
           post-step critics (DDPG: resc * (-mean Q0 + lambda * mean Q1))
  adam     both Adam steps and the Polyak updates applied to the device's own gradients
  alpha    the automatic temperature step

The float64 networks take their ReLU masks from the device's saved activations: a unit whose
pre-activation is within fp32 rounding of zero may switch on one side only, and one such row moves a
column of the weight gradient by ~1/sqrt(B) of its size.  The tanh squash uses the device's fp32
sample a (from ``keep``) for its value and its derivative 1 - a^2: where |u| > ~9, fp32 tanh rounds
to +-1 and -log(1 - a^2 + eps) is as ill-conditioned as the rounding of a, so the float64 reference
evaluates the loss at the sample the device drew; a itself is checked against tanh(u) in float64."""
import math

import numpy as np
import pytest
import torch

from helpers import adam64, synthetic_ring, upd_noise

pytestmark = pytest.mark.gpu

TASK_BY_A = {2: "SafetyCarRun-v0", 3: "SafetyHopperVelocityGymnasium-v1", 4: "SafetyDroneRun-v0",
             6: "SafetyHalfCheetahVelocityGymnasium-v1", 8: "SafetyAntRun-v0"}
BUTTON = "SafetyCarButton1Gymnasium-v0"             # D = 76: critic input 78 of FSRL_ENG_DX_LD = 80
F32_EPS = float(np.finfo(np.float32).eps)
LOG_SQRT_2PI = 0.5 * math.log(2.0 * math.pi)

# Bounds: about 10x the worst value observed over all cases on an H100 80GB HBM3 (700 W power limit), which is
# given in each comment; every case prints its errors.
EPS_TOL = 1e-7       # |eps - eps64| / (1 + |eps64|), replayed Philox normals: observed 0 (bit-exact)
ACT_TOL = 1e-5       # |a - tanh(u64)| / (1 + |u64|), DDPG |a - a64| / max_action, and sigma relative: 1.3e-6
LOGP_TOL = 5e-6      # |logp - logp64| / sum_j |terms_j| (the row's own condition number): 5.1e-7
NSTEP_TOL = 2e-15    # gamma^k and the discounted sums, float64 on both sides: 2.1e-16
TARGET_TOL = 7e-6    # |target - ref| / (|partial| + gamma^k (sum |terms| of Q' + alpha |logp'|)): 7.0e-7
GRAD_TOL = 1e-4      # per tensor |got - ref|max / max|ref|: 8.4e-6 on a DDPG critic's b2 (a sum over the rows
                     # that cancels), <= 1.9e-6 on every other tensor
DOUT_TOL = 1e-6      # actor-phase d loss / d Q per critic, relative to max|ref|: 7.5e-8
LOSS_TOL = 1e-5      # loss/q*, loss/actor_*: relative to the mean |term|: 7.8e-7
ULP_TOL = 8.0        # Adam / Polyak results in fp32 ulps of their operands' scale: 2.6 (Adam), 1.15 (Polyak)
ALPHA_TOL = 2e-6     # log alpha (in units of its step), m, v, alpha_loss, alpha_value against their scales: 1.9e-7


class _BoxEnv:
    """The two spaces an agent reads: a user env with Box(-high, high) actions."""

    def __init__(self, D, A, high):
        from fsrl_b200.spaces import Box
        self.observation_space = Box(-np.inf, np.inf, (D,), np.float32)
        self.action_space = Box(-high, high, (A,), np.float32)


def _policy(algo, task=None, env=None, hidden=(64, 64), bounded=True, lam=0.8, seed=3, **kw):
    from fsrl_b200 import envs
    from fsrl_b200.agent import DDPGLagAgent, SACLagAgent
    env = env if env is not None else envs.make(task)
    if algo == "sac":
        agent = SACLagAgent(env, seed=seed, hidden_sizes=hidden, unbounded=not bounded, **kw)
    else:
        agent = DDPGLagAgent(env, seed=seed, hidden_sizes=hidden, **kw)
    p = agent.policy
    if p.lag_optims:
        p.lag_optims[0].lagrangian = lam
    return p


def _blocks(s):
    """(name, lo, hi) of the slot's tensors relative to its offset"""
    w1, b1, w2, b2, w3, b3, ex = (o - s.offset for o in s.offsets())
    return [("w1", w1, b1), ("b1", b1, w2), ("w2", w2, b2), ("b2", b2, w3), ("w3", w3, b3), ("b3", b3, ex)]


def _tensors(s, v, split=0):
    """the slot vector v (arena layout) as named tensors; split = A separates the mu and sigma columns of the
    SAC actor's head"""
    d = {n: v[lo:hi] for n, lo, hi in _blocks(s)}
    d["w3"] = d["w3"].reshape(s.H, s.out)
    if split:
        d["w3.mu"], d["w3.sigma"] = d["w3"][:, :split], d["w3"][:, split:]
        d["b3.mu"], d["b3.sigma"] = d["b3"][:split], d["b3"][split:]
        del d["w3"], d["b3"]
    return d


def _mlp64(th, s, x, masks=None, cond=False):
    """the slot's MLP in float64 from its arena vector th; masks = the device's (h1 > 0, h2 > 0), or ReLU.
    cond=True also returns the head's sum of |terms| |h2| |W3| + |b3|, the scale of its rounding error"""
    t = {n: th[lo:hi] for n, lo, hi in _blocks(s)}
    act = (lambda z, k: z * masks[k]) if masks is not None else (lambda z, k: torch.relu(z))
    h = act(x @ t["w1"].view(s.D, s.H) + t["b1"], 0)
    h = act(h @ t["w2"].view(s.H, s.H) + t["b2"], 1)
    out = h @ t["w3"].view(s.H, s.out) + t["b3"]
    if cond:
        return out, (h.abs() @ t["w3"].view(s.H, s.out).abs() + t["b3"].abs()).detach()
    return out


def _rel(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    m = np.abs(ref).max()
    return float(np.abs(got - ref).max() / m) if m > 0 else float(np.abs(got).max())


def _grad_errs(errs, tag, s, got_vec, ref_vec, dout, split=0):
    """per tensor |got - ref|max / max|ref|; a head bias's gradient is a sum over the rows of d loss / d out that
    may cancel, so it is measured against sum_b |d loss / d out_b| of its column instead"""
    got, ref = _tensors(s, got_vec, split), _tensors(s, ref_vec, split)
    dsum = dout.abs().sum(0).numpy()
    cols = {"b3": dsum, "b3.mu": dsum[:split], "b3.sigma": dsum[split:]}
    for k in ref:
        if k in cols:
            g, r, c = (np.asarray(v, np.float64) for v in (got[k], ref[k], cols[k]))
            errs[f"{tag}.{k}"] = float(np.where(c > 0, np.abs(g - r) / np.where(c > 0, c, 1), np.abs(g)).max())
        else:
            errs[f"{tag}.{k}"] = _rel(got[k], ref[k])
    return ref


def _ulps(got, ref, scale):
    sp = np.spacing(np.abs(np.asarray(scale, np.float64)).astype(np.float32)).astype(np.float64)
    return float((np.abs(np.asarray(got, np.float64) - np.asarray(ref, np.float64)) / sp).max())


def _nstep64(b, idx, gamma, n):
    """compute_nstep_returns' walk in float64: terminal index, gamma^k, discounted rew / cost sums, value mask"""
    cap, ptr = b["cap"], b["ptr"]
    env = idx // cap
    newest = env * cap + (ptr[env] - 1) % cap
    done = b["term"] | b["trunc"]
    cur, alive = idx.copy(), np.ones(len(idx), bool)
    g = np.zeros(len(idx), np.int64)
    rets = np.zeros((2, len(idx)))
    for k in range(n):
        rets += alive * gamma ** k * np.stack([b["rew"][cur], b["cost"][cur]]).astype(np.float64)
        g += alive
        end = done[cur] | (cur == newest)
        alive &= ~end
        if k < n - 1:
            cur = np.where(end, cur, env * cap + (cur % cap + 1) % cap)
    return cur, gamma ** g.astype(np.float64), rets, (~b["term"][cur]).astype(np.float64)


class _Step:
    """One checked gradient step: the device state before it, the call, and the device state after it."""

    def __init__(self, policy, buf, B, seed=1, edit=None):
        self.p, self.B = policy, B
        self.g = policy._groups()
        self.sac = "actor_old" not in self.g
        eng = policy._ensure_engine(B)
        np.random.seed(seed + 1000)
        policy.update_many(1, B, buf)                 # warm-up: Adam moments and log alpha away from their start
        if edit is not None:
            edit(policy, eng)
            eng.sync_mirror(policy.arena.slots)
        np.random.seed(seed)
        self.idx_t = policy.sample_batch_indices(buf, 1, B)[0]
        self.idx = self.idx_t.cpu().numpy().astype(np.int64)
        c = lambda t: t.detach().cpu().double().clone()
        ar = policy.arena
        # the critic phase's activation masks: the same forward launch the step makes, on the same inputs
        crit = self.g["critics"]
        eng.forward(crit, eng.make_input(buf.obs, self.idx_t, buf.act, self.idx_t), B, save=True)
        self.crit_masks = [(c(eng.slot_view(s, "h1")[:B]) > 0, c(eng.slot_view(s, "h2")[:B]) > 0) for s in crit]
        self.theta0, self.m0, self.v0 = c(ar.theta), c(eng.adam_m), c(eng.adam_v)
        self.noise_t, self.critic_t, self.actor_t = policy._noise_t, policy._critic_t, policy._actor_t
        if self.sac:
            self.alpha = float(policy._alpha_dev.item())
            self.alpha_state0 = c(policy._alpha_state)
        self.lam = policy.lagrangians()[0] if policy.lag_optims else 0.0
        self.lagr = bool(policy.use_lagrangian and policy.critics_num > 1)
        self.resc = policy.rescaling_factor() if policy.use_lagrangian else 1.0
        np.random.seed(seed)
        policy.update_many(1, B, buf)
        torch.cuda.synchronize()
        self.stats = {k: float(np.asarray(v)[0]) for k, v in policy.last_stats.items()}
        self.theta1, self.m1, self.v1, self.grad = c(ar.theta), c(eng.adam_m), c(eng.adam_v), c(ar.grad)
        self.w = {k: c(v) for k, v in policy._w.items()}
        self.dout = {id(s): c(eng.slot_view(s, "dout")[:B]) for s in crit}
        self.masks = {id(s): (c(eng.slot_view(s, "h1")[:B]) > 0, c(eng.slot_view(s, "h2")[:B]) > 0)
                      for s in crit + self.g["actor"]}
        if self.sac:
            self.alpha_state1 = c(policy._alpha_state)
        self.buf = {k: getattr(buf, k).cpu().numpy() for k in ("obs", "obs_next", "act", "rew", "cost")}
        self.buf.update(term=buf.terminated.cpu().numpy().astype(bool), trunc=buf.truncated.cpu().numpy().astype(bool),
                        ptr=buf.ptr.cpu().numpy().astype(np.int64), cap=buf.cap)

    def slot(self, theta, s, grad=False):
        v = theta[s.offset:s.offset + s.size].clone()
        return v.requires_grad_(True) if grad else v


def _target_errs(st, errs):
    p, B, A, b = st.p, st.B, st.p._A, st.buf
    C, per = p.critics_num, (2 if p._twin else 1)
    term, gpow, part, vmask = _nstep64(b, st.idx, p._gamma, p._n_step)
    w = st.w
    assert np.array_equal(w["term_idx"][:B].numpy().astype(np.int64), term)
    assert np.array_equal(w["vmask"][:B].numpy(), vmask)
    errs["gpow"] = _rel(w["gpow"][:B].numpy(), gpow)
    scale = np.abs(part).max()
    errs["partial"] = float(np.abs(w["partial"][:2 * B].numpy().reshape(2, B)[:C] - part[:C]).max() / scale)
    s_next = torch.from_numpy(b["obs_next"][term]).double()
    a_next = w["act_next"][:B]
    if st.sac:
        a = st.g["actor"][0]
        out = _mlp64(st.slot(st.theta0, a), a, s_next)
        out = out.detach()
        mu = p.actor._max * torch.tanh(out[:, :A]) if not p.actor._unbounded else out[:, :A]
        sig = out[:, A:].clamp(-20.0, 2.0).exp()
        eps = upd_noise(p._upd_seed, B, A, st.noise_t, 0).double()
        u = mu + sig * eps
        errs["act_next"] = float(((a_next - torch.tanh(u)).abs() / (1 + u.abs())).max())
        terms = torch.stack([-0.5 * eps ** 2, -sig.log(), torch.full_like(eps, -LOG_SQRT_2PI),
                             -torch.log(1 - a_next ** 2 + F32_EPS)])
        lp = terms.sum((0, 2))
        errs["logp_next"] = float(((w["logp_next"][:B] - lp).abs() / terms.abs().sum((0, 2))).max())
    else:
        a = st.g["actor_old"][0]
        ref = p.actor._max * torch.tanh(_mlp64(st.slot(st.theta0, a), a, s_next))
        errs["act_next"] = float((a_next - ref).abs().max() / p.actor._max)
    x = torch.cat([s_next, a_next], 1)
    tgt, scl = [], []
    for i in range(C):
        qc = [_mlp64(st.slot(st.theta0, s), s, x, cond=True) for s in st.g["critics_old"][per * i:per * i + per]]
        q = torch.minimum(*(o[:, 0] for o, _ in qc)) if per == 2 else qc[0][0][:, 0]
        mag = torch.stack([c[:, 0] for _, c in qc]).max(0).values      # a Q value near 0 is still a long sum
        if st.sac:
            q = q - st.alpha * w["logp_next"][:B]
            mag = mag + st.alpha * w["logp_next"][:B].abs()
        tgt.append(q.numpy() * vmask * gpow + part[i])
        scl.append(np.abs(part[i]) + gpow * mag.numpy())
    got = w["target"][:C * B].numpy().reshape(C, B)
    errs["target"] = float((np.abs(got - np.stack(tgt)) / np.stack(scl)).max())
    return errs


def _critic_errs(st, errs):
    p, B, b = st.p, st.B, st.buf
    C, per = p.critics_num, (2 if p._twin else 1)
    x = torch.from_numpy(np.concatenate([b["obs"][st.idx], b["act"][st.idx]], 1)).double()
    tgt = st.w["target"][:C * B].view(C, B)
    loss, li = 0.0, []
    nets = []
    for i in range(C):
        l_i = 0.0
        for j in range(per):
            n = per * i + j
            s = st.g["critics"][n]
            th = st.slot(st.theta0, s, grad=True)
            q = _mlp64(th, s, x, st.crit_masks[n])
            q.retain_grad()
            nets.append((s, th, q))
            l_i = l_i + ((q[:, 0] - tgt[i]) ** 2).mean()
        li.append(float(l_i))
        loss = loss + l_i
    loss.backward()
    for n, (s, th, q) in enumerate(nets):
        _grad_errs(errs, f"gq{n}", s, st.slot(st.grad, s), th.grad, q.grad)
    for i in range(C):
        errs[f"loss/q{i}"] = abs(st.stats[f"loss/q{i}"] - li[i]) / li[i]
    return errs


def _actor_errs(st, errs):
    p, B, A, b = st.p, st.B, st.p._A, st.buf
    C, per = p.critics_num, (2 if p._twin else 1)
    obs = torch.from_numpy(b["obs"][st.idx]).double()
    a_s = st.g["actor"][0]
    th = st.slot(st.theta0, a_s, grad=True)
    out = _mlp64(th, a_s, obs, st.masks[id(a_s)])
    out.retain_grad()
    w = st.w
    if st.sac:
        keep = w["keep"][:B]
        eps_d, sig_d, a_d = keep[:, :A], keep[:, 8:8 + A], keep[:, 16:16 + A]
        eps = upd_noise(p._upd_seed, B, A, st.noise_t, 1).double()
        errs["eps"] = float(((eps_d - eps).abs() / (1 + eps.abs())).max())
        mu = p.actor._max * torch.tanh(out[:, :A]) if not p.actor._unbounded else out[:, :A]
        sig = out[:, A:].clamp(-20.0, 2.0).exp()
        errs["sigma"] = _rel(sig_d / sig.detach(), torch.ones_like(sig))
        u = mu + sig * eps
        errs["act"] = float(((a_d - torch.tanh(u.detach())).abs() / (1 + u.detach().abs())).max())
        assert torch.equal(w["act"][:B], a_d)
        act = a_d + (u - u.detach()) * (1 - a_d ** 2)        # the device's sample, tanh' taken at it
        logp = torch.distributions.Normal(mu, sig).log_prob(u).sum(-1) - torch.log(1 - act ** 2 + F32_EPS).sum(-1)
        lp_scale = (0.5 * eps ** 2 + sig.detach().log().abs() + LOG_SQRT_2PI + torch.log(1 - a_d ** 2 + F32_EPS).abs()).sum(-1)
        errs["logp"] = float(((w["logp"][:B] - logp.detach()).abs() / lp_scale).max())
    else:
        act = p.actor._max * torch.tanh(out)
        errs["act"] = float((w["act"][:B] - act.detach()).abs().max() / p.actor._max)
    x = torch.cat([obs, act], 1)
    qmin, qs = [], []
    for i in range(C):
        q_i = []
        for j in range(per):
            s = st.g["critics"][per * i + j]
            q = _mlp64(st.slot(st.theta1, s), s, x, st.masks[id(s)])[:, 0]
            q.retain_grad()
            q_i.append(q); qs.append((s, q))
        qmin.append(torch.minimum(*q_i) if per == 2 else q_i[0])
    rew = (st.alpha * logp - qmin[0]).mean() if st.sac else -qmin[0].mean()
    saf = st.lam * qmin[1].mean() if st.lagr else torch.zeros((), dtype=torch.float64)
    loss = st.resc * (rew + saf)
    loss.backward()
    # relative to the mean magnitude of the terms, which a cancelling sum cannot make small
    rew_terms = (st.alpha * logp.detach()).abs() + qmin[0].detach().abs() if st.sac else qmin[0].detach().abs()
    errs["loss/actor_rew"] = abs(st.stats["loss/actor_rew"] - float(rew)) / float(rew_terms.mean())
    if st.lagr:
        errs["loss/actor_safety"] = abs(st.stats["loss/actor_safety"] - float(saf)) / float(st.lam * qmin[1].detach().abs().mean())
    for n, (s, q) in enumerate(qs):
        # a cost critic outside the loss (use_lagrangian=False) gets no gradient: the device writes zeros
        errs[f"dq{n}"] = _rel(st.dout[id(s)][:, 0], q.grad if q.grad is not None else torch.zeros_like(q))
    st.actor_grad_ref = _grad_errs(errs, "ga", a_s, st.slot(st.grad, a_s), th.grad, out.grad, A if st.sac else 0)
    return errs


def _adam_errs(st, errs):
    p = st.p
    for name, slots, lr, t in (("adam_c", st.g["critics"], p._critic_lr, st.critic_t + 1),
                               ("adam_a", st.g["actor"], p._actor_lr, st.actor_t + 1)):
        e = 0.0
        for s in slots:
            sl = slice(s.offset, s.offset + s.size)
            g = st.grad[sl]
            ref, m, v = adam64(st.theta0[sl], g, st.m0[sl], st.v0[sl], t, lr)
            e = max(e, _ulps(st.theta1[sl], ref, ref.abs() + lr),
                    _ulps(st.m1[sl], m, st.m0[sl].abs() + g.abs()),
                    _ulps(st.v1[sl], v, st.v0[sl] + g * g))
        errs[name] = e
    pairs = list(zip(st.g["critics_old"], st.g["critics"]))
    if not st.sac:
        pairs.append((st.g["actor_old"][0], st.g["actor"][0]))
    e = 0.0
    for dst, src in pairs:
        d, s = st.slot(st.theta0, dst), st.slot(st.theta1, src)
        e = max(e, _ulps(st.slot(st.theta1, dst), p.tau * s + (1 - p.tau) * d, p.tau * s.abs() + (1 - p.tau) * d.abs()))
    errs["polyak"] = e
    return errs


def _alpha_errs(st, errs):
    p = st.p
    if not (st.sac and p._is_auto_alpha):
        if st.sac:      # a fixed temperature stays put
            assert torch.equal(st.alpha_state0, st.alpha_state1) and float(p._alpha_dev.item()) == st.alpha
        return errs
    la, m, v, t = st.alpha_state0.tolist()
    lp = st.w["logp"][:st.B]
    mean_lp, H = float(lp.mean()), p._target_entropy
    g = -(mean_lp + H)
    gs = float(lp.abs().mean()) + abs(H)                 # scale of g: the mean's own condition
    la1, m1, v1 = (float(z) for z in adam64(la, g, m, v, t + 1, p._alpha_lr))
    got = st.alpha_state1.tolist()
    assert got[3] == t + 1
    errs["alpha.log"] = abs(got[0] - la1) / p._alpha_lr          # in units of the step size
    errs["alpha.m"] = abs(got[1] - m1) / (0.1 * gs + 0.9 * abs(m))
    errs["alpha.v"] = abs(got[2] - v1) / (0.002 * gs * gs + v)
    errs["alpha.loss"] = abs(st.stats["loss/alpha_loss"] + la * (mean_lp + H)) / (abs(la) * gs)
    errs["alpha.value"] = abs(st.stats["loss/alpha_value"] - math.exp(la1)) / math.exp(la1)
    return errs


BOUNDS = [("eps", EPS_TOL), ("act", ACT_TOL), ("logp", LOGP_TOL), ("gpow", NSTEP_TOL), ("partial", NSTEP_TOL),
          ("target", TARGET_TOL), ("gq", GRAD_TOL), ("ga", GRAD_TOL), ("dq", DOUT_TOL), ("loss/", LOSS_TOL),
          ("adam", ULP_TOL), ("polyak", ULP_TOL), ("alpha", ALPHA_TOL), ("sigma", ACT_TOL)]


def _bound(k):
    for pre, tol in BOUNDS:
        if k.startswith(pre):
            return tol
    raise KeyError(k)


def _check(label, policy, buf, B, seed=1, edit=None):
    st = _Step(policy, buf, B, seed, edit)
    errs = {}
    for f in (_target_errs, _critic_errs, _actor_errs, _adam_errs, _alpha_errs):
        f(st, errs)
    worst = {}
    for k, v in errs.items():
        key = k if k.startswith("loss/") else k.split(".")[0].rstrip("0123456789")
        worst[key] = max(worst.get(key, (0.0, k)), (v, k))
    print(f"\n{label} B={B}: " + " ".join(f"{k}={v:.2e}" + (f"[{n}]" if n != k else "") + f"/{_bound(k):.0e}"
                                          for k, (v, n) in worst.items()))
    bad = {k: v for k, v in errs.items() if not v <= _bound(k)}
    assert not bad, bad
    return st


# ---- cases ---------------------------------------------------------------------------------------------------
def test_c4_configuration():
    """bench.py c4 verbatim: SafetyCarRun-v0, bounded SAC mean, 2x128, B = 256, gamma 0.97, n_step 2, auto alpha,
    lambda = 0.8 (rescaling 1/1.8)"""
    p = _policy("sac", "SafetyCarRun-v0", hidden=(128, 128), bounded=True, n_step=2, tau=0.05, gamma=0.97)
    buf = synthetic_ring(7, 2, 8, 128, "wrapped", seed=4)
    _check("c4", p, buf, 256)


WIDTHS = [(A, TASK_BY_A[A]) for A in (2, 3, 4, 6, 8)] + [(2, BUTTON)]


@pytest.mark.parametrize("A,task", WIDTHS, ids=[t for _, t in WIDTHS])
@pytest.mark.parametrize("algo,bounded,B,layout,n_step", [("sac", True, 256, "wrapped", 2), ("sac", False, 200, "mixed", 3),
                                                         ("ddpg", True, 256, "partial", 2)],
                         ids=["sac-bounded", "sac-unbounded", "ddpg"])
def test_action_widths(A, task, algo, bounded, B, layout, n_step):
    from fsrl_b200 import envs
    env = envs.make(task)
    D = env.observation_space.shape[0]
    assert env.action_space.shape[0] == A
    p = _policy(algo, env=env, bounded=bounded, n_step=n_step)
    buf = synthetic_ring(D, A, 8, 128, layout, seed=A + D)
    _check(f"{algo} {task} A={A} D={D} bounded={bounded} n_step={n_step} {layout}", p, buf, B)


@pytest.mark.parametrize("algo,B,n_step", [("sac", 2, 2), ("sac", 5000, 8), ("ddpg", 5000, 5)],
                         ids=["sac-B2", "sac-B5000-nstep8", "ddpg-B5000"])
def test_batch_sizes(algo, B, n_step):
    """B = 2, the least the C entry accepts, and 5000 rows, where the engine's wgrad splits the rows and adds the
    splits atomically"""
    p = _policy(algo, "SafetyHopperVelocityGymnasium-v1", bounded=True, n_step=n_step)
    buf = synthetic_ring(11, 3, 16, 512, "mixed", seed=B)
    _check(f"{algo} hopper n_step={n_step}", p, buf, B)


@pytest.mark.parametrize("bounded", [True, False])
def test_sigma_clamp_edges(bounded):
    """The sigma head at exactly 2.0 and -20.0 (the clamp's closed ends pass the gradient, as torch.clamp's does)
    and at 2.5 and -21 (outside: no gradient).  Zero weights make the raw value the bias, exactly."""
    p = _policy("sac", "SafetyDroneRun-v0", bounded=bounded)
    A = 4
    raw = torch.tensor([2.0, -20.0, 2.5, -21.0], device="cuda")

    def edit(policy, eng):
        s = policy._groups()["actor"][0]
        _, _, _, _, w3, b3, ex = s.offsets()
        policy.arena.theta[w3:b3].view(s.H, s.out)[:, A:] = 0.0
        policy.arena.theta[b3 + A:ex] = raw

    st = _check(f"sigma clamp bounded={bounded}", p, synthetic_ring(19, 4, 8, 128, "wrapped", seed=9), 256, edit=edit)
    a = st.g["actor"][0]
    got = _tensors(a, st.slot(st.grad, a), A)
    for name in ("w3.sigma", "b3.sigma"):
        g = got[name].reshape(-1, A)
        assert (g[:, :2] != 0).any(0).all(), name          # the boundaries pass a gradient ...
        assert (g[:, 2:] == 0).all(), name                 # ... outside the range nothing passes
        ref = st.actor_grad_ref[name].reshape(-1, A)
        assert (ref[:, 2:] == 0).all()


def test_tied_twin_critics():
    """Each stream's second Q network a copy of its first (weights and Adam moments): the device computes bit-equal
    q0 and q1, and each twin gets half the actor-loss gradient, as torch.minimum gives."""
    p = _policy("sac", "SafetyCarRun-v0", bounded=True)

    def edit(policy, eng):
        crit = policy._groups()["critics"]
        for i in range(2):
            s0, s1 = crit[2 * i], crit[2 * i + 1]
            for t in (policy.arena.theta, eng.adam_m, eng.adam_v):
                t[s1.offset:s1.offset + s1.size] = t[s0.offset:s0.offset + s0.size]

    st = _check("tied twins", p, synthetic_ring(7, 2, 8, 128, "wrapped", seed=5), 256, edit=edit)
    crit = st.g["critics"]
    for i in range(2):
        s0, s1 = crit[2 * i], crit[2 * i + 1]
        assert torch.equal(st.slot(st.grad, s0), st.slot(st.grad, s1))       # the tie is exact on the device
        d0, d1 = st.dout[id(s0)][:, 0], st.dout[id(s1)][:, 0]
        assert torch.equal(d0, d1) and (d0 != 0).all()


@pytest.mark.parametrize("algo,opt", [("sac", "no-lagrangian"), ("ddpg", "no-lagrangian"), ("sac", "fixed-alpha"),
                                      ("sac", "max-action-2"), ("sac", "max-action-2-unbounded"), ("ddpg", "max-action-2")])
def test_options(algo, opt):
    """use_lagrangian=False (rescaling 1, no cost term), a fixed alpha, and max_action = 2 through a user env with
    Box(-2, 2) actions"""
    kw, env, D, A = {}, None, 7, 2
    if opt == "no-lagrangian":
        kw["use_lagrangian"] = False
    elif opt == "fixed-alpha":
        kw.update(auto_alpha=False, alpha=0.2)
    else:
        D, A = 9, 3
        env = _BoxEnv(D, A, 2.0)
    bounded = not opt.endswith("unbounded")
    p = _policy(algo, "SafetyCarRun-v0" if env is None else None, env=env, bounded=bounded, **kw)
    assert p.actor._max == (2.0 if env is not None else 1.0)
    buf = synthetic_ring(D, A, 8, 128, "mixed", seed=11, max_action=p.actor._max)
    st = _check(f"{algo} {opt}", p, buf, 256)
    assert st.resc == (1.0 if opt == "no-lagrangian" else 1 / 1.8)


@pytest.mark.parametrize("B", [256, 600])
def test_chunk_boundary(B):
    """update_many(K, B, buf, chunk=c) with c < K against chunk=K and against K calls of update_many(1, ...), from
    the same np.random seed: critic_t / actor_t / noise_t carry across the C calls."""
    K, c = 5, 2
    runs = []
    for mode in ("chunked", "whole", "single"):
        p = _policy("sac", "SafetyCarRun-v0", bounded=True)
        buf = synthetic_ring(7, 2, 8, 128, "wrapped", seed=6)
        np.random.seed(21)
        if mode == "single":
            stats = []
            for _ in range(K):
                p.update_many(1, B, buf)
                stats.append(p.last_stats)
            stats = {k: np.concatenate([np.asarray(s[k]) for s in stats]) for k in stats[0]}
        else:
            p.update_many(K, B, buf, chunk=c if mode == "chunked" else K)
            stats = {k: np.asarray(v) for k, v in p.last_stats.items()}
        torch.cuda.synchronize()
        runs.append((p.arena.theta.cpu().numpy(), p._alpha_state.cpu().numpy(), stats,
                     (p._critic_t, p._actor_t, p._noise_t)))
    ref = runs[1]
    assert ref[3] == (K, K, K)
    for theta, alpha, stats, counters in (runs[0], runs[2]):
        assert counters == ref[3]
        if B <= 256:
            # the stat reductions add at most two block partials onto zero: the order cannot change a bit
            assert np.array_equal(theta, ref[0]) and np.array_equal(alpha, ref[1])
            for k in ref[2]:
                assert np.array_equal(stats[k], ref[2][k]), k
        else:
            # five blocks add their partials of mean logp atomically in any order; alpha, and through it the actor
            # steps after the first, may differ in the last bits
            ulp = np.spacing(np.abs(ref[0]).astype(np.float32) + np.float32(1e-3))
            print(f"\nchunk B={B}: max |theta - theta_whole| = {(np.abs(theta - ref[0]) / ulp).max():.1f} ulps (bound 64)")
            assert (np.abs(theta - ref[0]) <= 64 * ulp).all()
            np.testing.assert_allclose(alpha, ref[1], rtol=1e-5, atol=1e-7)
            for k in ref[2]:
                np.testing.assert_allclose(stats[k], ref[2][k], rtol=1e-5, atol=1e-7, err_msg=k)
