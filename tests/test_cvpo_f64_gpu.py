"""CVPO gradient steps (fsrl_cvpo_steps) one step at a time against float64.  After ``update_many(1, B, buf)``
the device still holds what that step computed: the critic regression's gradient in the critic slots of
``arena.grad`` and the M-step's in the actor slot, the n-step / target work arrays in ``policy._w``, the particles,
their observation rows, the old distribution, the combined Q values and the weights in ``policy._cw``, the Q values
of the K*B particle rows in the critics' ``out`` scratch, the M-step forward at theta0 in the actor's scratch
(mstep_iter_num = 1), and both dual states.  Each stage is checked against its own float64 value, fed the device's
output of the stage before it, so that an error points at the kernel that made it:

  target     the n-step walk, the next action of the current actor (Philox stream 0) and the n-step target
  critic     d/dtheta of the critics' regression loss at theta0
  particles  mu_old / std_old of actor_old, the K particles (stream 1, row k*B + b) and their observation rows
  Q pass     the critics at theta1 over all K*B particle rows
  E-step     a float64 replay of every dual iteration from the pre-step state on the device's Q values: the
             combined Q with its cumulative lambda subtraction, the dual gradient, Adam and the clamp; then the
             weights from the device's combined Q and eta
  M-step     the actor's forward at theta0; at the device's output, the KL, MLE and entropy statistics, the M-step
             duals' Adam step and clip, and the head gradient by float64 autograd of the M-step loss; the actor's
             weight gradient backpropagated in float64 from the device's head gradient through its ReLU masks
  adam       both Adam steps and the Polyak update of critics_old; actor_old does not move

Errors are measured against each quantity's own condition, the sum of the magnitudes of its terms, never
against a result that a cancelling sum can make small."""
import math

import numpy as np
import pytest
import torch

from helpers import adam64, synthetic_ring
from test_cvpo_host import cvpo_noise
from test_offpolicy_f64_gpu import BUTTON, TASK_BY_A, _grad_errs, _mlp64, _nstep64, _rel, _tensors, _ulps

pytestmark = pytest.mark.gpu

LOG_SQRT_2PI = 0.5 * math.log(2.0 * math.pi)
DUAL_EPS = float(np.float32(np.finfo(np.float32).eps * 10))     # the floor of the E-step duals (cvpo.cu)
FLT_MIN = float(np.finfo(np.float32).tiny)
f32 = np.float32

# Bounds: about 10x the worst value observed over all cases on an H100 80GB HBM3 (700 W power limit), which is
# given in each comment; every case prints its errors.
NSTEP_TOL = 2e-15    # gamma^k and the discounted sums, float64 on both sides: 2.2e-16
EPS_TOL = 8e-6       # act_next, mu_old / std_old, particles: relative to the magnitudes of mu and sigma * eps: 7.3e-7
TARGET_TOL = 1e-5    # |target - ref| / (|partial| + gamma^k sum |terms| of Q'): 1.0e-6
FWD_TOL = 3e-5       # particle Q values and the M-step forward, relative to |h2| |W3| + |b3|: 2.9e-6 (H = 512)
GRAD_TOL = 5e-5      # per tensor |got - ref|max / max|ref| (a head bias: against sum_b |d loss / d out_b|): 4.6e-6
DOUT_TOL = 3e-6      # M-step head gradient relative to the magnitude of its terms: 2.9e-7
LOSS_TOL = 5e-6      # loss / KL / MLE / entropy statistics relative to the magnitude of their terms: 4.3e-7
COMB_TOL = 1e-6      # combined Q relative to |q_r| + sum |lambda q_c|: 0, the replay's fp32 rounding matches
DUAL_TOL = 2e-5      # duals in units of their step size, Adam moments relative to their scale: 1.6e-6
WEIGHT_TOL = 4e-6    # weights relative to p_k (1 + |x_k| + sum_j p_j |x_j|), x = (c - max c) / eta: 3.6e-7
ULP_TOL = 24.0       # Adam / Polyak results in fp32 ulps of their operands' scale: 2.4


def _policy(task=None, H=128, K=16, cond=True, bounded=True, double=False, est=1, seed=3):
    """cvpo_cfg's learner: gamma 0.97, n_step 2, tau 0.05, one M-step iteration"""
    from fsrl_b200 import envs
    from fsrl_b200.agent import CVPOAgent
    agent = CVPOAgent(envs.make(task), seed=seed, hidden_sizes=(H, H), sample_act_num=K, estep_iter_num=est,
                      mstep_iter_num=1, double_critic=double, conditioned_sigma=cond, unbounded=not bounded,
                      gamma=0.97, n_step=2, tau=0.05)
    return agent.policy


def _ring(p, seed):
    D, A = p.arena.slots[0].D, p._action_dim()
    return synthetic_ring(D, A, 8, 128, "wrapped", seed=seed, max_action=p.actor._max)


class _Step:
    """One checked gradient step: the device state before it, the call, and the device state after it."""

    def __init__(self, policy, buf, B, seed=1, edit=None, warm_B=None):
        p = self.p = policy
        self.B, self.K, self.A = B, p._sample_act_num, p._action_dim()
        self.g = p._groups()
        np.random.seed(seed + 1000)
        p.update_many(1, warm_B or B, buf)            # warm-up: Adam moments and duals away from their start
        eng = self.eng0 = p._eng
        if edit is not None:
            edit(p, eng)
            eng.sync_mirror(p.arena.slots)
        c = lambda t: t.detach().cpu().double().clone()
        np.random.seed(seed)
        self.idx_t = p.sample_batch_indices(buf, 1, B)[0]
        self.idx = self.idx_t.cpu().numpy().astype(np.int64)
        crit = self.g["critics"]
        # the critic phase's activation masks: the same forward launch the step makes, on the same inputs
        eng.forward(crit, eng.make_input(buf.obs, self.idx_t, buf.act, self.idx_t), B, save=True)
        self.crit_masks = [(c(eng.slot_view(s, "h1")[:B]) > 0, c(eng.slot_view(s, "h2")[:B]) > 0) for s in crit]
        ar = p.arena
        self.theta0, self.m0, self.v0 = c(ar.theta), c(eng.adam_m), c(eng.adam_v)
        self.es0, self.ms0 = c(p._estep_state), c(p._mstep_state)
        self.noise_t, self.critic_t, self.actor_t = p._noise_t, p._critic_t, p._actor_t
        np.random.seed(seed)
        p.update_many(1, B, buf)
        torch.cuda.synchronize()
        eng = p._eng                                  # a larger K*B than the warm-up's grows the engine
        self.stats = {k: float(np.asarray(v)[0]) for k, v in p.last_stats.items()}
        self.theta1, self.m1, self.v1, self.grad = c(ar.theta), c(eng.adam_m), c(eng.adam_v), c(ar.grad)
        self.es1, self.ms1 = c(p._estep_state), c(p._mstep_state)
        self.w = {k: c(v) for k, v in p._w.items()}
        self.cw = {k: c(v) for k, v in p._cw.items()}
        KB = self.K * B
        self.qout = [c(eng.slot_view(s, "out")[:KB, 0]) for s in crit]
        a = self.g["actor"][0]
        self.a_out, self.a_dout = c(eng.slot_view(a, "out")[:B]), c(eng.slot_view(a, "dout")[:B])
        self.a_masks = (c(eng.slot_view(a, "h1")[:B]) > 0, c(eng.slot_view(a, "h2")[:B]) > 0)
        self.buf = {k: getattr(buf, k).cpu().numpy() for k in ("obs", "obs_next", "act", "rew", "cost")}
        self.buf.update(term=buf.terminated.cpu().numpy().astype(bool), trunc=buf.truncated.cpu().numpy().astype(bool),
                        ptr=buf.ptr.cpu().numpy().astype(np.int64), cap=buf.cap)

    def slot(self, theta, s, grad=False):
        v = theta[s.offset:s.offset + s.size].clone()
        return v.requires_grad_(True) if grad else v


def _head(p, s, th, out, mag):
    """(mu, sigma) of a Gaussian actor slot from its float64 output, and the magnitudes of mu and sigma from the
    output's rounding scale mag"""
    A, act = p._action_dim(), p.actor
    z = out[:, :A]
    mu = act._max * torch.tanh(z) if not act._unbounded else z
    if act._c_sigma:
        raw = out[:, A:2 * A]
        sig = raw.clamp(-20.0, 2.0).exp()
    else:
        ex = s.offsets()[6] - s.offset
        sig = th[ex:ex + A].view(1, -1).exp().expand_as(mu)
    mmu = mu.abs() + act._max * mag[:, :A] if not act._unbounded else mag[:, :A]
    msig = sig * (1 + mag[:, A:2 * A]) if act._c_sigma else sig
    return mu, sig, mmu.detach(), msig.detach()


def _target_errs(st, errs):
    p, B, A, b = st.p, st.B, st.A, st.buf
    C, per = p.critics_num, (2 if p._twin else 1)
    term, gpow, part, vmask = _nstep64(b, st.idx, p._gamma, p._n_step)
    w = st.w
    assert np.array_equal(w["term_idx"][:B].numpy().astype(np.int64), term)
    assert np.array_equal(w["vmask"][:B].numpy(), vmask)
    errs["gpow"] = _rel(w["gpow"][:B].numpy(), gpow)
    errs["partial"] = float(np.abs(w["partial"][:2 * B].numpy().reshape(2, B)[:C] - part[:C]).max() / np.abs(part).max())
    s_next = torch.from_numpy(b["obs_next"][term]).double()
    a = st.g["actor"][0]
    th = st.slot(st.theta0, a)
    out, mag = _mlp64(th, a, s_next, cond=True)
    mu, sig, mmu, msig = _head(p, a, th, out, mag)
    eps = torch.from_numpy(cvpo_noise(p._upd_seed, B, A, st.noise_t, 0)).double()
    a_next = w["act_next"][:B]
    errs["act_next"] = float(((a_next - (mu + sig * eps)).abs() / (mmu + msig * eps.abs())).max())
    x = torch.cat([s_next, a_next], 1)
    tgt, scl = [], []
    for i in range(C):
        qc = [_mlp64(st.slot(st.theta0, s), s, x, cond=True) for s in st.g["critics_old"][per * i:per * i + per]]
        q = torch.minimum(*(o[:, 0] for o, _ in qc)) if per == 2 else qc[0][0][:, 0]
        mq = torch.stack([m[:, 0] for _, m in qc]).max(0).values
        tgt.append(q.numpy() * vmask * gpow + part[i])
        scl.append(np.abs(part[i]) + gpow * mq.numpy())
    got = w["target"][:C * B].numpy().reshape(C, B)
    errs["target"] = float((np.abs(got - np.stack(tgt)) / np.stack(scl)).max())
    st.target = got


def _critic_errs(st, errs):
    p, B, b = st.p, st.B, st.buf
    C, per = p.critics_num, (2 if p._twin else 1)
    x = torch.from_numpy(np.concatenate([b["obs"][st.idx], b["act"][st.idx]], 1)).double()
    tgt = torch.from_numpy(st.target)
    loss, li, lm, nets = 0.0, [], [], []
    for i in range(C):
        l_i, m_i = 0.0, 0.0
        for j in range(per):
            n = per * i + j
            s = st.g["critics"][n]
            th = st.slot(st.theta0, s, grad=True)
            q = _mlp64(th, s, x, st.crit_masks[n])
            q.retain_grad()
            nets.append((s, th, q))
            l_i = l_i + ((q[:, 0] - tgt[i]) ** 2).mean()
            m_i += float(((q[:, 0].detach().abs() + tgt[i].abs()) ** 2).mean())
        li.append(float(l_i))
        lm.append(m_i)
        loss = loss + l_i
    loss.backward()
    for n, (s, th, q) in enumerate(nets):
        _grad_errs(errs, f"gq{n}", s, st.slot(st.grad, s), th.grad, q.grad)
    for i in range(C):
        errs[f"loss/loss_q{i}"] = abs(st.stats[f"loss/loss_q{i}"] - li[i]) / lm[i]


def _particle_errs(st, errs):
    p, B, K, A = st.p, st.B, st.K, st.A
    obs = torch.from_numpy(st.buf["obs"][st.idx]).double()
    ao = st.g["actor_old"][0]
    th = st.slot(st.theta0, ao)
    out, mag = _mlp64(th, ao, obs, cond=True)
    mu, sig, mmu, msig = _head(p, ao, th, out, mag)
    mo, so = st.cw["mu_old"][:B], st.cw["std_old"][:B]
    errs["mu_old"] = float(((mo - mu).abs() / mmu).max())
    errs["std_old"] = float(((so - sig).abs() / msig).max())
    eps = torch.from_numpy(cvpo_noise(p._upd_seed, K * B, A, st.noise_t, 1)).double().view(K, B, A)
    parts = st.cw["particles"][:K * B].view(K, B, A)
    errs["particles"] = float(((parts - (mo + so * eps)).abs() / (mo.abs() + so * eps.abs())).max())
    assert np.array_equal(st.cw["part_idx"][:K * B].numpy().astype(np.int64), np.tile(st.idx, K))


def _qpass_errs(st, errs):
    B, K = st.B, st.K
    pidx = st.cw["part_idx"][:K * B].numpy().astype(np.int64)
    x = torch.cat([torch.from_numpy(st.buf["obs"][pidx]).double(), st.cw["particles"][:K * B]], 1)
    for n, s in enumerate(st.g["critics"]):
        q, mag = _mlp64(st.slot(st.theta1, s), s, x, cond=True)
        errs[f"qpass{n}"] = float(((st.qout[n] - q[:, 0]).abs() / mag[:, 0]).max())


def _estep_errs(st, errs):
    """the E-step replayed in float64 from the pre-step dual state on the device's Q values.  The combined Q is
    rounded to fp32 as the device does (c <- fl(c - fl(lambda q_c))), since a Q value's own fp32 rounding is
    |Q| * 2^-24, a large share of eta when |Q| / eta is large."""
    p, B, K = st.p, st.B, st.K
    C, per = p.critics_num, (2 if p._twin else 1)
    qmin = lambda i: (np.minimum(st.qout[2 * i].numpy(), st.qout[2 * i + 1].numpy()) if per == 2
                      else st.qout[i].numpy()).astype(np.float32)
    q0 = qmin(0)
    qc = qmin(1) if C > 1 else np.zeros_like(q0)
    e = st.es0.numpy().copy()
    dual, m, v, t = e[0:2].copy(), e[2:4].copy(), e[4:6].copy(), e[6]
    mscale, vscale = np.abs(m), v.copy()
    kl, thr, lr, logK = p._estep_kl, (p.qc_thres[0] if C > 1 else 0.0), p._estep_dual_lr, math.log(K)
    comb = q0.copy()
    cscale = np.abs(q0).astype(np.float64)
    for _ in range(p._estep_iter_num):
        eta, lam = dual[0], (dual[1] if C > 1 else 0.0)
        if C > 1:
            comb = (comb - (f32(lam) * qc).astype(np.float32)).astype(np.float32)
            cscale = cscale + abs(lam) * np.abs(qc)
        c = comb.astype(np.float64).reshape(K, B)
        cm = c.max(0)
        x = (c - cm) / eta
        ex = np.exp(x)
        se = ex.sum(0)
        pk = ex / se
        g = np.array([kl + np.mean(np.log(se) - (pk * x).sum(0)) - logK,
                      thr - np.mean((pk * qc.reshape(K, B)).sum(0))])
        gs = np.array([kl + np.mean(np.abs(np.log(se)) + (pk * np.abs(x)).sum(0)) + logK,
                       abs(thr) + np.mean((pk * np.abs(qc.reshape(K, B))).sum(0))])
        loss = eta * kl + np.mean(cm + eta * (np.log(se) - logK)) + (lam * thr if C > 1 else 0.0)
        lscale = eta * kl + np.mean(np.abs(cm) + eta * (np.abs(np.log(se)) + logK)) + (abs(lam * thr) if C > 1 else 0.0)
        t += 1
        for i in range(C):
            d1, m1, v1 = adam64(dual[i], g[i], m[i], v[i], t, lr)
            dual[i], m[i], v[i] = float(d1), float(m1), float(v1)
            mscale[i] = 0.9 * mscale[i] + 0.1 * gs[i]
            vscale[i] = 0.999 * vscale[i] + 0.001 * gs[i] ** 2
    dual = np.clip(dual, DUAL_EPS, p._estep_dual_max)
    got = st.es1.numpy()
    assert got[6] == t
    for i in range(C):
        errs[f"estep.dual{i}"] = abs(got[i] - dual[i]) / lr
        errs[f"estep.m{i}"] = abs(got[2 + i] - m[i]) / mscale[i]
        errs[f"estep.v{i}"] = abs(got[4 + i] - v[i]) / vscale[i]
        assert st.stats[f"estep/dual{i}"] == got[i]
        tg = st.target[i]
        errs[f"loss/val_q{i}"] = abs(st.stats[f"estep/val_q{i}"] - tg.mean()) / np.abs(tg).mean()
    errs["loss/estep_loss"] = abs(st.stats["loss/estep_loss"] - loss) / lscale
    # the weights' pass subtracts lambda q_c once more, with the clamped dual the device stored
    if C > 1:
        comb = (comb - (f32(got[1]) * qc).astype(np.float32)).astype(np.float32)
        cscale = cscale + abs(got[1]) * np.abs(qc)
    comb_d = st.cw["comb"][:K * B].numpy()
    errs["comb"] = float((np.abs(comb_d - comb) / np.maximum(cscale, FLT_MIN)).max())
    c = comb_d.reshape(K, B)
    x = (c - c.max(0)) / got[0]
    ex = np.exp(x)
    pk = ex / ex.sum(0)
    wd = st.cw["weights"][:K * B].numpy().reshape(K, B)
    wscale = pk * (1 + np.abs(x) + (pk * np.abs(x)).sum(0))
    errs["weights"] = float((np.maximum(np.abs(wd - pk) - FLT_MIN, 0) / np.maximum(wscale, FLT_MIN)).max())
    st.dual_grad = g


def _mstep_errs(st, errs):
    """the actor's forward at theta0 against float64; then the head's statistics, the duals' step and d loss / d head
    by float64 autograd at the device's output, and the weight gradient backpropagated in float64 from the device's
    d loss / d head"""
    p, B, K, A = st.p, st.B, st.K, st.A
    a = st.g["actor"][0]
    cond = p.actor._c_sigma
    obs = torch.from_numpy(st.buf["obs"][st.idx]).double()
    th = st.slot(st.theta0, a, grad=True)
    out64 = _mlp64(th, a, obs, st.a_masks)
    _, mag = _mlp64(st.slot(st.theta0, a), a, obs, st.a_masks, cond=True)
    W = a.out
    errs["fwd"] = float(((st.a_out[:, :W] - out64.detach()).abs() / mag).max())
    ex = a.offsets()[6] - a.offset
    raw = st.a_out[:, A:2 * A] if cond else st.theta0[a.offset + ex:a.offset + ex + A].view(1, -1).expand(B, A)
    hd = torch.cat([st.a_out[:, :A], raw], 1).requires_grad_(True)
    z, r = hd[:, :A], hd[:, A:]
    mu = p.actor._max * torch.tanh(z) if not p.actor._unbounded else z
    sig = r.clamp(-20.0, 2.0).exp() if cond else r.exp()
    mo, so = st.cw["mu_old"][:B], st.cw["std_old"][:B]
    parts = st.cw["particles"][:K * B].view(K, B, A)
    w = st.cw["weights"][:K * B].view(K, B)
    vo, var = (so ** 2).clamp_min(1e-6), (sig ** 2).clamp_min(1e-6)
    kl_mu = (0.5 * (mo - mu) ** 2 / vo).sum(-1).mean()
    kl_std = (0.5 * (torch.log(var / vo) + vo / var - 1)).sum(-1).mean()
    z1, z2 = (parts - mu) / so, (parts - mo) / sig
    lik = (-0.5 * z1 ** 2 - so.log() - 0.5 * z2 ** 2 - sig.log() - 2 * LOG_SQRT_2PI).sum(-1)
    mle = (w * lik).mean()
    ent = (1 + 2 * LOG_SQRT_2PI + so.log() + sig.log()).sum(-1).mean()
    with torch.no_grad():           # every square (u - v)^2 expanded into its terms: (|u| + |v|)^2
        amu, asig, apart = mu.abs(), sig.abs(), parts.abs()
        s_klmu = (0.5 * (mo.abs() + amu) ** 2 / vo).sum(-1).mean()
        s_klstd = (0.5 * ((var.log()).abs() + vo.log().abs() + vo / var + 1)).sum(-1).mean()
        s_lik = (0.5 * ((apart + amu) / so) ** 2 + so.log().abs() + 0.5 * ((apart + mo.abs()) / asig) ** 2
                 + asig.log().abs() + 2 * LOG_SQRT_2PI).sum(-1)
        s_mle = (w * s_lik).mean()
        s_ent = (1 + 2 * LOG_SQRT_2PI + so.log().abs() + asig.log().abs()).sum(-1).mean()
    S = st.stats
    thr = (p._mstep_kl_mu, p._mstep_kl_std)
    # the M-step duals' Adam step from the pre-step state on the device's KL statistics, then the clip of their uses
    e = st.ms0.numpy()
    t = e[6] + 1
    kls, kls_s = (S["mstep/mstep_kl_mu"], S["mstep/mstep_kl_std"]), (float(s_klmu), float(s_klstd))
    got = st.ms1.numpy()
    assert got[6] == t
    dual = []
    for i in range(2):
        d1, m1, v1 = (float(q) for q in adam64(e[i], thr[i] - kls[i], e[2 + i], e[4 + i], t, p._mstep_dual_lr))
        gs = thr[i] + kls_s[i]
        errs[f"mdual.dual{i}"] = abs(got[i] - d1) / p._mstep_dual_lr
        errs[f"mdual.m{i}"] = abs(got[2 + i] - m1) / (0.1 * gs + 0.9 * abs(e[2 + i]))
        errs[f"mdual.v{i}"] = abs(got[4 + i] - v1) / (0.002 * gs * gs + e[4 + i])
        dual.append(min(max(d1, 0.0), p._mstep_dual_max))
    for i, k in enumerate(("mstep/mstep_dual_mu", "mstep/mstep_dual_std")):
        errs[f"mdual.use{i}"] = abs(S[k] - dual[i]) / p._mstep_dual_lr
    dmu, dstd = S["mstep/mstep_dual_mu"], S["mstep/mstep_dual_std"]
    loss_kl = dmu * (kl_mu - thr[0]) + dstd * (kl_std - thr[1])
    s_kl = dmu * (s_klmu + thr[0]) + dstd * (s_klstd + thr[1])
    for k, ref, scl in (("mstep_kl_mu", kl_mu, s_klmu), ("mstep_kl_std", kl_std, s_klstd), ("entropy", ent, s_ent),
                        ("mstep_loss_mle", -mle, s_mle), ("mstep_loss_kl", loss_kl, s_kl),
                        ("mstep_loss_total", loss_kl - mle, s_kl + s_mle)):
        errs[f"loss/{k}"] = abs(S["mstep/" + k] - float(ref)) / max(float(scl), FLT_MIN)
    loss = -mle + dmu * kl_mu + dstd * kl_std
    (dref,) = torch.autograd.grad(loss, hd)
    # d loss / d head: every term by magnitude, through tanh' and the clamp gate / d sigma / d raw
    with torch.no_grad():
        wsum = w.sum(0).view(B, 1)
        n_mu = (w[..., None] * ((apart + amu) / so ** 2)).sum(0) / (K * B) + dmu * (amu + mo.abs()) / vo / B
        n_sig = ((w[..., None] * (apart + mo.abs()) ** 2).sum(0) / asig ** 3 + wsum / asig) / (K * B) \
            + dstd * (1 / var + vo / var ** 2) * asig / B
        tp = torch.tanh(z).abs()
        dmag = torch.cat([n_mu * (p.actor._max * (1 + tp ** 2) if not p.actor._unbounded else 1), n_sig * asig], 1)
    errs["dout"] = float((((st.a_dout[:, :2 * A] - dref).abs() - FLT_MIN).clamp_min(0) / dmag.clamp_min(FLT_MIN)).max())
    # the weight gradient: float64 backpropagation of the device's head gradient through the device's masks
    (gref,) = torch.autograd.grad(out64, th, grad_outputs=st.a_dout[:, :W])
    if cond:
        _grad_errs(errs, "ga", a, st.slot(st.grad, a), gref, st.a_dout[:, :W], A)
    else:
        gref = gref.clone()
        gref[ex:ex + A] = st.a_dout[:, A:2 * A].sum(0)
        _grad_errs(errs, "ga", a, st.slot(st.grad, a), gref, st.a_dout[:, :W])
        got_ls = st.slot(st.grad, a)[ex:ex + A]
        errs["ga.log_sigma"] = float(((got_ls - gref[ex:ex + A]).abs() / st.a_dout[:, A:2 * A].abs().sum(0)).max())
    st.dref = dref


def _adam_errs(st, errs):
    p = st.p
    for name, slots, lr, t in (("adam_c", st.g["critics"], p._critic_lr, st.critic_t + 1),
                               ("adam_a", st.g["actor"], p._actor_lr, st.actor_t + 1)):
        e = 0.0
        for s in slots:
            sl = slice(s.offset, s.offset + s.size)
            g = st.grad[sl]
            ref, m, v = adam64(st.theta0[sl], g, st.m0[sl], st.v0[sl], t, lr)
            e = max(e, _ulps(st.theta1[sl], ref, ref.abs() + lr), _ulps(st.m1[sl], m, st.m0[sl].abs() + g.abs()),
                    _ulps(st.v1[sl], v, st.v0[sl] + g * g))
        errs[name] = e
    e = 0.0
    for dst, src in zip(st.g["critics_old"], st.g["critics"]):
        d, s = st.slot(st.theta0, dst), st.slot(st.theta1, src)
        e = max(e, _ulps(st.slot(st.theta1, dst), p.tau * s + (1 - p.tau) * d, p.tau * s.abs() + (1 - p.tau) * d.abs()))
    errs["polyak"] = e
    ao = st.g["actor_old"][0]
    assert torch.equal(st.slot(st.theta1, ao), st.slot(st.theta0, ao))


BOUNDS = [("gpow", NSTEP_TOL), ("partial", NSTEP_TOL), ("act_next", EPS_TOL), ("target", TARGET_TOL),
          ("gq", GRAD_TOL), ("ga", GRAD_TOL), ("loss/", LOSS_TOL), ("mu_old", EPS_TOL), ("std_old", EPS_TOL),
          ("particles", EPS_TOL), ("qpass", FWD_TOL), ("estep", DUAL_TOL), ("mdual", DUAL_TOL), ("comb", COMB_TOL),
          ("weights", WEIGHT_TOL), ("fwd", FWD_TOL), ("dout", DOUT_TOL), ("adam", ULP_TOL), ("polyak", ULP_TOL)]


def _bound(k):
    for pre, tol in BOUNDS:
        if k.startswith(pre):
            return tol
    raise KeyError(k)


def _check(label, policy, buf, B, seed=1, edit=None, warm_B=None):
    st = _Step(policy, buf, B, seed, edit, warm_B)
    errs = {}
    for f in (_target_errs, _critic_errs, _particle_errs, _qpass_errs, _estep_errs, _mstep_errs, _adam_errs):
        f(st, errs)
    worst = {}
    for k, v in errs.items():
        key = k if k.startswith("loss/") else k.split(".")[0].rstrip("0123456789")
        worst[key] = max(worst.get(key, (0.0, k)), (v, k))
    print(f"\n{label} B={B} K={st.K}: " + " ".join(f"{k}={v:.2e}" + (f"[{n}]" if n != k else "") + f"/{_bound(k):.0e}"
                                                  for k, (v, n) in worst.items()))
    bad = {k: v for k, v in errs.items() if not v <= _bound(k)}
    assert not bad, bad
    return st


# ---- cases ---------------------------------------------------------------------------------------------------
def test_cvpo_cfg_defaults():
    """cvpo_cfg: SafetyCarCircle-v0, 2x128, B = 256, K = 16, conditioned sigma, bounded mean, single critics"""
    p = _policy("SafetyCarCircle-v0")
    _check("cvpo_cfg", p, _ring(p, 4), 256)


@pytest.mark.parametrize("H", [64, 256, 512])
def test_hidden_widths(H):
    """the engine's other hidden widths (cvpo_cfg's 128 is the case above)"""
    p = _policy("SafetyCarCircle-v0", H=H)
    _check(f"H={H}", p, _ring(p, H), 256)


WIDTHS = [  # A, task, conditioned sigma, bounded mean, double critics
    (2, TASK_BY_A[2], True, True, False), (3, TASK_BY_A[3], False, False, True), (4, TASK_BY_A[4], True, False, True),
    (6, TASK_BY_A[6], False, True, False), (8, TASK_BY_A[8], True, True, True), (2, BUTTON, False, False, False)]


@pytest.mark.parametrize("A,task,cond,bounded,double", WIDTHS, ids=[f"{t}-A{a}" for a, t, *_ in WIDTHS])
def test_action_widths(A, task, cond, bounded, double):
    p = _policy(task, H=64, cond=cond, bounded=bounded, double=double)
    assert p._action_dim() == A
    _check(f"{task} A={A} D={p.arena.slots[0].D} cond={cond} bounded={bounded} double={double}", p, _ring(p, A), 256)


@pytest.mark.parametrize("B,K", [(2, 16), (300, 16), (600, 16), (256, 1), (256, 64)],
                         ids=["B2", "B300", "B600", "K1", "K64"])
def test_batch_shapes(B, K):
    """B = 2, the least the C entry accepts; B = 300 and 600, past one and two strides of the 256-thread E- and
    M-step CTAs; one particle; and K = 64 at B = 256, 16384 rows in the Q pass"""
    p = _policy("SafetyHopperVelocityGymnasium-v1", H=64, K=K, double=B == 600)
    _check(f"hopper double={p._twin}", p, _ring(p, B + K), B)


def test_estep_lambda():
    """three E-step iterations from lambda = 0.5 with non-zero moments: the combined Q loses lambda q_c in every
    iteration and once more for the weights"""
    p = _policy("SafetyCarCircle-v0", H=64, est=3, double=True)

    def edit(policy, eng):
        policy._estep_state[:6] = torch.tensor([0.8, 0.5, 0.05, -0.03, 2e-3, 1e-3], device="cuda")

    st = _check("lambda", p, _ring(p, 5), 256, edit=edit)
    assert np.abs(st.qout[2].numpy()).mean() > 1e-2          # the cost stream's Q values are not zero


def _set_sigma(policy, slot_name, raw):
    """zero sigma-head weights and the bias raw: the slot's raw sigma is exactly raw on every row"""
    s = policy._groups()[slot_name][0]
    A = policy._action_dim()
    _, _, _, _, w3, b3, ex = s.offsets()
    th = policy.arena.theta
    th[w3:b3].view(s.H, s.out)[:, A:] = 0.0
    th[b3 + A:ex] = torch.as_tensor(raw, dtype=torch.float32, device="cuda")


@pytest.mark.parametrize("case", ["eta-floor", "eta-max", "mstep-duals"])
def test_dual_clamps(case):
    p = _policy("SafetyCarCircle-v0", H=64)

    def edit(policy, eng):
        es, ms = policy._estep_state, policy._mstep_state
        if case == "eta-floor":          # particles of sigma e^-20: a tiny Q spread drives eta down onto the floor
            es[0], es[2], es[4] = DUAL_EPS, 2e-3, 4e-6
            _set_sigma(policy, "actor_old", -20.0)
        elif case == "eta-max":
            es[0] = 25.0
        else:
            ms[0], ms[1] = -0.3, 0.9

    st = _check(f"clamp {case}", p, _ring(p, 6), 256, edit=edit)
    got = st.es1.numpy()
    if case == "eta-floor":
        assert got[0] == DUAL_EPS
    elif case == "eta-max":
        assert got[0] == p._estep_dual_max
    else:
        assert st.stats["mstep/mstep_dual_mu"] == 0.0 and st.stats["mstep/mstep_dual_std"] == p._mstep_dual_max


def test_large_q_over_eta():
    """reward Q values of about 30 +- 1e-2 (head bias +30, particles of sigma e^-5) at eta = 1e-3: without the
    shift by each row's largest Q, the eta gradient and the weights lose |Q| / eta * 2^-24"""
    p = _policy("SafetyCarCircle-v0", H=64)

    def edit(policy, eng):
        s = policy._groups()["critics"][0]
        b3 = s.offsets()[5]
        policy.arena.theta[b3] += 30.0
        policy._estep_state[0] = 1e-3
        _set_sigma(policy, "actor_old", -5.0)

    st = _check("large Q / eta", p, _ring(p, 7), 256, edit=edit)
    q = st.qout[0].numpy().reshape(st.K, st.B)
    assert abs(q.mean() - 30) < 3 and np.median(q.max(0) - q.min(0)) < 0.1
    print(f"Q {q.mean():.2f}, median row spread {np.median(q.max(0) - q.min(0)):.2e}")


@pytest.mark.parametrize("case", ["sigma-ends-bounded", "sigma-ends-unbounded", "old-sigma-floor"])
def test_mstep_gates(case):
    """raw sigma at exactly 2.0 and -20.0 (the clamp's closed ends pass the gradient, as torch.clamp's does) and at
    2.5 and -21 (no gradient); an old sigma of e^-8, whose variance is under the KL's 1e-6 floor"""
    bounded = case != "sigma-ends-unbounded"
    p = _policy("SafetyDroneRun-v0", H=64, bounded=bounded)
    A = 4
    raw = [2.0, -20.0, 2.5, -21.0]

    def edit(policy, eng):
        if case == "old-sigma-floor":
            _set_sigma(policy, "actor_old", -8.0)
        else:
            _set_sigma(policy, "actor", raw)

    st = _check(case, p, _ring(p, 8), 256, edit=edit)
    if case == "old-sigma-floor":
        assert (st.cw["std_old"][:st.B] ** 2 < 1e-6).all()
        return
    d = st.a_dout[:, A:2 * A]
    assert (d[:, :2] != 0).all() and (d[:, 2:] == 0).all()
    assert (st.dref[:, A + 2:] == 0).all()
    a = st.g["actor"][0]
    got = _tensors(a, st.slot(st.grad, a), A)
    for name in ("w3.sigma", "b3.sigma"):
        g = got[name].reshape(-1, A)
        assert (g[:, :2] != 0).any(0).all() and (g[:, 2:] == 0).all(), name


def test_engine_growth():
    """update_many at B = 64 and then at B = 256 (K = 16): the engine grows from 1024 to 4096 rows, and the second
    step's Adam continues the moments of the first"""
    p = _policy("SafetyCarCircle-v0", H=64)
    st = _check("growth", p, _ring(p, 9), 256, warm_B=64)
    assert st.eng0.bmax == 1024 and p._eng.bmax == 4096
    assert st.m0.abs().max() > 0
