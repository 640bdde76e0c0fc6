"""Float64 restatement of one PPO-Lagrangian minibatch update (fsrl_b200/policy/ppo_lag.py, csrc/ppo.cu), split
into the stages the kernels compute: advantage moments, forward, the loss gradient at the head outputs, the
backward pass through layers 3 and 2, and the weight-gradient contractions.  Each stage takes its inputs as
arguments, so the device tests can feed it what the device left from the stage before, and the host test can
chain the stages and compare the result with the oracle's autograd (oracle/ppo.py).

A network is a dict of float64 tensors in the arena's layout: w1 [D][H], b1, w2 [H][H], b2, w3 [H][out], b3 and,
for the actor, ls (log sigma).  Every value comes with a magnitude scale: the same expression evaluated on the
absolute values of its terms, which bounds the rounding of any order of summation."""
import math
from dataclasses import dataclass

import torch

LOG_SQRT_2PI = 0.5 * math.log(2.0 * math.pi)
KEYS = ("w1", "b1", "w2", "b2", "w3", "b3", "ls")


@dataclass
class Opts:
    """the loss options of one update, as the kernels see them"""
    A: int
    C: int                       # critics: 1 (reward) or 2 (reward, cost)
    max_action: float = 1.0
    bounded: bool = True
    eps_clip: float = 0.2
    dual_clip: float = 0.0       # 0: off
    vf_coef: float = 0.25
    value_clip: bool = False
    norm_adv: bool = True
    use_saf: bool = True         # the lambda-weighted cost term is on (use_lagrangian with a cost critic)
    lag: float = 0.0
    resc: float = 1.0            # 1 / (lambda + 1) with rescaling, else 1


@dataclass
class Rows:
    """one minibatch in float64: act [B][A], lpo [B], adv / ret / values [C][B]"""
    act: torch.Tensor
    lpo: torch.Tensor
    adv: torch.Tensor
    ret: torch.Tensor
    values: torch.Tensor


def adv_stats(adv, norm_adv):
    """mean and 1 / std (unbiased) of every advantage column, or (0, 1) without normalisation"""
    C = adv.shape[0]
    if not norm_adv:
        return torch.zeros(C, dtype=adv.dtype, device=adv.device), torch.ones(C, dtype=adv.dtype, device=adv.device)
    return adv.mean(1), 1.0 / adv.std(1)


def forward(P, x, masks=None):
    """pre-activations z1, z2 and h1, h2, out; ReLU masks given (the device's) or taken from z"""
    z1 = x @ P["w1"] + P["b1"]
    h1 = z1 * masks[0] if masks is not None else torch.relu(z1)
    z2 = h1 @ P["w2"] + P["b2"]
    h2 = z2 * masks[1] if masks is not None else torch.relu(z2)
    return z1, z2, h1, h2, h2 @ P["w3"] + P["b3"]


def forward_mag(P, x, masks):
    """the forward pass on magnitudes: the scale of h1, h2 and out"""
    Q = {k: v.abs() for k, v in P.items()}
    h1 = (x.abs() @ Q["w1"] + Q["b1"]) * masks[0]
    h2 = (h1 @ Q["w2"] + Q["b2"]) * masks[1]
    return h1, h2, h2 @ Q["w3"] + Q["b3"]


def head(o, outs, ls, R, mean, rstd):
    """The loss of the minibatch at the head outputs outs = [actor [B][A], critic_i [B][1]...], evaluated like
    ppo_lag.py's policy_loss + critics_loss.  Returns
      douts  per net, d loss / d head: the actor's [B][2A] (d/dmu-head columns, then d/dlog sigma of each row),
             a critic's [B][1];
      dmags  the magnitude scale of every element of douts;
      stats  actor_rew, actor_safety, kl, vf_i, entropy, total (floats) and their scales under "s_" + key."""
    A, B = o.A, outs[0].shape[0]
    z = outs[0][:, :A].clone().requires_grad_(True)
    lsr = ls.view(1, -1).expand(B, A).clone().requires_grad_(True)
    vs = [q[:, 0].clone().requires_grad_(True) for q in outs[1:]]
    mu = o.max_action * torch.tanh(z) if o.bounded else z
    sg = lsr.exp()
    zz = (R.act - mu) / sg
    logp = (-0.5 * zz ** 2 - lsr - LOG_SQRT_2PI).sum(1)
    ratio = torch.exp(logp - R.lpo)
    ar = (R.adv[0] - mean[0]) * rstd[0]
    surr1, surr2 = ratio * ar, ratio.clamp(1.0 - o.eps_clip, 1.0 + o.eps_clip) * ar
    lower = torch.min(surr1, surr2)
    if o.dual_clip:
        lower = torch.where(ar < 0, torch.max(lower, o.dual_clip * ar), lower)
    rew = -lower.mean()
    saf = torch.zeros((), dtype=z.dtype, device=z.device)
    if o.use_saf:
        ac = (R.adv[1] - mean[1]) * rstd[1]
        saf = (ratio * ac * o.lag).mean()
    vf = []
    for i, v in enumerate(vs):
        ret = R.ret[i]
        if o.value_clip:
            vold = R.values[i]
            vc = vold + (v - vold).clamp(-o.eps_clip, o.eps_clip)
            vf.append(torch.max((ret - v) ** 2, (ret - vc) ** 2).mean())
        else:
            vf.append(((ret - v) ** 2).mean())
    total = o.resc * (rew + saf) + o.vf_coef * sum(vf)
    grads = torch.autograd.grad(total, [z, lsr] + vs)
    douts = [torch.cat([grads[0], grads[1]], 1)] + [g.view(-1, 1) for g in grads[2:]]
    with torch.no_grad():
        zz, ratio, mu, sg = zz.detach(), ratio.detach(), mu.detach(), sg.detach()
        s_lp = (0.5 * zz ** 2 + ls.abs().view(1, -1) + LOG_SQRT_2PI).sum(1) + R.lpo.abs()   # condition of the ratio
        ar_m = (R.adv[0].abs() + mean[0].abs()) * rstd[0].abs()
        ac_m = (R.adv[1].abs() + mean[1].abs()) * rstd[1].abs() if o.use_saf else torch.zeros_like(ar_m)
        rr = ratio * (1.0 + s_lp)
        ga = (o.resc * (ar_m * (1.0 + o.dual_clip) + ac_m * abs(o.lag)) * rr / B).view(-1, 1)
        mup = o.max_action * (1.0 + torch.tanh(z.detach()) ** 2) if o.bounded else torch.ones_like(mu)
        dmags = [torch.cat([ga * (R.act.abs() + mu.abs()) / sg ** 2 * mup, ga * (zz ** 2 + 1.0)], 1)]
        s_vf = []
        for i, v in enumerate(vs):
            m = v.detach().abs() + R.ret[i].abs() + (R.values[i].abs() if o.value_clip else 0.0)
            dmags.append((o.vf_coef * 4.0 * m / B).view(-1, 1))
            s_vf.append(float((m ** 2).mean()))
        stats = {"actor_rew": float(rew), "actor_safety": float(saf), "kl": float((R.lpo - logp.detach()).mean()),
                 "entropy": float((0.5 + LOG_SQRT_2PI + ls).sum()), "total": float(total)}
        s_rew = float((ar_m * rr * (1.0 + o.dual_clip)).mean())
        s_saf = float((ac_m * rr * abs(o.lag)).mean())
        stats.update({"s_actor_rew": s_rew, "s_actor_safety": s_saf, "s_kl": float(s_lp.mean()),
                      "s_entropy": float((0.5 + LOG_SQRT_2PI + ls.abs()).sum()),
                      "s_total": o.resc * (s_rew + s_saf) + o.vf_coef * sum(s_vf)})
        for i, v in enumerate(vf):
            stats["vf%d" % i], stats["s_vf%d" % i] = float(v), s_vf[i]
        stats["ratio"], stats["ar"] = ratio, ar.detach()
    return douts, dmags, stats


def backward_dz2(P, dout, nout, h2):
    """dz2 = (dout[:, :nout] W3^T) masked by h2 > 0, and its magnitude scale"""
    m = (h2 > 0).to(dout.dtype)
    return (dout[:, :nout] @ P["w3"].t()) * m, (dout[:, :nout].abs() @ P["w3"].abs().t()) * m


def backward_dz1(P, dz2, h1):
    """dz1 = (dz2 W2^T) masked by h1 > 0, and its magnitude scale"""
    m = (h1 > 0).to(dz2.dtype)
    return (dz2 @ P["w2"].t()) * m, (dz2.abs() @ P["w2"].abs().t()) * m


def wgrad(x, h1, h2, dz1, dz2, dout, out, n_extra):
    """every parameter group's gradient as the contractions of the saved activations; called on magnitudes it
    gives the scale of each element"""
    g = {"w1": x.t() @ dz1, "b1": dz1.sum(0), "w2": h1.t() @ dz2, "b2": dz2.sum(0),
         "w3": h2.t() @ dout[:, :out], "b3": dout[:, :out].sum(0)}
    if n_extra:
        g["ls"] = dout[:, out:out + n_extra].sum(0)
    return g


def wgrad_mag(x, h1, h2, dz1, dz2, dout, out, n_extra):
    return wgrad(x.abs(), h1.abs(), h2.abs(), dz1.abs(), dz2.abs(), dout.abs(), out, n_extra)


def gradients(o, nets, x, R, masks=None):
    """The whole float64 update gradient of one minibatch: stats, per net the weight gradients and their scales.
    Without masks every ReLU decides on its float64 pre-activation."""
    mean, rstd = adv_stats(R.adv, o.norm_adv)
    fw = [forward(P, x, masks[i] if masks is not None else None) for i, P in enumerate(nets)]
    outs = [f[4] for f in fw]
    douts, dmags, stats = head(o, outs, nets[0]["ls"], R, mean, rstd)
    grads, scales = [], []
    for i, P in enumerate(nets):
        _, _, h1, h2, _ = fw[i]
        nout = o.A if i == 0 else 1
        dz2, dz2m = backward_dz2(P, douts[i], nout, h2)
        dz1, dz1m = backward_dz1(P, dz2, h1)
        n_extra = o.A if i == 0 else 0
        grads.append(wgrad(x, h1, h2, dz1, dz2, douts[i], nout, n_extra))
        hm = forward_mag(P, x, ((h1 > 0).double(), (h2 > 0).double()))
        dz1mm = backward_dz1({"w2": P["w2"].abs()}, dz2m, h1)[0]
        scales.append(wgrad(x.abs(), hm[0], hm[1], dz1mm, dz2m, dmags[i], nout, n_extra))
    return stats, grads, scales
