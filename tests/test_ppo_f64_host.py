"""The float64 stage functions of tests/ppo64.py (the reference of tests/test_ppo_f64_gpu.py) chained into one
minibatch update agree with the oracle's autograd run in float64 (oracle/ppo.py learn(..., grads_out=...), pinned on
the reference implementation by tests/test_oracle_golden.py): the head gradient, backward pass and weight
contractions give every parameter group's gradient, and the head gives the logged statistics, for every loss
option the device tests use.  Runs on the CPU."""
import copy

import numpy as np
import pytest
import torch

import ppo64

TOL = 1e-12      # float64 against float64: both sides sum the same terms in different orders


def _nets(D, A, H, max_action, bounded, C, seed):
    from oracle import nets as onets
    torch.manual_seed(seed)
    actor = onets.GaussActor(D, A, [H, H], max_action=max_action, unbounded=not bounded).double()
    critics = [onets.ValueNet(D, [H, H]).double() for _ in range(C)]
    with torch.no_grad():
        actor.sigma_param.copy_(-0.5 + 0.3 * torch.randn(A, 1, dtype=torch.float64))
        for m in [actor] + critics:
            for lin in m.modules():
                if isinstance(lin, torch.nn.Linear):
                    lin.bias.copy_(0.1 * torch.randn_like(lin.bias))
    return actor, critics


def _as_ppo64(m):
    """an oracle module's weights in the arena layout"""
    L = m.body.layers
    last = m.mu if hasattr(m, "mu") else m.last
    P = {"w1": L[0].weight.detach().t(), "b1": L[0].bias.detach(), "w2": L[1].weight.detach().t(),
         "b2": L[1].bias.detach(), "w3": last.weight.detach().t(), "b3": last.bias.detach()}
    if hasattr(m, "sigma_param"):
        P["ls"] = m.sigma_param.detach().view(-1)
    return P


def _oracle_grads(grads, m):
    """the oracle's gradients of one module (parameters() order), in the arena layout"""
    named = [n for n, _ in m.named_parameters()]
    g = dict(zip(named, grads))
    last = "mu" if hasattr(m, "mu") else "last"
    out = {"w1": g["body.layers.0.weight"].t(), "b1": g["body.layers.0.bias"], "w2": g["body.layers.1.weight"].t(),
           "b2": g["body.layers.1.bias"], "w3": g[last + ".weight"].t(), "b3": g[last + ".bias"]}
    if "sigma_param" in g:
        out["ls"] = g["sigma_param"].view(-1)
    return out


# name: (A, C, options of oracle.ppo.learn / ppo64.Opts)
CASES = {
    "default": (2, 2, dict(lag=0.7)),
    "lag0": (2, 2, dict(lag=0.0)),
    "max2.5": (3, 2, dict(lag=0.4, max_action=2.5)),
    "unbounded": (2, 2, dict(lag=0.4, bounded=False)),
    "one-critic": (2, 1, dict(lag=0.0)),
    "no-lagrangian": (2, 2, dict(lag=0.6, use_lagrangian=False)),
    "no-rescaling": (2, 2, dict(lag=0.6, rescaling=False)),
    "no-adv-norm": (2, 2, dict(lag=0.6, norm_adv=False)),
    "vclip-dclip": (3, 2, dict(lag=0.6, value_clip=True, dual_clip=1.5)),
    "A1": (1, 2, dict(lag=0.3)),
    "A8": (8, 2, dict(lag=0.3, bounded=False)),
}


@pytest.mark.parametrize("name", list(CASES))
def test_stage_functions_match_oracle_autograd(name):
    from oracle import ppo as oppo
    A, C, kw = CASES[name]
    kw = dict(kw)
    lag = kw.pop("lag")
    max_action, bounded = kw.pop("max_action", 1.0), kw.pop("bounded", True)
    use_lag, resc_on = kw.get("use_lagrangian", True), kw.get("rescaling", True)
    D, H, n = 7, 32, 48
    actor, critics = _nets(D, A, H, max_action, bounded, C, seed=len(name))
    g = np.random.default_rng(len(name))
    obs = g.standard_normal((n, D))
    with torch.no_grad():
        mu, sg = actor(torch.from_numpy(obs))
        v = torch.stack([c(torch.from_numpy(obs)).flatten() for c in critics], 1).numpy()
    # ratios spread over both sides of the clip range and of the dual clip, value targets away from the critics
    act = (mu + sg * torch.from_numpy(g.standard_normal((n, A)))).numpy()
    dist = torch.distributions.Independent(torch.distributions.Normal(mu, sg), 1)
    logp = dist.log_prob(torch.from_numpy(act)).numpy()
    logp_old = logp - np.log(g.uniform(0.4, 2.2, n))
    values = v + g.choice([-1.0, 1.0], (n, C)) * g.uniform(0.0, 0.6, (n, C))
    batch = dict(obs=obs, act=act, logp_old=logp_old, advs=g.standard_normal((n, C)) * 2.0 + 0.3,
                 rets=v + g.standard_normal((n, C)), values=values)
    grads = []
    a, c = copy.deepcopy(actor), copy.deepcopy(critics)
    np.random.seed(3)
    st = oppo.learn(a, c, torch.optim.Adam([p for m in [a] + c for p in m.parameters()], lr=1e-3), batch, n, 1, lag,
                    max_grad_norm=None, target_kl=1e9, grads_out=grads, **kw)[0]
    resc = 1.0 / (lag + 1.0) if (resc_on and use_lag) else 1.0
    o = ppo64.Opts(A=A, C=C, max_action=max_action, bounded=bounded, dual_clip=kw.get("dual_clip") or 0.0,
                   value_clip=kw.get("value_clip", False), norm_adv=kw.get("norm_adv", True),
                   use_saf=use_lag and C > 1, lag=lag, resc=resc)
    t = lambda k: torch.from_numpy(np.ascontiguousarray(batch[k]))
    R = ppo64.Rows(act=t("act"), lpo=t("logp_old"), adv=t("advs").t(), ret=t("rets").t(), values=t("values").t())
    nets = [_as_ppo64(m) for m in [actor] + critics]
    stats, gref, gscale = ppo64.gradients(o, nets, t("obs"), R)
    errs = {}
    k = 0
    for i, m in enumerate([actor] + critics):
        n_par = len(list(m.parameters()))
        want = _oracle_grads(grads[k:k + n_par], m)
        k += n_par
        for key, w in want.items():
            errs["net%d.%s" % (i, key)] = float(((gref[i][key] - w).abs() / gscale[i][key].clamp(min=1e-300)).max())
    for key in ["actor_rew", "kl", "entropy", "total"] + ["vf%d" % i for i in range(C)] + \
               (["actor_safety"] if o.use_saf else []):
        errs[key] = abs(stats[key] - st["loss/" + key]) / max(stats["s_" + key], 1e-300)
    ratio = stats["ratio"].numpy()
    print("\n%s: ratios below / inside / above the clip range: %d / %d / %d; worst %s = %.1e"
          % (name, (ratio < 0.8).sum(), ((ratio >= 0.8) & (ratio <= 1.2)).sum(), (ratio > 1.2).sum(),
             max(errs, key=errs.get), max(errs.values())))
    assert min((ratio < 0.8).sum(), (ratio > 1.2).sum(), ((ratio > 0.8) & (ratio < 1.2)).sum()) >= 5
    bad = {k: v for k, v in errs.items() if not v <= TOL}
    assert not bad, bad
