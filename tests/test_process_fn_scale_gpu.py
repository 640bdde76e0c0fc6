"""process_fn at the benchmarked collect sizes against float64: c2 (PPO-Lagrangian, SafetyCarCircle-v0, 2048 envs x 300
steps, 2x256), c3 (CPO, SafetyPointGoal1Gymnasium-v0, 2048 envs x 1000 steps, 2x128) and c5 (PPO-Lagrangian,
SafetyAntCircle-v0, 1024 envs x 500 steps, 2x512), each built by bench.py's own builder and collected once.

Checked in stages, so that a failure names its stage:

1. values: batch.v (and the device's V(obs_next)) against a float64 twin of the critics carrying the same weights, run
   with torch float64 on the GPU.  The fp32 torch twin's own error is printed beside the device's.  Bound: |dv| <=
   V_RTOL |v64| + V_ATOL.  Observed on an H100 80GB HBM3 (700 W), max |dv| device / fp32 twin: c2 3.9e-7 / 6.8e-8
   (max |v| 0.22), c3 1.8e-6 / 5.6e-7 (max |v| 1.19), c5 7.9e-7 / 9.2e-8 (max |v| 0.27); the device's 3xTF32
   products sit 3 to 9 times above an fp32 FMA chain, and a wrong term shows up orders of magnitude above the bound.
2. scan and glue, exact: oracle.returns.dual_gae on batch.v, the device's V(obs_next) from net_forward over every
   obs_next row, and the buffer's flags including unfinished_index().  fsrl_mlp_forward computes a row by the same
   operation sequence wherever the row sits and whether or not it is gathered, so that V(obs_next) is bit-identical to
   the one compute_gae_returns assembles from V(obs[i+1]) and its gathered end-row pass.  adv / ret must then meet the
   GAE contract: <= 1 f32 ulp, bit-equal on >= 99.99 %.  This checks the de-duplicated value pass and the end-flag glue.
3. end to end, against an all-float64 pipeline (f64 values -> f64 GAE): |dadv| <= (1 + gamma) max|dv| / (1 - gamma
   lambda) + 1 ulp, with max|dv| measured in stage 1 (over V(obs) and V(obs_next)); |dret| <= that + max|dv| + 1 ulp.
4. c3 only: the standardised advantages (fsrl_standardize, one CTA over 2 048 000 rows) against float64 (x - mean) /
   std(ddof=1) of the advantages before standardisation, within STD_ULPS f32 ulps of max(1, |y64|) (observed 1.43
   and 0.80 ulp; the f32 mean contributes |mean| / (2 std) ulp, the f32 subtraction, rstd and product about 1.5 ulp
   of |y| together); batch.mean_old against the float64 actor twin (same bound as the values; observed 1.1e-6 device,
   4.6e-7 fp32 twin).

Two more index sets at c2 size: unfinished tails (the last stored row of every third env turned into a running
episode's, the way the reference's ring looks after a partial collect), and a caller-chosen shuffled subset of the
indices whose row order breaks the obs_next / next-obs adjacency at every block border."""
import copy

import numpy as np
import pytest
import torch

from helpers import oracle_nets

pytestmark = pytest.mark.gpu

TILE = 2048                  # rows per GAE tile (csrc/gae.cu)
V_RTOL, V_ATOL = 2e-5, 2e-6
STD_ULPS = 4
ULP1 = 2.0 ** -23            # f32 spacing at 1
CHUNK = 1 << 18


def _ulp_diff(a, b):
    ai = a.view(np.int32).astype(np.int64)
    bi = b.view(np.int32).astype(np.int64)
    ai = np.where(ai < 0, np.int64(-2**31) - ai, ai)
    bi = np.where(bi < 0, np.int64(-2**31) - bi, bi)
    return np.abs(ai - bi)


def _collect(config):
    """bench.py's build() for `config` (task, envs, widths, agent and seeds as benchmarked) and one collect."""
    import bench
    cfg = bench.CONFIGS[config]
    agent, _, col, buf, T = bench.build(cfg, "cuda:0", 0)
    col.collect(n_episode=cfg["envs"])
    assert len(buf) == cfg["envs"] * T
    return agent.policy, buf, cfg


@pytest.fixture(scope="module")
def c2():
    return _collect("c2")


@torch.no_grad()
def _eval(net, x, dtype, head=lambda y: y):
    out = []
    for s in range(0, x.shape[0], CHUNK):
        out.append(head(net(x[s:s + CHUNK].to(dtype))))
    return torch.cat(out)


def _twins(policy, hidden):
    actor, critics = oracle_nets(policy, hidden)
    dev = torch.device("cuda", 0)
    c32 = [copy.deepcopy(c).to(dev) for c in critics]
    c64 = [copy.deepcopy(c).double().to(dev) for c in critics]
    return actor, c32, c64


def _process(policy, buf, idx):
    """policy.process_fn, keeping a copy of the advantages as they leave the GAE when the policy standardises them."""
    pre = []
    std = getattr(policy, "_standardize", None)
    if std is not None:
        def spy(x, n):
            pre.append(x[:n].clone())
            std(x, n)
        policy._standardize = spy
    try:
        batch = policy.process_fn(None, buf, idx)
    finally:
        if std is not None:
            del policy._standardize
    torch.cuda.synchronize()
    adv_gae = torch.stack(pre) if pre else batch.adv
    return batch, adv_gae


def _gae64(v, vn, rew, term, end, gamma, lam):
    """base_policy.py's gae_return in float64 throughout (values included)."""
    delta = (rew + np.where(term, 0.0, vn) * gamma) - v
    disc = np.where(end, 0.0, gamma * lam).tolist()
    d = delta.tolist()
    out = [0.0] * len(d)
    g = 0.0
    for i in range(len(d) - 1, -1, -1):
        g = d[i] + disc[i] * g
        out[i] = g
    return np.asarray(out)


def _check_process_fn(name, policy, buf, idx, hidden):
    from oracle import returns
    batch, adv_gae = _process(policy, buf, idx)
    C, gamma, lam = policy.critics_num, float(policy._gamma), float(policy._lambda)
    n = int(idx.numel())
    assert batch.n == n
    obs, obs_next = buf.obs[idx].contiguous(), buf.obs_next[idx].contiguous()
    _, c32, c64 = _twins(policy, hidden)

    # ---- 1. values ----------------------------------------------------------------------------------------------
    vn_dev = torch.stack([policy.net_forward(1 + i, obs_next).flatten() for i in range(C)])
    dv = []
    for i in range(C):
        for what, x, got in (("V(obs)", obs, batch.v[i]), ("V(obs_next)", obs_next, vn_dev[i])):
            w64 = _eval(c64[i], x, torch.float64).flatten()
            w32 = _eval(c32[i], x, torch.float32).flatten().double()
            e_dev, e_32 = (got.double() - w64).abs(), (w32 - w64).abs()
            bad = e_dev > V_RTOL * w64.abs() + V_ATOL
            print("\n%s critic %d %-11s max |v - v64|: device %.3e, fp32 twin %.3e (max |v64| %.3g, n %d)"
                  % (name, i, what, e_dev.max().item(), e_32.max().item(), w64.abs().max().item(), n), end="")
            assert not bool(bad.any()), ("stage 1: values", name, i, what, e_dev.max().item(), int(bad.sum()))
            dv.append(e_dev.max().item())
    dv_max = [max(dv[2 * i], dv[2 * i + 1]) for i in range(C)]

    # ---- 2. scan and glue against the oracle, on the device's own values ------------------------------------
    g = lambda t: t.detach().cpu().numpy()
    ih = g(idx)
    term, trunc = g(buf.terminated)[ih].astype(bool), g(buf.truncated)[ih].astype(bool)
    unf = np.isin(ih, g(buf.unfinished_index()))
    rew, cost = g(buf.rew)[ih], g(buf.cost)[ih]
    v, vn = g(batch.v), g(vn_dev)
    _, rets, advs = returns.dual_gae(v, vn, rew, cost, term, trunc, unf, gamma, lam)
    adv, ret = g(adv_gae), g(batch.ret)
    for i in range(C):
        ua, ur = _ulp_diff(adv[i], advs[:, i]), _ulp_diff(ret[i], rets[:, i])
        print("\n%s critic %d scan: max ulp adv %d ret %d, bit-equal adv %.6f ret %.6f"
              % (name, i, ua.max(), ur.max(), (ua == 0).mean(), (ur == 0).mean()), end="")
        assert ua.max() <= 1 and ur.max() <= 1, ("stage 2: scan", name, i, ua.max(), ur.max())
        assert (ua == 0).mean() >= 0.9999 and (ur == 0).mean() >= 0.9999, ("stage 2: scan", name, i)

    # ---- 3. end to end against f64 values -> f64 GAE ------------------------------------------------------------
    end = term | trunc | unf
    m = [rew.astype(np.float64), cost.astype(np.float64)]
    for i in range(C):
        v64 = g(_eval(c64[i], obs, torch.float64).flatten())
        vn64 = g(_eval(c64[i], obs_next, torch.float64).flatten())
        a64 = _gae64(v64, vn64, m[i], term, end, gamma, lam)
        r64 = a64 + v64
        prop = (1.0 + gamma) * dv_max[i] / (1.0 - gamma * lam)
        ea, er = np.abs(adv[i] - a64), np.abs(ret[i] - r64)
        ba = prop + np.spacing(np.abs(a64).astype(np.float32)).astype(np.float64)
        br = prop + dv_max[i] + np.spacing(np.abs(r64).astype(np.float32)).astype(np.float64)
        print("\n%s critic %d end to end: max |adv - adv64| %.3e (propagated bound %.3e), max |ret - ret64| %.3e"
              % (name, i, ea.max(), prop, er.max()), end="")
        assert (ea <= ba).all(), ("stage 3: adv", name, i, ea.max(), prop)
        assert (er <= br).all(), ("stage 3: ret", name, i, er.max(), prop)
    return batch, adv_gae, obs


def _check_standardize_and_mean_old(name, policy, batch, adv_gae, obs, hidden):
    for i in range(policy.critics_num):
        x64 = adv_gae[i].double()
        y64 = (x64 - x64.mean()) / x64.std(unbiased=True)
        err = (batch.adv[i].double() - y64).abs() / y64.abs().clamp(min=1.0) / ULP1
        print("\n%s critic %d standardised advantages: max error %.2f ulp of max(1, |y64|) (|mean| / std %.3g)"
              % (name, i, err.max().item(), (x64.mean().abs() / x64.std()).item()), end="")
        assert err.max().item() <= STD_ULPS, ("stage 4: standardize", name, i, err.max().item())
    actor, _, _ = _twins(policy, hidden)
    dev = torch.device("cuda", 0)
    a64, a32 = copy.deepcopy(actor).double().to(dev), copy.deepcopy(actor).to(dev)
    mu = lambda out: out[0]
    m64 = _eval(a64, obs, torch.float64, mu)
    e_dev = (batch.mean_old.double() - m64).abs()
    e_32 = (_eval(a32, obs, torch.float32, mu).double() - m64).abs()
    print("\n%s mean_old max |mu - mu64|: device %.3e, fp32 twin %.3e" % (name, e_dev.max().item(), e_32.max().item()),
          end="")
    assert not bool((e_dev > V_RTOL * m64.abs() + V_ATOL).any()), ("stage 4: mean_old", name, e_dev.max().item())


def test_c2_process_fn(c2):
    policy, buf, cfg = c2
    _check_process_fn("c2", policy, buf, buf.sample_indices(0), cfg["hidden"])


def test_c3_process_fn():
    """CPO at c3: 2 048 000 rows, 1000 GAE tiles (several per CTA), advantages standardised by fsrl_standardize."""
    policy, buf, cfg = _collect("c3")
    idx = buf.sample_indices(0)
    n = int(idx.numel())
    W = 3 * torch.cuda.get_device_properties(0).multi_processor_count
    assert n == 2048 * 1000 and -(-n // TILE) > W
    assert policy._norm_adv
    batch, adv_gae, obs = _check_process_fn("c3", policy, buf, idx, cfg["hidden"])
    _check_standardize_and_mean_old("c3", policy, batch, adv_gae, obs, cfg["hidden"])


def test_c5_process_fn():
    policy, buf, cfg = _collect("c5")
    _check_process_fn("c5", policy, buf, buf.sample_indices(0), cfg["hidden"])


def test_c2_unfinished_tails(c2):
    """Every third env's last stored row loses its truncation: unfinished_index() reports it, and compute_gae_returns
    must end the segment there through its isin over the whole index set (and evaluate V(obs_next) for it)."""
    policy, buf, cfg = c2
    last = buf.last_index()[::3]
    saved = buf.truncated.clone(), buf.terminated.clone()
    try:
        buf.truncated[last] = 0
        buf.terminated[last] = 0
        unf = buf.unfinished_index()
        assert unf.numel() == last.numel() > 100
        assert torch.equal(torch.sort(unf).values, torch.sort(last).values)
        _check_process_fn("c2 unfinished", policy, buf, buf.sample_indices(0), cfg["hidden"])
    finally:
        buf.truncated.copy_(saved[0])
        buf.terminated.copy_(saved[1])


def test_c2_shuffled_index_subset(c2):
    """A caller-chosen index set: blocks of 64 chronological rows in shuffled order, a quarter of the blocks left out.
    Inside a block V(obs_next[i]) = V(obs[i+1]); at every block border the successor is an unrelated row, so
    compute_gae_returns must run its second critic pass there."""
    policy, buf, cfg = c2
    idx = buf.sample_indices(0)
    blocks = idx.view(-1, 64)
    gen = torch.Generator(device="cpu").manual_seed(3)
    order = torch.randperm(blocks.shape[0], generator=gen)[: blocks.shape[0] * 3 // 4].to(idx.device)
    sub = blocks[order].reshape(-1).contiguous()
    n = int(sub.numel())
    assert n < buf.maxsize                            # gathered, not the zero-copy dense batch
    obs, obs_next = buf.obs[sub], buf.obs_next[sub]
    end = (buf.terminated[sub] | buf.truncated[sub]).bool()
    broken = (obs_next[:-1] != obs[1:]).any(1) & ~end[:-1]
    same = ~(obs_next[:-1] != obs[1:]).any(1)
    assert int(broken.sum()) > 1000 and float(same.float().mean()) > 0.5, (int(broken.sum()), float(same.float().mean()))
    _check_process_fn("c2 shuffled subset", policy, buf, sub, cfg["hidden"])
