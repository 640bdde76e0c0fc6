"""Shared builders for the parity tests: product-side policy on the GPU and its oracle twin
(plain torch-CPU nets carrying the SAME weights)."""
import numpy as np
import torch
from torch.distributions import Independent, Normal


def build_ppo(task="SafetyCarCircle-v0", hidden=(64, 64), seed=10, n_env=8, buffer_size=None,
              cost_limit=10.0, lr=5e-4, max_grad_norm=0.5, device="cuda", **policy_kw):
    from fsrl_b200 import envs, nets
    from fsrl_b200.data import FastCollector, VectorReplayBuffer
    from fsrl_b200.optim import FusedAdam
    from fsrl_b200.policy import PPOLagrangian
    torch.manual_seed(seed)
    np.random.seed(seed)
    env = envs.make(task)
    D, A = env.observation_space.shape[0], env.action_space.shape[0]
    actor = nets.ActorProb(nets.Net(D, hidden_sizes=hidden), A, max_action=1.0)
    critics = [nets.Critic(nets.Net(D, hidden_sizes=hidden)) for _ in range(2)]
    torch.nn.init.constant_(actor.sigma_param, -0.5)
    for m in list(actor.modules()) + [mm for c in critics for mm in c.modules()]:
        if isinstance(m, torch.nn.Linear):
            torch.nn.init.orthogonal_(m.weight)
            torch.nn.init.zeros_(m.bias)
    actor.device = device
    policy = PPOLagrangian(actor, critics, FusedAdam(lr=lr), lambda *l: Independent(Normal(*l), 1),
                           cost_limit=cost_limit, max_grad_norm=max_grad_norm,
                           observation_space=env.observation_space, action_space=env.action_space,
                           **policy_kw)
    policy.arena  # adopt the nets
    policy.set_action_seed(seed + 1)
    venv = envs.DeviceVectorEnv(task, n_env, device=device, seed=seed + 2)
    T = env.spec.max_episode_steps
    buf = VectorReplayBuffer(buffer_size if buffer_size else n_env * T, n_env, device=device)
    col = FastCollector(policy, venv, buf, exploration_noise=True)
    return policy, venv, buf, col


def oracle_nets(policy, hidden):
    from oracle import nets as onets
    sd = policy.state_dict()
    D = policy.arena.slots[0].D
    A = policy.arena.slots[0].out
    actor = onets.load_from_state_dict(onets.GaussActor(D, A, list(hidden)), sd, "actor.")
    critics = [onets.load_from_state_dict(onets.ValueNet(D, list(hidden)), sd, f"critics.{i}.")
               for i in range(policy.critics_num)]
    return actor, critics


def adam64(p, g, m, v, t, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
    """One torch.optim.Adam step (single-tensor form) in float64; returns (p, m, v)."""
    b1, b2 = betas
    p, g, m, v = (torch.as_tensor(a, dtype=torch.float64) for a in (p, g, m, v))
    g = g + weight_decay * p
    m = m + (1.0 - b1) * (g - m)
    v = v * b2 + (1.0 - b2) * g * g
    denom = v.sqrt() / np.sqrt(1.0 - b2 ** t) + eps
    return p - (lr / (1.0 - b1 ** t)) * m / denom, m, v


def cg64(mvp, b, nsteps=10, tol=1e-8):
    """Conjugate gradients in float64 with the trust-region learners' early exit (stop once
    r.r < tol, after x and r have been updated).  Returns x and r.r after every iteration run."""
    b = torch.as_tensor(b, dtype=torch.float64)
    x, r, p = torch.zeros_like(b), b.clone(), b.clone()
    rs_old = float(r @ r)
    res = []
    for _ in range(nsteps):
        z = mvp(p)
        alpha = rs_old / float(p @ z)
        x = x + alpha * p
        r = r - alpha * z
        rs_new = float(r @ r)
        res.append(rs_new)
        if rs_new < tol:
            break
        p = r + (rs_new / rs_old) * p
        rs_old = rs_new
    return x, res


def cg_stop_tol(res, lo=2, hi=7):
    """A residual_tol that stops cg64 right after iteration k (0-based) of a run whose r.r were
    `res`: the geometric mean of min(res[:k]) and res[k], for the k in [lo, hi) with the widest
    gap between the two.  Returns (k, tol)."""
    k = max(range(lo, min(hi, len(res))), key=lambda j: min(res[:j]) / res[j])
    return k, (min(res[:k]) * res[k]) ** 0.5


KEY_UPD = 0x55504454


def upd_noise(seed, B, A, step, stream_id):
    """eps [B, A] of the off-policy update's reparameterised samples at gradient step `step`
    (csrc/offpolicy.cu sac_sample_kernel): stream 0 draws the target-side sample, stream 1 the actor's."""
    from oracle.philox import normal_pair, philox4x32
    out = np.zeros((B, A), np.float32)
    b = np.arange(B, dtype=np.uint32)
    for c in range((A + 3) // 4):
        r = philox4x32(b, np.uint32(step & 0xFFFFFFFF), np.uint32((step >> 32) * 8 + c), np.uint32(stream_id), seed, KEY_UPD)
        n = list(normal_pair(r[0], r[1])) + list(normal_pair(r[2], r[3]))
        for j in range(4):
            if 4 * c + j < A:
                out[:, 4 * c + j] = n[j]
    return torch.from_numpy(out)


def synthetic_ring(D, A, n_env, cap, layout, seed=0, max_action=1.0, p_term=0.02, p_trunc=0.01):
    """A VectorReplayBuffer filled directly, without collecting.  layout: "wrapped" (every ring full,
    ptr mid-ring), "partial" (every ring partly filled) or "mixed" (alternate envs).  Besides the
    random flags, env e gets a termination (even e) or a truncation (odd e) 1 + e % 8 steps before
    its ptr, so n-step walks from near the newest slot meet both kinds of ends at every distance."""
    from fsrl_b200.data import VectorReplayBuffer
    g = np.random.default_rng(seed)
    buf = VectorReplayBuffer(n_env * cap, n_env, device="cuda")
    buf.allocate(D, A)
    n = n_env * cap
    f32 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()
    buf.obs.copy_(f32(g.standard_normal((n, D))))
    buf.obs_next.copy_(f32(g.standard_normal((n, D))))
    buf.act.copy_(f32(max_action * g.uniform(-1.0, 1.0, (n, A))))
    buf.rew.copy_(f32(g.standard_normal(n)))
    buf.cost.copy_(f32(g.random(n) < 0.3))
    term, trunc = g.random(n) < p_term, g.random(n) < p_trunc
    ptr, ln = np.zeros(n_env, np.int64), np.zeros(n_env, np.int64)
    for e in range(n_env):
        full = layout == "wrapped" or (layout == "mixed" and e % 2 == 0)
        ptr[e] = g.integers(1, cap) if full else g.integers(max(cap // 3, 9), cap)
        ln[e] = cap if full else ptr[e]
        k = e * cap + (ptr[e] - 1 - e % 8) % cap
        term[k], trunc[k] = e % 2 == 0, e % 2 == 1
    buf.terminated.copy_(torch.from_numpy(term.astype(np.uint8)).cuda())
    buf.truncated.copy_(torch.from_numpy(trunc.astype(np.uint8)).cuda())
    buf.ptr.copy_(torch.from_numpy(ptr.astype(np.int32)).cuda())
    buf.len.copy_(torch.from_numpy(ln.astype(np.int32)).cuda())
    return buf


def buffer_to_numpy(buf):
    g = lambda t: t.detach().cpu().numpy()
    return dict(obs=g(buf.obs), obs_next=g(buf.obs_next), act=g(buf.act), rew=g(buf.rew),
                cost=g(buf.cost), logp=g(buf.logp), terminated=g(buf.terminated).astype(bool),
                truncated=g(buf.truncated).astype(bool), ptr=g(buf.ptr), len=g(buf.len))
