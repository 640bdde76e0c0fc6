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


def buffer_to_numpy(buf):
    g = lambda t: t.detach().cpu().numpy()
    return dict(obs=g(buf.obs), obs_next=g(buf.obs_next), act=g(buf.act), rew=g(buf.rew),
                cost=g(buf.cost), logp=g(buf.logp), terminated=g(buf.terminated).astype(bool),
                truncated=g(buf.truncated).astype(bool), ptr=g(buf.ptr), len=g(buf.len))
