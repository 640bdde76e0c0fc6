"""The persistent PPO-Lagrangian update (csrc/ppo_persist.cu) at the narrowest and the widest observation its gate
admits (D = 8 and D = 40 = pp::MAXD), 2x256 MLP, batch 256, 16 minibatch steps of one repeat.

Work on this launch's schedule (operand ring, copy order, where partials are kept) must not change a single bit of its
result: the MMAs, their operands and the order of every sum are fixed.  So the parameters and Adam moments after the
repeat are compared, as int32 views, with digests of a recorded run (tests/golden/ppo_persist_golden.json, written by
tools/persist_golden.py).  Inputs are synthetic and come from seeded CPU generators only, so they are the same on every
machine."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ppo_persist_golden.json")
SHAPES = {8: 2, 40: 8}          # D -> A
N_MB = 16


def _policy(D, A, seed):
    from torch.distributions import Independent, Normal

    from fsrl_b200 import nets
    from fsrl_b200.optim import FusedAdam
    from fsrl_b200.policy import PPOLagrangian
    from fsrl_b200.spaces import Box
    gen = torch.Generator().manual_seed(seed)
    actor = nets.ActorProb(nets.Net(D, hidden_sizes=(256, 256)), A, max_action=1.0)
    critics = [nets.Critic(nets.Net(D, hidden_sizes=(256, 256))) for _ in range(2)]
    with torch.no_grad():
        actor.sigma_param.fill_(-0.5)
        for m in list(actor.modules()) + [mm for c in critics for mm in c.modules()]:
            if isinstance(m, torch.nn.Linear):
                m.weight.copy_(torch.randn(m.weight.shape, generator=gen) / np.sqrt(m.weight.shape[1]))
                m.bias.copy_(0.1 * torch.randn(m.bias.shape, generator=gen))
    actor.device = "cuda"
    policy = PPOLagrangian(actor, critics, FusedAdam(lr=5e-4), lambda *l: Independent(Normal(*l), 1),
                           cost_limit=10.0, max_grad_norm=0.5,
                           observation_space=Box(-np.inf, np.inf, shape=(D,)), action_space=Box(-1.0, 1.0, shape=(A,)))
    policy.arena  # adopt the nets
    policy.lag_optims[0].lagrangian = 0.3
    return policy


def _batch(D, A, n, seed):
    from fsrl_b200.policy.base_policy import DeviceBatch
    gen = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=gen)
    b = DeviceBatch()
    b.n = n
    act = torch.tanh(r(n, A))
    logp = (-0.5 * ((act / np.exp(-0.5)) ** 2) - (-0.5) - 0.5 * np.log(2 * np.pi)).sum(1) + 0.1 * r(n)
    b.obs, b.act, b.logp_old = r(n, D).cuda(), act.cuda(), logp.cuda()
    b.v, b.adv, b.ret = r(2, n).cuda(), r(2, n).cuda(), r(2, n).cuda()
    b.values, b.rets, b.advs = b.v.t(), b.ret.t(), b.adv.t()
    return b


def run_repeat(D):
    """One repeat of N_MB persistent steps at observation width D: (launch active, {array: sha256 of its int32 view})."""
    from fsrl_b200 import _lib
    A = SHAPES[D]
    policy = _policy(D, A, seed=100 + D)
    batch = _batch(D, A, N_MB * 256, seed=200 + D)
    policy._ensure_update_state(256, batch.n, 1)
    u = policy._descriptor(batch, torch.zeros(batch.n, dtype=torch.int32, device="cuda"))
    active = _lib.lib.fsrl_ppo_persist_active(ctypes.byref(u), batch.n, 256) == 1
    policy._target_kl = 1e9
    np.random.seed(300 + D)
    policy.learn(batch, batch_size=256, repeat=1)
    torch.cuda.synchronize()
    arrays = dict(theta=policy.arena.theta, m=policy.optim.m, v=policy.optim.v)
    digests = {k: hashlib.sha256(t.detach().cpu().contiguous().view(torch.int32).numpy().tobytes()).hexdigest()
               for k, t in arrays.items()}
    assert np.isfinite(policy.arena.theta.cpu().numpy()).all()
    return active, digests


@pytest.mark.gpu
@pytest.mark.parametrize("D", sorted(SHAPES))
def test_persistent_repeat_bit_identical_to_recording(D):
    with open(GOLDEN) as f:
        want = json.load(f)["D%d" % D]
    active, got = run_repeat(D)
    assert active
    assert got == want
