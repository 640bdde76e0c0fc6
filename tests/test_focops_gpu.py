"""FOCOPS parity (SURVEY.md 8f-2): critic regression + actor step with the KL-indicator mask on
the device (csrc/cpo.cu::focops_head_kernel + the generic engine) against the torch-CPU autograd
restatement of fsrl/policy/focops.py:157-251 -- same weights, same collected batch, same
permutations.  Tolerances: per-minibatch losses rtol 2e-3 (3xTF32 GEMMs + fp32 reductions in a
different order), parameters atol 2e-4 after 2 x 5 optimiser steps."""
import numpy as np
import pytest
import torch

from helpers import buffer_to_numpy

pytestmark = pytest.mark.gpu


def _setup(hidden=(64, 64), task="SafetyCarCircle-v0", n_env=4, **kw):
    from fsrl_b200 import envs
    from fsrl_b200.agent import FOCOPSAgent
    from fsrl_b200.data import FastCollector, VectorReplayBuffer
    env = envs.make(task)
    agent = FOCOPSAgent(env, seed=10, hidden_sizes=hidden, **kw)
    policy = agent.policy
    venv = envs.DeviceVectorEnv(task, n_env, seed=12)
    buf = VectorReplayBuffer(n_env * env.spec.max_episode_steps, n_env)
    col = FastCollector(policy, venv, buf, exploration_noise=True)
    return policy, venv, buf, col


def test_nu_update_matches_reference_arithmetic():
    from oracle import focops as ofoc
    policy, venv, buf, col = _setup()
    policy._ave_cost_return = 31.5
    st = policy.nu_loss()
    want, loss_nu = ofoc.nu_step(0.0, 1e-2, 2.0, 10.0, 31.5)
    assert st["loss/nu_value"] == pytest.approx(want, abs=1e-7) and st["loss/nu_loss"] == loss_nu
    for cost in (50.0, 300.0, 0.0):              # clamp at nu_max and at 0
        policy._ave_cost_return = cost
        got = policy.nu_loss()["loss/nu_value"]
        want, _ = ofoc.nu_step(want, 1e-2, 2.0, 10.0, cost)
        assert got == pytest.approx(want, abs=1e-7)


@pytest.mark.parametrize("eta,hidden,n_env,batch_size", [
    pytest.param(0.02, (64, 64), 4, 256, id="0.02"),
    pytest.param(1e-4, (64, 64), 4, 256, id="0.0001"),
    # one minibatch of ~4800 rows (merge_last): the actor's wgrad splits the rows and the default
    # max_grad_norm clips with the norm of the combined gradient
    pytest.param(0.02, (128, 128), 16, 99999, id="h128-16env-whole-batch"),
])
def test_focops_learn_matches_oracle(eta, hidden, n_env, batch_size):
    from oracle import focops as ofoc, nets as onets
    policy, venv, buf, col = _setup(hidden, n_env=n_env, eta=eta, delta=1e9)
    stats = col.collect(n_episode=n_env)
    policy.pre_update_fn(stats_train=stats)
    sd = policy.state_dict()
    D, A = venv.D, venv.A
    actor = onets.load_from_state_dict(onets.GaussActor(D, A, list(hidden)), sd, "actor.")
    critics = [onets.load_from_state_dict(onets.ValueNet(D, list(hidden)), sd, f"critics.{i}.") for i in range(2)]
    idx = buf.sample_indices(0)
    batch = policy.process_fn(None, buf, idx)
    b = buffer_to_numpy(buf)
    sel = idx.cpu().numpy()
    ob = {k: b[k][sel] for k in ("obs", "obs_next", "act", "rew", "cost", "terminated", "truncated")}
    ob = ofoc.process(actor, critics, ob, 0.99, 0.95)
    # the GAE / old-distribution parity is covered elsewhere: continue from the device batch
    ob["advs"] = batch.advs.cpu().numpy().copy(); ob["rets"] = batch.rets.cpu().numpy().copy()
    ob["logp_old"] = batch.logp_old.cpu().numpy().copy()
    assert np.allclose(ob["mean_old"], batch.mean_old.cpu().numpy(), atol=2e-5)
    ob["mean_old"] = batch.mean_old.cpu().numpy().copy(); ob["std_old"] = batch.std_old.cpu().numpy().copy()
    aopt = torch.optim.Adam(actor.parameters(), lr=5e-4)
    copt = torch.optim.Adam([p for c in critics for p in c.parameters()], lr=1e-3)
    nu, _ = ofoc.nu_step(0.0, 1e-2, 2.0, 10.0, stats["cost"])
    whole = batch_size >= batch.n
    if whole:
        assert batch.n > 4096 and policy._grad_norm == 0.5
    np.random.seed(4)
    ostats = ofoc.learn(actor, critics, aopt, copt, ob, batch_size, 2, nu, eta=eta, delta=1e9)
    np.random.seed(4)
    policy.learn(batch, batch_size=batch_size, repeat=2)
    st = policy.last_stats
    assert len(st["loss/kl"]) == len(ostats) >= (2 if whole else 8)
    assert st["loss/nu_value"][0] == pytest.approx(nu, abs=1e-7)
    for key in ("loss/actor_loss", "loss/kl", "loss/entropy", "loss/vf0", "loss/vf1", "loss/vf_total"):
        want = np.array([s[key] for s in ostats]); got = np.array(st[key])
        assert np.allclose(got, want, rtol=2e-3, atol=2e-5), (key, np.abs(got - want).max(), got[:3], want[:3])
    if eta < 1e-3:      # the indicator must actually bite in this case
        assert max(s["loss/kl"] for s in ostats[1:]) > eta
    sd2 = policy.state_dict()
    pairs = [("actor.preprocess.model.model.0.weight", actor.body.layers[0].weight),
             ("actor.preprocess.model.model.2.weight", actor.body.layers[1].weight),
             ("actor.mu.model.0.weight", actor.mu.weight), ("actor.mu.model.0.bias", actor.mu.bias),
             ("actor.sigma_param", actor.sigma_param)]
    for i, c in enumerate(critics):
        pairs += [(f"critics.{i}.preprocess.model.model.0.weight", c.body.layers[0].weight),
                  (f"critics.{i}.preprocess.model.model.2.weight", c.body.layers[1].weight),
                  (f"critics.{i}.last.model.0.weight", c.last.weight)]
    for key, ref in pairs:
        got = sd2[key].detach().cpu()
        assert torch.allclose(got, ref.detach().reshape(got.shape), atol=3e-4), (key, (got - ref.detach().reshape(got.shape)).abs().max())
