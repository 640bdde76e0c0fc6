"""The host plumbing the learners and agent presets share, without a GPU: the trust-region learners' minibatch
schedule (tianshou's Batch.split with merge_last, on NumPy's global stream), FusedAdam.from_optimizer, and the
presets' device='cpu' warning."""
import types
import warnings

import numpy as np
import pytest
import torch

from fsrl_b200.optim import FusedAdam
from fsrl_b200.policy.trust_region import TrustRegionMixin


def _tianshou_split(n, size):
    """tianshou's Batch.split(size, shuffle=True, merge_last=True), as row-index chunks."""
    indices = np.random.permutation(n)
    merge_last = n % size > 0
    out = []
    for idx in range(0, n, size):
        if merge_last and idx + size + size >= n:
            out.append(indices[idx:])
            break
        out.append(indices[idx:idx + size])
    return out


def _ppo_epoch_lengths(n_total, batch_size):
    """Minibatch lengths of the loop in csrc/ppo.cu:fsrl_ppo_lag_epoch, which checks its count against the one
    the statistics buffer is sized by."""
    merge_last = n_total % batch_size > 0
    lengths, off = [], 0
    while off < n_total:
        B, last = batch_size, False
        if merge_last and off + 2 * batch_size >= n_total:
            B, last = n_total - off, True
        B = min(B, n_total - off)
        lengths.append(B)
        if last:
            break
        off += batch_size
    n_mb = n_total // batch_size if merge_last else (n_total + batch_size - 1) // batch_size
    assert len(lengths) == max(n_mb, 1)
    return lengths


def _minibatches(n_all, batch_size):
    return TrustRegionMixin._minibatches(types.SimpleNamespace(device="cpu"), n_all, batch_size)


@pytest.mark.parametrize("batch_size", [1, 2, 7, 64, 256, 99999])
def test_minibatches_split_like_tianshou_and_the_ppo_driver(batch_size):
    for n_all in range(1, 601):
        np.random.seed(n_all)
        want = _tianshou_split(n_all, batch_size)
        np.random.seed(n_all)
        got = _minibatches(n_all, batch_size)
        assert len(got) == len(want), n_all
        for (perm, n), w in zip(got, want):
            assert perm.dtype == torch.int32 and n == len(w)
            np.testing.assert_array_equal(perm.numpy(), w)
        assert [n for _, n in got] == _ppo_epoch_lengths(n_all, batch_size), n_all


@pytest.mark.parametrize("n_all,batch_size", [(300, 128), (4800, 99999), (10000, 4000), (1, 1)])
def test_minibatches_consume_one_permutation(n_all, batch_size):
    np.random.seed(123)
    want = np.random.permutation(n_all)
    state_after = np.random.get_state()
    np.random.seed(123)
    got = _minibatches(n_all, batch_size)
    np.testing.assert_array_equal(np.concatenate([p.numpy() for p, _ in got]), want)
    after = np.random.get_state()
    assert after[0] == state_after[0] and after[2:] == state_after[2:]
    np.testing.assert_array_equal(after[1], state_after[1])


def test_fused_adam_from_optimizer_keeps_lr_betas_and_eps():
    p = torch.nn.Parameter(torch.zeros(3))
    for opt, want in ((torch.optim.Adam([p], lr=3e-4, betas=(0.8, 0.95), eps=1e-6), (3e-4, (0.8, 0.95), 1e-6)),
                      (torch.optim.Adam([p]), (1e-3, (0.9, 0.999), 1e-8))):
        f = FusedAdam.from_optimizer(opt)
        assert isinstance(f, FusedAdam)
        g = f.param_groups[0]
        assert (g["lr"], g["betas"], g["eps"]) == want
    fused = FusedAdam(lr=2e-3, betas=(0.5, 0.9), eps=1e-7)
    assert FusedAdam.from_optimizer(fused) is fused


@pytest.mark.parametrize("agent", ["PPOLagAgent", "CPOAgent", "TRPOLagAgent", "FOCOPSAgent", "SACLagAgent",
                                   "DDPGLagAgent", "CVPOAgent"])
def test_agent_cpu_device_warning_points_at_the_caller(monkeypatch, agent):
    import fsrl_b200.agent as A_
    from fsrl_b200.policy.base_policy import BasePolicy
    from fsrl_b200.spaces import Box
    monkeypatch.setattr(BasePolicy, "_build_arena",
                        lambda self, device=None: setattr(self, "_arena", types.SimpleNamespace(device="cpu")) or self._arena)
    env = types.SimpleNamespace(observation_space=Box(low=-np.ones(8, np.float32), high=np.ones(8, np.float32)),
                                action_space=Box(low=-np.ones(2, np.float32), high=np.ones(2, np.float32)),
                                spec=types.SimpleNamespace(max_episode_steps=100))
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        getattr(A_, agent)(env, device="cpu", hidden_sizes=(16, 16))
    hits = [w for w in caught if issubclass(w.category, RuntimeWarning) and "device='cpu'" in str(w.message)]
    assert len(hits) == 1
    assert hits[0].filename == __file__
