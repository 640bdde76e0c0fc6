"""The persistent PPO-Lagrangian update (csrc/ppo_persist.cu) at the widest observation and action the gate admits
among the tasks: SafetyAntCircle-v0 (D = 34, A = 8), 2x256 MLP, 64 envs, batch 256.  The dW1 / db1 partials the G2
CTAs keep on chip grow with D, so this is the shape where their shared-memory layout and the reducers' 8-way sums
over distributed shared memory cover the most rows.  Same criteria as the D = 8 case in test_ppo_scale_gpu.py."""
import copy
import ctypes

import numpy as np
import pytest
import torch

from test_ppo_scale_gpu import KEYS, _adam, _assert_params_within_fp32_noise, _collect, _sub_batch

pytestmark = pytest.mark.gpu


def test_persistent_path_widest_input_matches_oracle():
    from fsrl_b200 import _lib
    from oracle import ppo as oppo
    lag = 0.3
    policy, batch, ob, actor, critics = _collect("SafetyAntCircle-v0", (256, 256), 64, lag)
    assert ob["obs"].shape[1] == 34 and ob["act"].shape[1] == 8
    assert batch.n % 256 == 0
    policy._ensure_update_state(256, batch.n, 1)
    u = policy._descriptor(batch, torch.zeros(batch.n, dtype=torch.int32, device="cuda"))
    assert _lib.lib.fsrl_ppo_persist_active(ctypes.byref(u), batch.n, 256) == 1
    sd0 = copy.deepcopy(policy.state_dict())
    # the first 8 steps of a whole repeat
    a1, c1 = copy.deepcopy(actor), copy.deepcopy(critics)
    np.random.seed(41)
    ostats = oppo.learn(a1, c1, _adam(a1, c1), ob, 256, 1, lag, max_grad_norm=0.5, target_kl=1e9, max_steps=8)
    np.random.seed(41)
    policy._target_kl = 1e9
    policy.learn(batch, batch_size=256, repeat=1)
    st = policy.last_stats
    assert len(st["loss/kl"]) == batch.n // 256
    for key in KEYS:
        want = np.array([s[key] for s in ostats])
        np.testing.assert_allclose(np.asarray(st[key])[:8], want, rtol=3e-4, atol=3e-6, err_msg=key)
        assert np.isfinite(np.asarray(st[key])).all(), key
    # the parameters after a complete 8-step epoch
    policy.load_state_dict(sd0)
    policy.optim.m.zero_(); policy.optim.v.zero_(); policy.optim.step_count = 0
    n = 8 * 256
    sub = _sub_batch(policy, batch, n)
    osub = {k: v[:n].copy() for k, v in ob.items()}
    a2, c2 = copy.deepcopy(actor), copy.deepcopy(critics)
    np.random.seed(42)
    oppo.learn(a2, c2, _adam(a2, c2), osub, 256, 1, lag, max_grad_norm=0.5, target_kl=1e9)
    np.random.seed(42)
    policy.learn(sub, batch_size=256, repeat=1)
    _assert_params_within_fp32_noise(policy, [a2] + c2, actor, critics, osub, lag, 42)
