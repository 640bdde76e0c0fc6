"""Oracle (test infrastructure): numpy twin of the device Philox4x32-10 stream and of the
normal / uniform transforms in fsrl_b200/csrc/common.cuh + envs.cuh.  This RNG stream is
OUR documented design (the reference draws actions from torch's CPU generator, which no GPU
kernel can replay); the oracle exists so that device rollouts are reproducible on the CPU."""
from __future__ import annotations

import numpy as np

M0 = np.uint64(0xD2511F53)
M1 = np.uint64(0xCD9E8D57)
W0 = np.uint32(0x9E3779B9)
W1 = np.uint32(0xBB67AE85)
KEY_RESET = 0x52534554
KEY_ACT = 0x4143544E
KEY_GOAL = 0x474F414C


def philox4x32(c0, c1, c2, c3, k0, k1):
    """All arguments broadcastable uint32 arrays/scalars -> tuple of 4 uint32 arrays."""
    c0, c1, c2, c3 = np.broadcast_arrays(*(np.asarray(x, dtype=np.uint32) for x in (c0, c1, c2, c3)))
    c0, c1, c2, c3 = c0.copy(), c1.copy(), c2.copy(), c3.copy()
    k0 = np.uint32(k0); k1 = np.uint32(k1)
    with np.errstate(over="ignore"):
        for _ in range(10):
            p0 = M0 * c0.astype(np.uint64)
            p1 = M1 * c2.astype(np.uint64)
            hi0 = (p0 >> np.uint64(32)).astype(np.uint32); lo0 = p0.astype(np.uint32)
            hi1 = (p1 >> np.uint64(32)).astype(np.uint32); lo1 = p1.astype(np.uint32)
            n0 = hi1 ^ c1 ^ k0
            n2 = hi0 ^ c3 ^ k1
            c0, c1, c2, c3 = n0, lo1, n2, lo0
            k0 = np.uint32(k0 + W0); k1 = np.uint32(k1 + W1)
    return c0, c1, c2, c3


def usym(x):
    """uniform in [-1, 1): (x >> 8) * 2^-23 - 1, f32 exact (envs.cuh usym)."""
    return ((x >> np.uint32(8)).astype(np.float32) * np.float32(2.0 / 16777216.0) - np.float32(1.0)).astype(np.float32)


def normal_pair(xa, xb):
    """Box-Muller in f64 from two u32 words (common.cuh gauss_pair): u1 = (a+1)*2^-32 in
    (0,1], u2 = b*2^-32; returns two f32 normals."""
    u1 = (xa.astype(np.float64) + 1.0) * (1.0 / 4294967296.0)
    u2 = xb.astype(np.float64) * (1.0 / 4294967296.0)
    r = np.sqrt(-2.0 * np.log(u1))
    ang = 2.0 * np.pi * u2
    return (r * np.cos(ang)).astype(np.float32), (r * np.sin(ang)).astype(np.float32)


def action_uniform(seed, env_ids, act_ctr, A):
    """u[e, a] in [-1, 1) of a random-mode action with per-env counter act_ctr[e] (rollout.cu):
    actions 4c .. 4c + 3 come from the draw with counter word 2 = c"""
    env_ids = np.asarray(env_ids, dtype=np.uint32)
    act_ctr = np.asarray(act_ctr, dtype=np.uint32)
    out = np.zeros((env_ids.shape[0], A), dtype=np.float32)
    for call in range((A + 3) // 4):
        r = philox4x32(env_ids, act_ctr, np.uint32(call), np.uint32(0), seed, KEY_ACT)
        for j in range(min(4, A - 4 * call)):
            out[:, 4 * call + j] = usym(r[j])
    return out


def action_noise(seed, env_ids, act_ctr, A):
    """eps[e, a] for the action sampled with per-env counter act_ctr[e] (rollout.cu)."""
    env_ids = np.asarray(env_ids, dtype=np.uint32)
    act_ctr = np.asarray(act_ctr, dtype=np.uint32)
    out = np.zeros((env_ids.shape[0], A), dtype=np.float32)
    for call in range((A + 3) // 4):
        r = philox4x32(env_ids, act_ctr, np.uint32(call), np.uint32(0), seed, KEY_ACT)
        n0, n1 = normal_pair(r[0], r[1])
        n2, n3 = normal_pair(r[2], r[3])
        for j, n in enumerate((n0, n1, n2, n3)):
            a = 4 * call + j
            if a < A:
                out[:, a] = n
    return out
