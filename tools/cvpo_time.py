"""Time CVPO on the device: microseconds per gradient step (CUDA events around update_many, after warm-up),
kernel launches per step (fsrl_launch_count), env-steps/s of a few trainer cycles, and the card name and power
limit read in the same run.  Prints one JSON line per sample_act_num.

    python tools/cvpo_time.py [--task SafetyCarCircle-v0] [--k 16 64] [--steps 1000]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                      text=True, timeout=30).strip()
    except Exception as e:                      # noqa: BLE001 - report what is known
        out = f"unavailable ({type(e).__name__})"
    return name, out


def run(task, K, steps, warmup, batch, hidden, n_env, cycles):
    import numpy as np
    import torch
    from fsrl_b200 import _lib, envs
    from fsrl_b200.agent import CVPOAgent
    from fsrl_b200.data import FastCollector, VectorReplayBuffer
    env = envs.make(task)
    agent = CVPOAgent(env, seed=1, hidden_sizes=(hidden, hidden), sample_act_num=K)
    pol = agent.policy
    venv = envs.DeviceVectorEnv(task, n_env, seed=2)
    buf = VectorReplayBuffer(n_env * env.spec.max_episode_steps, n_env)
    col = FastCollector(pol, venv, buf)
    pol.train()
    col.collect(n_episode=n_env)
    pol.pre_update_fn()
    np.random.seed(0)
    pol.update_many(warmup, batch, buf)
    torch.cuda.synchronize()
    n0 = _lib.lib.fsrl_launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    pol.update_many(steps, batch, buf)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / steps
    launches = (_lib.lib.fsrl_launch_count() - n0) / steps
    # trainer cycles: collect n_env episodes, update_per_step 0.2, like cvpo_cfg
    t0, env_steps = time.perf_counter(), 0
    for _ in range(cycles):
        pol.pre_update_fn()
        st = col.collect(n_episode=n_env)
        env_steps += int(st["n/st"])
        pol.update_many(max(1, int(st["n/st"] * 0.2)), batch, buf)
        pol.post_update_fn()
    torch.cuda.synchronize()
    sps = env_steps / (time.perf_counter() - t0)
    return dict(task=task, K=K, B=batch, H=hidden, steps=steps, us_per_step=round(us, 1),
                launches_per_step=launches, env_steps_per_s=round(sps), cycle_envs=n_env, cycles=cycles)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--task", default="SafetyCarCircle-v0")
    ap.add_argument("--k", type=int, nargs="+", default=[16, 64])
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--hidden", type=int, default=128)
    ap.add_argument("--envs", type=int, default=20)
    ap.add_argument("--cycles", type=int, default=5)
    a = ap.parse_args()
    name, plimit = _card()
    for K in a.k:
        r = run(a.task, K, a.steps, a.warmup, a.batch, a.hidden, a.envs, a.cycles)
        r.update(gpu=name, power_limit=plimit)
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
