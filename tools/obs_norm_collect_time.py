"""Time FastCollector.collect on wrapped (VectorEnvNormObs) and unwrapped device envs, alternated in one process.

An unwrapped inline collect is one launch for the whole episode loop; a wrapped one takes six launches per vector
step (step, two per statistics update, resolve).  Shapes: c2's (SafetyCarCircle-v0, 2048 envs x 300 steps,
2x256 actor) and SafetyHalfCheetahVelocityGymnasium-v1 (2048 envs x 1000 steps).  Train-mode collects with
n_episode = envs (every env runs one episode).  Prints one JSON line per measurement, with the card name and power
limit read in the same run.

  python tools/obs_norm_collect_time.py [--reps 5]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

SHAPES = [("SafetyCarCircle-v0", 2048, (256, 256)), ("SafetyHalfCheetahVelocityGymnasium-v1", 2048, (256, 256))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    from env_collect_time import _card
    from fsrl_b200 import _lib
    from fsrl_b200.data import FastCollector
    from fsrl_b200.envs import VectorEnvNormObs
    from helpers import build_ppo
    assert torch.cuda.is_available(), "obs_norm_collect_time needs a GPU"
    name, plimit = _card()
    for task, E, hidden in SHAPES:
        policy, venv, buf, plain = build_ppo(task, hidden=hidden, n_env=E)
        policy.train()
        wrapped = FastCollector(policy, VectorEnvNormObs(venv), buf, exploration_noise=True)
        for c in (plain, wrapped):                      # warm-up: first launches, attribute setup
            c.collect(n_episode=E)
        for rep in range(a.reps):
            for label, c in (("unwrapped", plain), ("wrapped", wrapped)):
                torch.cuda.synchronize()
                l0 = int(_lib.lib.fsrl_launch_count())
                t0 = time.perf_counter()
                st = c.collect(n_episode=E)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                print(json.dumps(dict(task=task, envs=E, hidden=list(hidden), mode=label, rep=rep, env_steps=st["n/st"],
                                      s_per_collect=round(dt, 5), env_steps_per_s=round(st["n/st"] / dt),
                                      launches=int(_lib.lib.fsrl_launch_count()) - l0, gpu=name,
                                      power_limit=plimit)), flush=True)


if __name__ == "__main__":
    main()
