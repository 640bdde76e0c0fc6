"""Time what a TrajectoryBuffer harvest adds to collecting on host-stepped envs (FastCollector's host path).

Per (task, E): two collectors over two HostVectorEnvs of the task's CPU twin (tests/host_twin.py, the vectorised numpy
env) with the same seed, both storing into a ring of E * T slots, one of them also feeding a TrajectoryBuffer (keep
everything).  After a warm-up collect each, --reps collects of n_episode = E alternate between the two.  A collect's
wall time (host clock, ending in a device synchronise) over the number of vector steps it ran (the env's ``step``
calls) is the time per host vector step: env step, the one launch that acts and stores, and with the buffer the
per-episode offers and the copy launches.  SafetyDroneRun-v0 terminates episodes at different steps, so copies are
spread over the collect; SafetyCarCircle-v0 only truncates, so every copy lands on the last step.

Prints one JSON line per (task, E, arm), with the card name and power limit read in the same run.

    python tools/host_traj_time.py [--envs 64 512 2048] [--reps 5]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
TASKS = ("SafetyDroneRun-v0", "SafetyCarCircle-v0")


def _arm(task, E, policy, traj, seed=3):
    from host_twin import TwinVectorEnv, twin

    from fsrl_b200.data import FastCollector, TrajectoryBuffer, VectorReplayBuffer
    from fsrl_b200.envs import HostVectorEnv

    class Counting(TwinVectorEnv):
        steps = 0

        def step(self, action, id=None):
            self.steps += 1
            return super().step(action, id)

    tv = Counting(twin(task, E, seed), task)
    venv = HostVectorEnv.from_vector_env(tv)
    T = venv.max_episode_steps
    tb = TrajectoryBuffer() if traj else None
    col = FastCollector(policy, venv, VectorReplayBuffer(E * T, E), exploration_noise=True, traj_buffer=tb)
    return col, tv, tb


def _timed(col, tv, E):
    import torch
    tv.steps = 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    st = col.collect(n_episode=E)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, tv.steps, int(st["n/st"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, nargs="+", default=[64, 512, 2048])
    ap.add_argument("--tasks", nargs="+", default=list(TASKS))
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    from env_collect_time import _card
    from helpers import build_ppo
    assert torch.cuda.is_available(), "host_traj_time needs a GPU"
    name, plimit = _card()
    for task in a.tasks:
        policy = build_ppo(task, hidden=(64, 64), n_env=1)[0]
        policy.train()
        for E in a.envs:
            arms = {traj: _arm(task, E, policy, traj) for traj in (False, True)}
            for col, tv, _ in arms.values():
                col.collect(n_episode=E)                       # warm-up
            runs = {False: [], True: []}
            for _ in range(a.reps):
                for traj in (False, True):
                    col, tv, _ = arms[traj]
                    runs[traj].append(_timed(col, tv, E))
            for traj in (False, True):
                per_step = [s / n for s, n, _ in runs[traj]]
                tb = arms[traj][2]
                print(json.dumps(dict(
                    task=task + " (CPU twin)", envs=E, traj_buffer=traj, hidden=64, reps=a.reps,
                    vector_steps=[n for _, n, _ in runs[traj]], env_steps=[m for _, _, m in runs[traj]],
                    us_per_vector_step_median=round(statistics.median(per_step) * 1e6, 1),
                    us_per_vector_step_all=[round(x * 1e6, 1) for x in per_step],
                    trajectories=len(tb.buffer) if tb is not None else None,
                    gpu=name, power_limit=plimit)), flush=True)


if __name__ == "__main__":
    main()
