"""Time collect-only env-steps/s of every device environment.

For each task (every device environment by default) a PPO-Lagrangian actor 2x256 (2 x --hidden) collects one episode in each of 2048 envs
(FastCollector.collect(n_episode=2048), the inline path); the collect is timed with CUDA events after a
warm-up collect, the best of --reps.  An env-step is one stored transition (the collect's ``n/st``), so
the Drone tasks, whose episodes end early on a crash, report the rate of the steps actually taken.  The
card name and power limit are read in the same run.  Prints one JSON line per task.

    python tools/env_collect_time.py [--envs 2048] [--reps 5] [--hidden 256] [--tasks SafetyDroneRun-v0,...]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
TASKS = ["SafetyCarCircle-v0", "SafetyCarRun-v0", "SafetyBallCircle-v0", "SafetyBallRun-v0", "SafetyAntCircle-v0",
         "SafetyPointGoal1Gymnasium-v0", "SafetyAntRun-v0", "SafetyDroneCircle-v0", "SafetyDroneRun-v0",
         "SafetyPointCircle1Gymnasium-v0", "SafetyPointCircle2Gymnasium-v0", "SafetyCarCircle1Gymnasium-v0",
         "SafetyCarCircle2Gymnasium-v0", "SafetyPointGoal2Gymnasium-v0", "SafetyCarGoal1Gymnasium-v0",
         "SafetyCarGoal2Gymnasium-v0", "SafetyPointButton1Gymnasium-v0", "SafetyPointButton2Gymnasium-v0",
         "SafetyCarButton1Gymnasium-v0", "SafetyCarButton2Gymnasium-v0", "SafetyPointPush1Gymnasium-v0",
         "SafetyPointPush2Gymnasium-v0", "SafetyCarPush1Gymnasium-v0", "SafetyCarPush2Gymnasium-v0",
         "SafetyHalfCheetahVelocityGymnasium-v1", "SafetyHopperVelocityGymnasium-v1",
         "SafetySwimmerVelocityGymnasium-v1", "SafetyWalker2dVelocityGymnasium-v1", "SafetyAntVelocityGymnasium-v1"]


def _card():
    import subprocess

    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                      text=True, timeout=30).strip()
    except Exception as e:                      # noqa: BLE001 - report what is known
        out = f"unavailable ({type(e).__name__})"
    return name, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--hidden", type=int, default=256)
    ap.add_argument("--tasks", default=",".join(TASKS))
    ap.add_argument("--episodes", type=int, default=0,
                    help="n_episode of each collect (default: --envs, one episode per env; more takes the resolve path)")
    a = ap.parse_args()
    import torch
    from helpers import build_ppo
    assert torch.cuda.is_available(), "env_collect_time needs a GPU"
    name, plimit = _card()
    E = a.envs
    for task in a.tasks.split(","):
        policy, venv, buf, col = build_ppo(task, hidden=(a.hidden, a.hidden), n_env=E)
        n_ep = a.episodes or E
        col.collect(n_episode=n_ep)                 # warm-up
        times, steps = [], []
        for _ in range(a.reps):
            buf.reset()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            st = col.collect(n_episode=n_ep)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
            steps.append(int(st["n/st"]))
        i = min(range(len(times)), key=lambda k: times[k] / steps[k])
        print(json.dumps(dict(task=task, envs=E, episodes=n_ep, hidden=a.hidden, horizon=venv.max_episode_steps, D=venv.D, A=venv.A,
                              env_steps=steps[i], ms=round(times[i], 3),
                              env_steps_per_s=round(steps[i] / (times[i] / 1e3)), terminated=st["terminated"],
                              ms_all=[round(t, 3) for t in times], gpu=name, power_limit=plimit)), flush=True)
        del policy, venv, buf, col
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
