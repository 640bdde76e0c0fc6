"""Time the three ways of driving the device envs at the c2 shape (SafetyCarCircle-v0, 2048 envs x 300 steps):

* ``step``:    300 calls of DeviceVectorEnv.step with one fixed (E, A) device action tensor;
* ``generic``: FastCollector.collect(n_episode=2048) of a 2x256 torch MLP policy (the generic path: one torch
               forward + one step kernel + one resolve kernel per vector step);
* ``fused``:   the same collect by a PPO-Lagrangian 2x256 actor inside the fused rollout kernel.

Each is timed with CUDA events after a warm-up run, best of --reps; a collect's window includes its end-of-collect
reset of every env (part of collect()), the buffer reset before it is outside.  Prints one JSON line per mode, with the card
name and power limit read in the same run.

    python tools/env_step_time.py [--envs 2048] [--reps 5]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
TASK = "SafetyCarCircle-v0"


def _timed(fn, reps, prep):
    """prep() (buffer / env resets) runs outside the timed window, as in env_collect_time.py"""
    import torch
    prep()
    fn()                                            # warm-up
    times, out = [], None
    for _ in range(reps):
        prep()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return times, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    from env_collect_time import _card
    from helpers import build_ppo

    from fsrl_b200.data import Batch, FastCollector, VectorReplayBuffer
    from fsrl_b200.envs import DeviceVectorEnv
    assert torch.cuda.is_available(), "env_step_time needs a GPU"
    name, plimit = _card()
    E = a.envs
    rows = []

    venv = DeviceVectorEnv(TASK, E, seed=3)
    T = venv.max_episode_steps
    act = torch.rand((E, venv.A), device="cuda") * 2 - 1

    def step_loop():
        for _ in range(T):
            venv.step(act)
        return E * T
    rows.append(("step", _timed(step_loop, a.reps, venv.reset)))

    class Mlp(torch.nn.Module):
        def __init__(self, D, A):
            super().__init__()
            self.net = torch.nn.Sequential(torch.nn.Linear(D, 256), torch.nn.ReLU(), torch.nn.Linear(256, 256),
                                           torch.nn.ReLU(), torch.nn.Linear(256, A), torch.nn.Tanh()).cuda()

        def forward(self, batch, state=None, **kw):
            return Batch(act=self.net(batch.obs))

    gvenv = DeviceVectorEnv(TASK, E, seed=4)
    gbuf = VectorReplayBuffer(E * T, E)
    gcol = FastCollector(Mlp(venv.D, venv.A), gvenv, gbuf)
    assert not gcol.fused

    def generic():
        return int(gcol.collect(n_episode=E)["n/st"])
    rows.append(("generic", _timed(generic, a.reps, gbuf.reset)))

    policy, fvenv, fbuf, fcol = build_ppo(TASK, hidden=(256, 256), n_env=E)
    assert fcol.fused

    def fused():
        return int(fcol.collect(n_episode=E)["n/st"])
    rows.append(("fused", _timed(fused, a.reps, fbuf.reset)))

    for mode, (times, steps) in rows:
        best = min(times)
        print(json.dumps(dict(mode=mode, task=TASK, envs=E, horizon=T, hidden=256, env_steps=steps, ms=round(best, 3),
                              env_steps_per_s=round(steps / (best / 1e3)), ms_all=[round(t, 3) for t in times],
                              gpu=name, power_limit=plimit)), flush=True)


if __name__ == "__main__":
    main()
