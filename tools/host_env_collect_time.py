"""Time the device side of collecting on host-stepped envs (HostVectorEnv, csrc/rollout_host.cu).

* ``round_trip``: one ``HostVectorEnv.device_step`` per vector step -- the packed H2D copy, the store + act launch,
  the D2H copy of the actions and the stream synchronise -- with every env acting and storing, at --envs x
  --hidden, timed with a host clock around --steps calls after a warm-up (each call ends in a synchronise).  The
  env step is left out: this is what a vector step costs on top of an env whose ``step`` costs nothing.
* ``collect``: FastCollector.collect(n_episode=E) on the SafetyCarCircle-v0 CPU twin behind HostVectorEnv (a
  vectorised numpy env) at E = --collect-envs, whole-collect env-steps/s, best of --reps after a warm-up.

Prints one JSON line per measurement, with the card name and power limit read in the same run.

    python tools/host_env_collect_time.py [--envs 1 16 256 2048] [--hidden 64 256] [--steps 2000]
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
TASK = "SafetyCarCircle-v0"


class _NullVec:
    """E envs whose step and reset cost next to nothing (fixed arrays), behind the vector protocol."""

    def __init__(self, E, D, A):
        from fsrl_b200.spaces import Box
        self.E, self.D = E, D
        self.observation_space = Box(-1.0, 1.0, (D,))
        self.action_space = Box(-1.0, 1.0, (A,))

    def __len__(self):
        return self.E

    def reset(self, id=None, **kw):
        import numpy as np
        return np.zeros((self.E if id is None else len(id), self.D), np.float32)

    def step(self, action, id=None):
        import numpy as np
        n = len(action)
        return np.zeros((n, self.D), np.float32), np.zeros(n), np.zeros(n, bool), np.zeros(n, bool), {}


def round_trip(E, H, steps):
    import numpy as np
    import torch
    from helpers import build_ppo

    from fsrl_b200.data import FastCollector, VectorReplayBuffer
    from fsrl_b200.envs import HostVectorEnv
    policy = build_ppo(TASK, hidden=(H, H), n_env=1)[0]
    D, A = 8, 2                                        # SafetyCarCircle-v0's widths
    venv = HostVectorEnv.from_vector_env(_NullVec(E, D, A))
    buf = VectorReplayBuffer(E * 64, E)
    col = FastCollector(policy, venv, buf, exploration_noise=True)
    r = col._descriptor(False)
    ids = np.arange(E)
    obs = np.random.default_rng(0).standard_normal((E, D)).astype(np.float32)
    store = (ids, obs, np.ones(E, np.float32), np.zeros(E, np.float32), np.zeros(E, bool), np.zeros(E, bool))
    venv.device_step(r, ids, obs)
    for _ in range(20):                                # warm-up
        venv.device_step(r, ids, obs, store)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        venv.device_step(r, ids, obs, store)
    dt = time.perf_counter() - t0
    return dt / steps


def collect(E, H, reps):
    import torch
    from helpers import build_ppo
    from host_twin import host_twin

    from fsrl_b200.data import FastCollector, VectorReplayBuffer
    policy = build_ppo(TASK, hidden=(H, H), n_env=1)[0]
    venv = host_twin(TASK, E, 3)
    T = venv.max_episode_steps
    buf = VectorReplayBuffer(E * T, E)
    col = FastCollector(policy, venv, buf, exploration_noise=True)
    col.collect(n_episode=E)                           # warm-up
    times, steps = [], 0
    for _ in range(reps):
        buf.reset()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        steps = int(col.collect(n_episode=E)["n/st"])
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return steps, times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, nargs="+", default=[1, 16, 256, 2048])
    ap.add_argument("--hidden", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--collect-envs", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    from env_collect_time import _card
    assert torch.cuda.is_available(), "host_env_collect_time needs a GPU"
    name, plimit = _card()
    for H in a.hidden:
        for E in a.envs:
            s = round_trip(E, H, a.steps)
            print(json.dumps(dict(mode="round_trip", envs=E, hidden=H, steps=a.steps, us_per_step=round(s * 1e6, 2),
                                  gpu=name, power_limit=plimit)), flush=True)
    steps, times = collect(a.collect_envs, 64, a.reps)
    best = min(times)
    print(json.dumps(dict(mode="collect", task=TASK + " (CPU twin)", envs=a.collect_envs, hidden=64, env_steps=steps,
                          s=round(best, 3), env_steps_per_s=round(steps / best), s_all=[round(t, 3) for t in times],
                          gpu=name, power_limit=plimit)), flush=True)


if __name__ == "__main__":
    main()
