"""Time the offline-dataset harvest on the device.

One c2-shaped collect (SafetyCarCircle-v0, 2048 envs x 300 steps, PPO-Lagrangian actor 2x256) is timed with
CUDA events after warm-up, without a TrajectoryBuffer and with one attached (keep everything; and the
dataset example's grid filter, 1500 trajectories, filter_interval 1.5), the variants alternating.  Then the
scan, copy and gather kernels are timed alone over the ring of that collect, and their achieved bandwidth
(bytes computed from the shapes) is set against the H100 SXM's 3.35 TB/s.  The card name and power limit
are read in the same run.  Prints one JSON line per measurement.

    python tools/trajbuf_time.py [--envs 2048] [--reps 5] [--kernel_reps 50]
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
PEAK_BPS = 3.35e12


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


def _events_ms(fn, reps):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--task", default="SafetyCarCircle-v0")
    ap.add_argument("--envs", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--kernel_reps", type=int, default=50)
    a = ap.parse_args()
    import torch
    from helpers import build_ppo

    from fsrl_b200 import _lib
    from fsrl_b200.data import FastCollector, TrajectoryBuffer
    from fsrl_b200.data.traj_buf import TrajectoryHarvest
    name, plimit = _card()
    card = dict(gpu=name, power_limit=plimit)
    E = a.envs
    policy, venv, buf, _ = build_ppo(a.task, hidden=(256, 256), n_env=E)
    T, D, A = venv.max_episode_steps, venv.D, venv.A
    variants = {
        "none": lambda: FastCollector(policy, venv, buf, exploration_noise=True),
        "keep_all": lambda: FastCollector(policy, venv, buf, exploration_noise=True, traj_buffer=TrajectoryBuffer()),
        "grid_1500": lambda: FastCollector(policy, venv, buf, exploration_noise=True,
                                           traj_buffer=TrajectoryBuffer(1500, filter_interval=1.5)),
    }
    cols = {k: f() for k, f in variants.items()}
    for c in cols.values():                         # warm-up: every path once
        c.collect(n_episode=E)
    times = {k: [] for k in cols}
    for _ in range(a.reps):                         # alternate the variants
        for k, c in cols.items():
            buf.reset()
            times[k].append(_events_ms(lambda: c.collect(n_episode=E), 1))
    base = min(times["none"])
    for k, ts in times.items():
        print(json.dumps(dict(what="collect", variant=k, task=a.task, envs=E, steps=T, hidden=256, ms_min=round(min(ts), 3),
                              ms_all=[round(t, 3) for t in ts], overhead_vs_none=round(min(ts) / base - 1, 4),
                              env_steps_per_s=round(E * T / (min(ts) / 1e3)), **card)), flush=True)

    # kernels alone, over the ring of the last collect (every env ran one whole episode)
    buf.reset()
    col = cols["none"]
    col.collect(n_episode=E)
    r = col._descriptor(False)
    r.inline_done = 1
    stream = torch.cuda.current_stream().cuda_stream
    hv = TrajectoryHarvest(E, venv.device)
    hv.begin(r, stream)
    rows = hv.scan(r, E, T, stream)
    h = hv._desc(E)

    def scan():
        _lib.check(_lib.lib.fsrl_traj_begin(ctypes.byref(r), ctypes.byref(h), stream))
        _lib.check(_lib.lib.fsrl_traj_scan(ctypes.byref(r), ctypes.byref(h), E, stream))
    n_tr = int(rows["len"].sum())
    scan_ms = _events_ms(scan, a.kernel_reps)
    begin_ms = _events_ms(lambda: _lib.check(_lib.lib.fsrl_traj_begin(ctypes.byref(r), ctypes.byref(h), stream)),
                          a.kernel_reps)
    tb = TrajectoryBuffer()
    slots = [tb._index.offer(float(x["ret"]), float(x["cost"]), int(x["len"])) for x in rows]
    tb._arena.reserve(tb._index.n_slots, T, D, A, venv.device)
    jobs = torch.tensor([[int(x["env"]), int(x["start"]), int(x["len"]), s] for x, s in zip(rows, slots)],
                        dtype=torch.int32).to(venv.device)
    ad = tb._arena.descriptor()
    copy_ms = _events_ms(lambda: _lib.check(_lib.lib.fsrl_traj_copy(ctypes.byref(r), ctypes.byref(ad), jobs.data_ptr(),
                                                                    len(rows), stream)), a.kernel_reps)
    tb.get_all()
    gather_ms = _events_ms(lambda: tb.get_all(), a.kernel_reps)
    per_tr = 2 * (8 * D + 4 * A + 4 + 4 + 1 + 1)      # read + write of obs, obs_next, act, rew, cost, term, trunc
    out = [("scan", scan_ms - begin_ms, n_tr * (4 + 4 + 1 + 1)), ("copy", copy_ms, n_tr * per_tr),
           ("gather", gather_ms, n_tr * per_tr)]
    for what, ms, nbytes in out:
        bps = nbytes / (ms / 1e3)
        print(json.dumps(dict(what=what + "_kernel", transitions=n_tr, episodes=len(rows), D=D, A=A, ms=round(ms, 4),
                              bytes=nbytes, GBps=round(bps / 1e9, 1), share_of_3_35TBps=round(bps / PEAK_BPS, 3),
                              note="gather: get_all() incl. its small host-side job list" if what == "gather" else "",
                              **card)), flush=True)


if __name__ == "__main__":
    main()
