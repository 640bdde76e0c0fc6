"""Time DeviceVectorEnv.render (csrc/render.cu) at E in {16, 256} envs and 256x256 / 64x64 frames, after 40 random steps
of the task (default SafetyPointButton2Gymnasium-v0, the largest scene).  Each shape is timed with CUDA events over
--iters back-to-back render() calls after a warm-up, best of --reps; the output tensor's allocation is inside the window,
as a caller of render() pays it.  Prints one JSON line with frames/s per shape, the card name and its power limit.
``--header`` times a user-defined env instead: the plugin of a header whose struct defines draw (DESIGN §7), e.g.
tests/envs_render/car_circle_drawn.h beside the built-in SafetyCarCircle-v0 it restates.

    python tools/render_time.py [--task SafetyPointButton2Gymnasium-v0] [--iters 20] [--reps 5]
    python tools/render_time.py --header tests/envs_render/car_circle_drawn.h [--plugin_dir fsrl_b200/_obj/env_plugins]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--task", default="SafetyPointButton2Gymnasium-v0")
    ap.add_argument("--header", default=None, help="time the plugin of this header (its struct draws) instead of --task")
    ap.add_argument("--plugin_dir", default=None, help="where --header's plugin is built and cached")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import numpy as np
    import torch
    from env_collect_time import _card

    from fsrl_b200.envs import DeviceVectorEnv, build_device_env, register_device_env
    assert torch.cuda.is_available(), "render_time needs a GPU"
    if a.header is not None:
        a.task = "Plugin-" + os.path.splitext(os.path.basename(a.header))[0]
        register_device_env(a.task, build_device_env(a.header, out=a.plugin_dir))
    name, plimit = _card()
    res = {"tool": "render_time", "task": a.task, "header": a.header, "gpu": name, "power_limit_w": plimit, "iters": a.iters}
    for E in (16, 256):
        for size in ((256, 256), (64, 64)):
            venv = DeviceVectorEnv(a.task, E, seed=1, render_mode="rgb_array", render_size=size)
            venv.reset()
            rng = np.random.default_rng(0)
            for _ in range(40):
                venv.step(torch.from_numpy(rng.uniform(-1, 1, (E, venv.A)).astype(np.float32)).cuda())
            venv.render()                                      # warm-up
            best = float("inf")
            for _ in range(a.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                for _ in range(a.iters):
                    venv.render()
                e1.record()
                torch.cuda.synchronize()
                best = min(best, e0.elapsed_time(e1))
            ms = best / a.iters
            res[f"E{E}_{size[0]}x{size[1]}"] = {"ms_per_render": round(ms, 4), "frames_per_s": round(E / ms * 1e3)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
