"""Time the fused collect of built-in SafetyCarCircle-v0 against its same-struct plugin (tests/envs/car_circle.h) at
c2's shapes: 2048 envs x 300 steps (one episode each), actor H = 256, one launch per collect.  The two alternate in
one process after a warm-up; each line is one timed collect.  The plugin runs the same kernel instantiations, so the
only extra cost is the indirect call through the registered table per launch.

    python tools/env_plugin_time.py --reps 10 > profiles/h100_env_plugin_time.jsonl     (GPU)
    python tools/env_plugin_time.py --compile-time                                       (CPU: nvcc of the plugin)
    python tools/env_plugin_time.py --ptxas          (CPU: -Xptxas -v and SASS of the nine kernels, plugin vs library)
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HEADER = os.path.join(ROOT, "tests", "envs", "car_circle.h")
PLUGIN_DIR = os.path.join(ROOT, "fsrl_b200", "_obj", "env_plugins")
TASK, PLUGIN_TASK = "SafetyCarCircle-v0", "PluginCarCircle-v0"


def ptxas_report(log, kind=None):
    """{kernel: [ptxas lines]} of a -Xptxas -v log (compile times dropped); with `kind`, only the kernels
    instantiated for that env kind, keyed with the kind replaced by K."""
    out, cur = {}, None
    for line in open(log):
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            cur = m.group(1)
            if kind is not None:
                cur = cur.replace(f"ILi{kind}E", "ILiKE") if f"ILi{kind}E" in cur else None
            if cur:
                out[cur] = []
        elif cur and line.startswith("ptxas info") and "Compile time" not in line and "Function properties" not in line:
            out[cur].append(line.split(":", 1)[1].strip())
        elif cur and "bytes stack frame" in line:
            out[cur].append(line.strip())
    return out


def sass(binary, kind):
    """{kernel: [instructions]} of the kernels instantiated for `kind` in a cubin container (cuobjdump -sass)."""
    dump = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-sass", binary], capture_output=True, text=True,
                          check=True).stdout
    out, cur = {}, None
    for line in dump.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1).replace(f"ILi{kind}E", "ILiKE") if f"ILi{kind}E" in m.group(1) else None
            if cur:
                out[cur] = []
        elif cur:
            m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(.*?);", line)
            if m:
                out[cur].append(m.group(1))
    return out


def compare_ptxas():
    """The library's CarCircle kernels (kind 0, csrc/rollout.cu) against the plugin's (template argument 64)."""
    from fsrl_b200 import envs
    path = envs.plugin_path(HEADER, PLUGIN_DIR)
    lib = ptxas_report(os.path.join(ROOT, "fsrl_b200", "_obj", "rollout.ptxas.log"), 0)
    plug = ptxas_report(path + ".ptxas.log", 64)
    lib_sass = sass(os.path.join(ROOT, "fsrl_b200", "_obj", "rollout.o"), 0)
    plug_sass = sass(path, 64)
    for k in sorted(plug):
        print(json.dumps({"kernel": k, "library": lib.get(k), "plugin": plug[k], "sass_instructions": len(plug_sass[k]),
                          "sass_identical": lib_sass.get(k) == plug_sass[k]}))
    same = lib == plug and all(lib_sass.get(k) == v for k, v in plug_sass.items())
    print(json.dumps({"kernels": len(plug), "identical": same}))
    return 0 if same else 1


def compile_time(reps, header):
    from fsrl_b200 import envs
    for _ in range(reps):
        with tempfile.TemporaryDirectory() as d:
            t0 = time.perf_counter()
            envs.build_device_env(header, out=d)
            print(json.dumps({"what": "plugin compile", "header": os.path.relpath(header, ROOT),
                              "seconds": round(time.perf_counter() - t0, 2)}))


def time_collects(reps, warmup):
    import torch
    from fsrl_b200 import envs
    from fsrl_b200.agent import PPOLagAgent
    from fsrl_b200.data import FastCollector, VectorReplayBuffer
    envs.register_device_env(PLUGIN_TASK, envs.plugin_path(HEADER, PLUGIN_DIR))
    E = 2048
    gpu = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    cols = {}
    for task in (TASK, PLUGIN_TASK):
        agent = PPOLagAgent(envs.make(task), seed=1, hidden_sizes=(256, 256))
        venv = envs.DeviceVectorEnv(task, E, seed=2)
        cols[task] = FastCollector(agent.policy, venv, VectorReplayBuffer(E * 300, E), exploration_noise=True)
    for _ in range(warmup):
        for col in cols.values():
            col.reset_buffer()
            col.collect(n_episode=E)
    torch.cuda.synchronize()
    for r in range(reps):
        for task, col in cols.items():
            col.reset_buffer()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            st = col.collect(n_episode=E)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            print(json.dumps({"rep": r, "task": task, "envs": E, "steps": int(st["n/st"]), "H": 256,
                              "collect_ms": round(dt * 1e3, 3), "env_steps_per_s": round(st["n/st"] / dt),
                              "gpu": gpu, "power_limit": power}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--compile-time", action="store_true")
    ap.add_argument("--header", default=HEADER, help="the header --compile-time builds (default: the CarCircle one)")
    ap.add_argument("--ptxas", action="store_true")
    a = ap.parse_args()
    if a.ptxas:
        return compare_ptxas()
    if a.compile_time:
        return compile_time(a.reps, os.path.abspath(a.header))
    return time_collects(a.reps, a.warmup)


if __name__ == "__main__":
    sys.exit(main() or 0)
