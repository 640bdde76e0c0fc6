"""Kernel micro-benchmarks (CUDA events on the launching stream, L2 flushed between
iterations).  Usage: python tools/kbench.py gae [--envs 2048 --T 300]"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fsrl_b200 import ops  # noqa: E402
from fsrl_b200.utils.synth import synth_gae_inputs  # noqa: E402


def peaks():
    p = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")
    if os.path.exists(p):
        return json.load(open(p)), "measured"
    return {"hbm_gbs": 6650.0, "bf16_tflops": 1590.0}, "fallback"


def time_kernel(fn, iters=20, warmup=5, flush=None):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.zero_()
        s = torch.cuda.Event(enable_timing=True); e = torch.cuda.Event(enable_timing=True)
        s.record(); fn(); e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    return float(np.mean(ts)), float(np.min(ts))


def bench_gae(envs, T):
    d = synth_gae_inputs(envs, T, seed=10)
    N = envs * T
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    v, vn, r, c = dev(d["v"]), dev(d["vnext"]), dev(d["rew"]), dev(d["cost"])
    end = dev((d["terminated"] | d["truncated"]).astype(np.uint8))
    term = dev(d["terminated"].astype(np.uint8))
    adv = torch.empty_like(v); ret = torch.empty_like(v)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")  # > 50 MB L2
    fn = lambda: ops.gae_dual(v, vn, r, c, end, term, 0.99, 0.95, out=(adv, ret))
    mean_ms, min_ms = time_kernel(fn, flush=flush)
    alg_bytes = N * (16 * 2 + 10)   # SURVEY.md 8(d): 16*C + 10 B / transition (+1 B terminated)
    pk, how = peaks()
    gbs = alg_bytes / (mean_ms * 1e-3) / 1e9
    print(json.dumps({"kernel": "gae_dual", "N": N, "ms_mean": mean_ms, "ms_min": min_ms,
                      "alg_bytes": alg_bytes, "GBps": gbs, "frac_of_%s_hbm" % how: gbs / pk["hbm_gbs"]}))


def bench_ppo(iters):
    import bench
    agent, trainer, col, buf, T = bench.build("cuda:0", 0)
    print(json.dumps({"phase_ms(fwd,bwd,wgrad,adam)": bench.phase_times(agent, col, buf, iters=iters)}))
    import ctypes
    from fsrl_b200 import _lib
    ck = (ctypes.c_longlong * 32)()
    _lib.check(_lib.lib.fsrl_debug_clocks(ck))
    c = list(ck)
    print("ppo_bwd CTA(0,0,0) cycles [loads, advstats, sync, head, lossgrad, stats, dz2, wait_slab, slab_gemm]:",
          [c[i + 1] - c[i] for i in range(8)], "total", c[8] - c[0])
    print("ppo_fwd CTA(0,0,0) cycles [obs load, (pdl wait), slab issue+sync, layer1, wait_slab, slab_gemm]:",
          [c[i + 1] - c[i] for i in range(16, 22)], "total", c[22] - c[16])
    cc = (ctypes.c_longlong * 512)()
    _lib.check(_lib.lib.fsrl_debug_cta_cycles(cc))
    cc = list(cc)[:120]
    print("wgrad per-CTA cycles net0 roles:", cc[:40])
    print("wgrad tile CTA cycles [stage0 issue, chunk loop, finish]:", [c[11] - c[10], c[12] - c[11], c[13] - c[12]])


def bench_fused():
    import bench, ctypes
    from fsrl_b200 import _lib
    agent, trainer, col, buf, T = bench.build("cuda:0", 0)
    bench.one_cycle(trainer)
    torch.cuda.synchronize()
    cc = (ctypes.c_longlong * 512)()
    _lib.check(_lib.lib.fsrl_debug_cta_cycles(cc))
    cc = list(cc)
    print("fused wgrad: cycles to end of role compute, net0 roles [32 tiles | 4 L1 | 4 L3]:", cc[:40])
    print("fused wgrad: cycles to barrier exit, net0:", cc[256:296])


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("what")
    ap.add_argument("--envs", type=int, default=2048)
    ap.add_argument("--T", type=int, default=300)
    a = ap.parse_args()
    if a.what == "fused":
        bench_fused()
    if a.what == "ppo":
        bench_ppo(a.T if a.T != 300 else 50)
    if a.what == "gae":
        bench_gae(a.envs, a.T)
        bench_gae(a.envs * 16, a.T)
