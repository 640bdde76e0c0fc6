"""Where the time in front of the PPO update goes: the collect and the pieces of process_fn, on c2's shapes.

PPO-Lagrangian 2x256 (2 x --hidden) on SafetyCarCircle-v0 with 2048 envs, one episode each (FastCollector.collect,
the inline path).  After a warm-up collect and process_fn, each quantity is timed with CUDA events, best of --reps:

- collect: FastCollector.collect(n_episode=E), and per vector step (the collect's step count over E);
- process_fn: the whole compute_gae_returns;
- its pieces, run as compute_gae_returns runs them: end_flag (and the unfinished-index test), need / nonzero
  (which synchronises the host), the critic forward over all rows and the one over the `ends` rows for each
  critic, and gae_dual.

The card name and power limit are read in the same run.  Prints one JSON line.  FSRL_MLPFWD_TILED=1 in the
environment times the 16-row forward kernel instead of the 64-row one.

    python tools/collect_process_time.py [--envs 2048] [--reps 5] [--hidden 256] [--task SafetyCarCircle-v0]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--hidden", type=int, default=256)
    ap.add_argument("--task", default="SafetyCarCircle-v0")
    a = ap.parse_args()
    import torch
    from env_collect_time import _card
    from helpers import build_ppo
    from fsrl_b200 import ops
    assert torch.cuda.is_available(), "collect_process_time needs a GPU"
    name, plimit = _card()
    E = a.envs
    policy, venv, buf, col = build_ppo(a.task, hidden=(a.hidden, a.hidden), n_env=E)

    def ev(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), out

    res = {}

    def best(key, fn):
        t, out = ev(fn)
        res[key] = min(res.get(key, float("inf")), t)
        return out

    buf.reset()
    col.collect(n_episode=E)                                    # warm-up
    idx = buf.sample_indices(0)
    policy.process_fn(None, buf, idx)
    steps = 0
    for _ in range(a.reps):
        buf.reset()
        st = best("ms_collect", lambda: col.collect(n_episode=E))
        steps = int(st["n/st"])
        idx = buf.sample_indices(0)
        best("ms_process_fn", lambda: policy.process_fn(None, buf, idx))
        # the pieces of compute_gae_returns, in its order, on the batch it gathers
        b = policy.gather_batch(buf, idx)

        def flags():
            end_flag = b.terminated | b.truncated
            unfinished = buf.unfinished_index()
            if unfinished.numel():
                end_flag = end_flag.clone()
                end_flag[torch.isin(idx, unfinished)] = 1
            return end_flag
        end_flag = best("ms_end_flag", flags)

        def need_ends():
            need = end_flag.to(torch.bool).clone()
            need[-1] = True
            need[:-1] |= (b.obs_next[:-1] != b.obs[1:]).any(dim=1)
            return torch.nonzero(need, as_tuple=False).flatten().to(torch.int32)
        ends = best("ms_need_nonzero", need_ends)
        v = torch.empty((policy.critics_num, b.n), dtype=torch.float32, device=policy.device)
        vnext = torch.empty_like(v)
        for i in range(policy.critics_num):
            v[i] = best(f"ms_critic{i}_all_rows", lambda: policy.net_forward(1 + i, b.obs)).flatten()
            vnext[i, :-1] = v[i, 1:]
            ve = best(f"ms_critic{i}_ends", lambda: policy.net_forward(1 + i, b.obs_next, idx=ends)).flatten()
            vnext[i, ends.long()] = ve
        best("ms_gae_dual", lambda: ops.gae_dual(v, vnext, b.rew, b.cost, end_flag, b.terminated, policy._gamma, 0.95))
        res["ends_rows"] = int(ends.numel())
    res = {k: (round(v, 4) if isinstance(v, float) else v) for k, v in res.items()}
    print(json.dumps(dict(task=a.task, envs=E, hidden=a.hidden, rows=int(idx.numel()), env_steps=steps,
                          us_per_vector_step=round(res["ms_collect"] * 1e3 / (steps / E), 3),
                          mlpfwd_tiled=os.environ.get("FSRL_MLPFWD_TILED", "0"), **res, reps=a.reps, gpu=name,
                          power_limit=plimit)), flush=True)


if __name__ == "__main__":
    main()
