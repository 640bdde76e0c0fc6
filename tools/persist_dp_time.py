"""Per-phase clock stamps of one minibatch step of the persistent PPO kernel under data parallelism.
Run:  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tools/persist_dp_time.py
(config c2 of bench.py; stamps of step FSRL_PPO_PERSIST_DBG of the last repeat, rank 0's table is printed)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
from persist_check import DBG_N, N_CTA  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    device = f"cuda:{local}"
    dist.init_process_group("nccl", device_id=torch.device(device))
    cfg = bench.CONFIGS["c2"]
    agent, trainer, col, buf, T = bench.build(cfg, device, rank)
    from fsrl_b200 import parallel
    parallel.attach(agent.policy, dist, device=device)
    for _ in range(2):
        bench.one_cycle(trainer)
    torch.cuda.synchronize()
    os.environ["FSRL_PPO_PERSIST_DBG"] = "1000"
    agent.policy._persist_ws[-2 * N_CTA * DBG_N:].zero_()      # stamps a CTA does not take stay 0 and are left out below
    bench.one_cycle(trainer)
    torch.cuda.synchronize()
    del os.environ["FSRL_PPO_PERSIST_DBG"]
    ws = agent.policy._persist_ws.detach().cpu().numpy()
    dbg = ws[-2 * N_CTA * DBG_N:].view(np.int64).reshape(N_CTA, DBG_N)
    rel = dbg - dbg[:, :1]
    names = {1: "S done", 2: "G1 accumulators ready", 4: "hop B passed", 5: "dz2 + partials written", 6: "G2/G3 accumulators ready",
             7: "G2/G3 epilogue done", 8: "[reducer] dW1 partials arrived",
             17: "[reducer] W1/b1 reduced (DSMEM)", 32: "W2 tile pushed",
             41: "exchange done (W2 tile / slice: ranks' mean in)", 9: "sumsq (+ slice) out",
             10: "flag D2 passed", 11: "Adam done (step end)"}
    red = lambda i: i % 32 < 16 and (i % 32) // 8 == (i % 8) // 4      # reducers: CTAs 0-3 and 12-15 of a network
    for r in range(world):
        if r == rank:
            print("=== rank %d ===" % rank)
            for grp, sel in (("G2 reducer CTAs", [i for i in range(96) if red(i)]),
                             ("other G2 CTAs", [i for i in range(96) if i % 32 < 16 and not red(i)]),
                             ("G3 CTAs", [i for i in range(96) if i % 32 >= 16])):
                print("  --- %s: cycles since step start (mean / min / max over CTAs) ---" % grp)
                for i in names:
                    v = rel[sel, i][dbg[sel, i] != 0]
                    if len(v) == 0:
                        continue
                    print("    %2d %-40s %8.0f %8d %8d" % (i, names[i], v.mean(), v.min(), v.max()))
            cyc = (dbg[:, 29] - dbg[:, 0]) / 64.0
            ns = (dbg[:, 31] - dbg[:, 30]) / 64.0
            print("  over the next 64 steps: %.0f cycles / step, %.0f ns / step" % (cyc.mean(), ns.mean()), flush=True)
        dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
