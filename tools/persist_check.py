"""Bring-up / regression check of the persistent wgmma PPO path (csrc/ppo_persist.cu) on an H100:

1. ONE minibatch step: decode the operand images the kernel leaves in its workspace (h1 in both
   orientations, the W2 images) and the small-parameter gradient partials, compare them with a torch
   fp64 evaluation of the same minibatch, and compare parameters / Adam moments after the step with the
   three-launch chain (csrc/ppo.cu) and with the fp32 oracle;
2. a 75-step epoch (64 envs x 300 steps): per-step statistics and final parameters, persistent vs chain;
3. timing of both paths on the c2-shaped batch when --time is given.  The per-chunk table of the GEMM phases needs a
   library built with the chunk stamps:
       touch fsrl_b200/csrc/ppo_persist.cu && make -C fsrl_b200/csrc EXTRA_NVCCFLAGS=-DFSRL_PPO_CHUNK_STAMPS

Usage: python tools/persist_check.py [--time]"""
import copy
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from helpers import build_ppo, oracle_nets  # noqa: E402
from test_ppo_scale_gpu import _adam, _collect, _sub_batch  # noqa: E402

IMG = 65536
N_CTA = 96              # 32 CTAs per network, 3 networks
DBG_N = 96              # clock stamps per CTA: pp::DBG_N in csrc/ppo_persist.cu
DBG_CH, NCH = 48, 8     # first per-chunk stamp (pp::DBG_CH), chunks per GEMM phase (pp::NCH)
NAMES = ["H1A_HI", "H1A_LO", "H1T_HI", "H1T_LO", "DZA_HI", "DZA_LO", "DZT_HI", "DZT_LO", "W2A_HI", "W2A_LO", "W2B_HI", "W2B_LO"]


def dec_rows(img):      # [blk 4][plane 64][row 64][4] -> X[64 blk + row][4 plane + i]
    return img.reshape(4, 64, 64, 4).transpose(0, 2, 1, 3).reshape(256, 256)


def dec_w2a(img):       # [ob32 8][plane 64][o 32][4] -> w2t[k = 4 plane + i][o]
    return img.reshape(8, 64, 32, 4).transpose(1, 3, 0, 2).reshape(256, 256)


def state(policy):
    return (policy.arena.theta.clone(), policy.optim.m.clone(), policy.optim.v.clone(), policy.optim.step_count)


def restore(policy, st):
    policy.arena.theta.copy_(st[0]); policy.optim.m.copy_(st[1]); policy.optim.v.copy_(st[2]); policy.optim.step_count = st[3]
    policy._mirror_dirty = True


def run(policy, batch, bs, persist, seed=3):
    policy._persist_off = not persist
    policy._target_kl = 1e9
    np.random.seed(seed)
    policy.learn(batch, batch_size=bs, repeat=1)
    torch.cuda.synchronize()
    return {k: np.asarray(v).copy() for k, v in policy.last_stats.items()}


def chunk_report(dbg, red):
    """Per chunk of each GEMM phase (stamps DBG_CH ..): when the producer's bar_empty wait returned, when it had issued
    the chunk's copies and when warpgroup 0's bar_full wait returned (the chunk landed), in cycles since the phase's
    flag passed (stamp 12 / 14); issue -> land latency, the period between landings and, by Little's law, the bytes in
    flight (latency / period chunks of the phase's chunk size)."""
    rel = dbg - dbg[:, :1]
    for g, (name, flag, chunk_kb) in enumerate((("G1", 12, 24), ("G2 / G3", 14, 32))):
        base = DBG_CH + 3 * NCH * g
        for grp, sel in (("G2 reducer CTAs", [i for i in range(N_CTA) if red(i)]),
                         ("other G2 CTAs", [i for i in range(N_CTA) if i % 32 < 16 and not red(i)]),
                         ("G3 CTAs", [i for i in range(N_CTA) if i % 32 >= 16])):
            sel = [i for i in sel if dbg[i, base:base + 3 * NCH].all() and dbg[i, flag] != 0]
            if not sel:
                print("  (no per-chunk stamps: build with EXTRA_NVCCFLAGS=-DFSRL_PPO_CHUNK_STAMPS for the %s table)" % name)
                return
            t0 = rel[sel, flag][:, None]
            emp, iss, land = (rel[sel, base + e * NCH: base + (e + 1) * NCH] - t0 for e in range(3))
            lat = land - iss
            per = np.diff(land, axis=1)
            print("  --- %s chunks, %s (%d CTAs): cycles since the flag passed (means) ---" % (name, grp, len(sel)))
            print("     chunk   empty ok   issued   landed   issue->land   period")
            for j in range(NCH):
                print("    %5d %10.0f %8.0f %8.0f %13.0f %8s" % (j, emp[:, j].mean(), iss[:, j].mean(), land[:, j].mean(),
                                                                 lat[:, j].mean(), "%.0f" % per[:, j - 1].mean() if j else "-"))
            l_m, p_m = lat.mean(), per.mean()
            print("    %s: latency %.0f cycles (chunk min %.0f / max %.0f), period %.0f cycles, window flag -> last land %.0f "
                  "cycles, in flight latency / period = %.2f chunks = %.0f KB -> %.1f B/clk" % (
                      name, l_m, lat.mean(axis=0).min(), lat.mean(axis=0).max(), p_m, land[:, -1].mean(), l_m / p_m,
                      l_m / p_m * chunk_kb, chunk_kb * 1024 / p_m))


def main():
    lag = 0.3
    policy, batch, ob, actor, critics = _collect("SafetyCarCircle-v0", (256, 256), 64, lag)
    n = batch.n
    print("rows", n)
    policy._ensure_update_state(256, n, 1)
    # ---------------- 1. one step ---------------------------------------------------------------------
    sub = _sub_batch(policy, batch, 256)
    st0 = state(policy)
    sd0 = copy.deepcopy(policy.state_dict())
    s_old = run(policy, sub, 256, False)
    old = state(policy)
    restore(policy, st0)
    s_new = run(policy, sub, 256, True)
    new = state(policy)
    for k in s_old:
        print("  stat %-20s chain %+.6e persistent %+.6e" % (k, s_old[k][0], s_new[k][0]))
    print("  step 1: max |theta diff| %.3e   max |m diff| %.3e (|m| max %.3e)   max |v diff| %.3e (|v| max %.3e)" % (
        (old[0] - new[0]).abs().max().item(), (old[1] - new[1]).abs().max().item(), old[1].abs().max().item(),
        (old[2] - new[2]).abs().max().item(), old[2].abs().max().item()))
    # where do the parameters differ?
    for i, s in enumerate(policy.arena.slots):
        w1, b1, w2, b2, w3, b3, ex = s.offsets()
        ends = [("W1", w1, b1), ("b1", b1, w2), ("W2", w2, b2), ("b2", b2, w3), ("W3", w3, b3), ("b3", b3, ex), ("ex", ex, ex + s.n_extra)]
        for name, lo, hi in ends:
            if hi > lo:
                dm = (old[1][lo:hi] - new[1][lo:hi]).abs().max().item()
                mm = old[1][lo:hi].abs().max().item()
                print("    net %d %-3s max |m diff| %.3e of %.3e" % (i, name, dm, mm))
    # decode the images (they hold the operands of the LAST step = the only step)
    ws = policy._persist_ws.detach().cpu().numpy()
    from fsrl_b200 import _lib as _fl
    lib_net_ws = int(_fl.lib.fsrl_ppo_persist_ws_floats(2, 8, 256)) - int(_fl.lib.fsrl_ppo_persist_ws_floats(1, 8, 256)) - 2 * 32 - 2 * 32 * DBG_N   # minus one network's flag lines (A, C) and stamp rows
    x = sub.obs.cpu().double().numpy()
    perm = None
    for net in range(3):
        base = net * lib_net_ws
        im = {nm: ws[base + i * IMG: base + (i + 1) * IMG] for i, nm in enumerate(NAMES)}
        pre = "actor." if net == 0 else "critics.%d." % (net - 1)
        W1 = sd0[pre + "preprocess.model.model.0.weight"].cpu().double().numpy(); b1 = sd0[pre + "preprocess.model.model.0.bias"].cpu().double().numpy()
        W2 = sd0[pre + "preprocess.model.model.2.weight"].cpu().double().numpy()
        # the gathered minibatch is a permutation of the rows: compare as sets of rows via sorting by first column
        h1a = dec_rows(im["H1A_HI"]).astype(np.float64) + dec_rows(im["H1A_LO"])
        h1t = (dec_rows(im["H1T_HI"]).astype(np.float64) + dec_rows(im["H1T_LO"])).T
        w2a = dec_w2a(im["W2A_HI"]).astype(np.float64) + dec_w2a(im["W2A_LO"])
        w2b = (dec_rows(im["W2B_HI"]).astype(np.float64) + dec_rows(im["W2B_LO"]))
        print("  net %d: |h1A - h1T| %.3e   |W2A - W2t| %.3e   |W2B - W2t| %.3e" % (
            net, np.abs(h1a - h1t).max(), np.abs(w2a - W2.T).max(), np.abs(w2b - W2.T).max()))
        # h1 of the gathered rows: the gather buffer holds obs in permuted order
        g = policy._gather.detach().cpu().numpy()
        xg = g[:256 * x.shape[1]].reshape(256, x.shape[1]).astype(np.float64)
        h1_ref = np.maximum(xg @ W1.T + b1, 0.0)
        print("         |h1A - relu(x W1 + b1)| %.3e (max |h1| %.2f)" % (np.abs(h1a - h1_ref).max(), np.abs(h1_ref).max()))
    # against the fp32 oracle
    from oracle import ppo as oppo
    a1, c1 = copy.deepcopy(actor), copy.deepcopy(critics)
    osub = {k: v[:256].copy() for k, v in ob.items()}
    np.random.seed(3)
    os_ = oppo.learn(a1, c1, _adam(a1, c1), osub, 256, 1, lag, max_grad_norm=0.5, target_kl=1e9)
    for k in ("loss/actor_rew", "loss/actor_safety", "loss/vf0", "loss/vf1", "loss/kl", "loss/grad_norm"):
        print("  oracle %-20s %+.6e   persistent %+.6e   chain %+.6e" % (k, os_[0][k], s_new[k][0], s_old[k][0]))

    # ---------------- 2. a 75-step epoch ----------------------------------------------------------------
    restore(policy, st0)
    s_old = run(policy, batch, 256, False, seed=4)
    old = state(policy)
    restore(policy, st0)
    s_new = run(policy, batch, 256, True, seed=4)
    new = state(policy)
    for k in ("loss/actor_rew", "loss/actor_safety", "loss/vf0", "loss/vf1", "loss/kl", "loss/grad_norm"):
        d = np.abs(s_old[k] - s_new[k]) / (np.abs(s_old[k]) + 1e-6)
        print("  epoch %-20s max rel diff first 8: %.2e   all %d: %.2e" % (k, d[:8].max(), len(d), d.max()))
    print("  epoch: max |theta diff| %.3e" % (old[0] - new[0]).abs().max().item())

    if "--time" in sys.argv:
        policy2, batch2, _, _, _ = _collect("SafetyCarCircle-v0", (256, 256), 2048, lag)
        for persist in (False, True):
            run(policy2, batch2, 256, persist, seed=5)
            t0 = time.time()
            for _ in range(3):
                run(policy2, batch2, 256, persist, seed=5)
            dt = (time.time() - t0) / 3
            print("  c2 epoch (2400 steps) %s: %.1f ms -> %.2f us / step" % ("persistent" if persist else "chain", dt * 1e3, dt * 1e6 / 2400))
        # per-phase clock stamps of one step in the middle of the epoch (FSRL_PPO_PERSIST_DBG=<step>)
        os.environ["FSRL_PPO_PERSIST_DBG"] = "1000"
        policy2._persist_ws[-2 * N_CTA * DBG_N:].zero_()          # stamps a CTA does not take stay 0 and are left out below
        run(policy2, batch2, 256, True, seed=5)
        del os.environ["FSRL_PPO_PERSIST_DBG"]
        ws = policy2._persist_ws.detach().cpu().numpy()
        dbg = ws[-2 * N_CTA * DBG_N:].view(np.int64).reshape(N_CTA, DBG_N)
        names = {1: "S done (h1 tile + W2 images)", 2: "G1 accumulators ready", 3: "head partial written", 4: "hop B passed",
                 5: "dz2 + partials written", 6: "G2/G3 accumulators ready", 7: "G2/G3 epilogue done",
                 8: "[reducer] dW1 partials arrived", 9: "sumsq (+ slice) out", 10: "flag D2 passed",
                 11: "Adam done (step end)", 12: "[producer] flag A passed", 13: "[producer] G1 copies issued",
                 14: "[producer] flag C passed", 15: "[reducer wg1] flag C passed", 16: "[reducer wg1] b2/W3/b3 reduced",
                 17: "[reducer] W1/b1 reduced (DSMEM)", 18: "[G2] next step's h1 rows landed", 22: "G2: mask applied", 23: "G2: dW1 partial in smem",
                 24: "norm known (+ slice read)", 25: "small slices stepped", 26: "head gathered, loss gradient",
                 27: "dz2 images stored", 28: "partial sums exchanged"}
        rel = dbg - dbg[:, :1]
        red = lambda i: i % 32 < 16 and (i % 32) // 8 == (i % 8) // 4      # reducers: CTAs 0-3 and 12-15 of a network
        for grp, sel in (("G2 reducer CTAs", [i for i in range(96) if red(i)]),
                         ("other G2 CTAs", [i for i in range(96) if i % 32 < 16 and not red(i)]),
                         ("G3 CTAs", [i for i in range(96) if i % 32 >= 16])):
            print("  --- %s: cycles since step start (mean / min / max over CTAs) ---" % grp)
            for i in sorted(names):
                v = rel[sel, i][dbg[sel, i] != 0]
                if len(v):
                    print("    %2d %-34s %8.0f %8d %8d" % (i, names[i], v.mean(), v.min(), v.max()))
        for net in range(3):
            sel = list(range(32 * net, 32 * net + 32))
            s9 = [i for i in sel if dbg[i, 9] != 0]
            print("  net %d: dz2 done %6.0f  sumsq out %6.0f  step end %6.0f (mean cycles since step start)" % (
                net, rel[sel, 5].mean(), rel[s9, 9].mean(), rel[sel, 11].mean()))
            print("         G1 ready %6.0f | head out %6.0f | B passed %6.0f | loss %6.0f | images %6.0f | sums %6.0f | C arrive %6.0f" % tuple(
                rel[sel, i].mean() for i in (2, 3, 4, 26, 27, 28, 5)))
            b0 = [i for i in sel if i % 8 == 0]
            print("         (b == 0 CTAs)        B passed %6.0f | loss %6.0f | images %6.0f | sums %6.0f | C arrive %6.0f" % tuple(
                rel[b0, i].mean() for i in (4, 26, 27, 28, 5)))
        chunk_report(dbg, red)
        gt = dbg[:, 30]
        print("  step start skew across CTAs (globaltimer ns): %d" % (gt.max() - gt.min()))
        cyc = (dbg[:, 29] - dbg[:, 0]) / 64.0
        ns = (dbg[:, 31] - dbg[:, 30]) / 64.0
        print("  over the next 64 steps: %.0f cycles / step, %.0f ns / step -> SM clock %.0f MHz" % (cyc.mean(), ns.mean(), 1e3 * cyc.mean() / ns.mean()))


if __name__ == "__main__":
    main()
