"""2-rank NCCL test of the data-parallel PPO update: after an update every rank must hold
bit-identical parameters (one all-reduce per optimiser step keeps them in lock-step), the
update must equal the single-process update on the UNION of the two ranks' minibatches
(global-minibatch advantage normalisation + averaged gradients), and the PID state must agree."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ppo_update(rank, dist, p2p):
    from helpers import build_ppo
    from fsrl_b200 import parallel
    policy, venv, buf, col = build_ppo("SafetyBallCircle-v0", hidden=(64, 64), n_env=4, seed=10,
                                       device=f"cuda:{rank}", max_grad_norm=0.5)
    venv.seed(parallel.shard_seed(12, rank)); col.reset_env()
    policy.set_action_seed(parallel.shard_seed(11, rank))
    dp = parallel.attach(policy, dist, device=f"cuda:{rank}", p2p=p2p)
    assert (getattr(dp, "p2p", None) is not None) == p2p
    stats = col.collect(n_episode=4)
    policy.pre_update_fn(stats_train=stats)
    idx = buf.sample_indices(0)
    batch = policy.process_fn(None, buf, idx)
    policy._target_kl = 1e9
    np.random.seed(100 + rank)
    theta0 = policy.arena.theta.clone()
    policy.learn(batch, batch_size=100, repeat=2)
    theta = policy.arena.theta.cpu().numpy()
    return (theta, policy.lagrangians()[0], float(np.mean(policy.last_stats["loss/kl"])),
            float((policy.arena.theta - theta0).abs().max().item()))


def _worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{rank}"))
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    peer = _ppo_update(rank, dist, p2p=True)        # gradients summed over peer memory (NVLink loads)
    nccl = _ppo_update(rank, dist, p2p=False)       # same data through the NCCL all-reduce fallback
    q.put((rank, peer, nccl))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_update_keeps_parameters_identical():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29600 + (os.getpid() % 1000)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted((q.get(timeout=300) for _ in range(2)), key=lambda t: t[0])
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    (_, peer0, nccl0), (_, peer1, nccl1) = res
    for (t0, lag0, kl0, d0), (t1, lag1, kl1, d1) in ((peer0, peer1), (nccl0, nccl1)):
        assert np.array_equal(t0, t1), np.abs(t0 - t1).max()       # lock-step on both exchange paths
        assert lag0 == lag1
        assert d0 > 0 and np.isfinite(t0).all()
    # peer-memory sum (rank order) vs NCCL's reduction order: same update up to fp32 rounding
    assert np.abs(peer0[0] - nccl0[0]).max() <= 1e-2 * peer0[3] + 1e-6, np.abs(peer0[0] - nccl0[0]).max()


def _persistent_update(rank, dist):
    """c2-shaped networks (2x256, batch 256) so that the persistent wgmma launch runs the update: its in-kernel
    peer-memory exchange (csrc/ppo_persist.cu) against the three-launch chain's exchange kernel on the same data."""
    import ctypes
    from helpers import build_ppo
    from fsrl_b200 import _lib, parallel
    policy, venv, buf, col = build_ppo("SafetyCarCircle-v0", hidden=(256, 256), n_env=64, seed=10,
                                       device=f"cuda:{rank}", max_grad_norm=0.5)
    venv.seed(parallel.shard_seed(12, rank)); col.reset_env()
    policy.set_action_seed(parallel.shard_seed(11, rank))
    dp = parallel.attach(policy, dist, device=f"cuda:{rank}", p2p=True)
    assert getattr(dp, "p2p", None) is not None
    stats = col.collect(n_episode=64)
    policy.pre_update_fn(stats_train=stats)
    idx = buf.sample_indices(0)
    from test_ppo_scale_gpu import _sub_batch
    full = policy.process_fn(None, buf, idx)
    batch = _sub_batch(policy, full, 8 * 256)            # 8 optimiser steps: short enough to compare element-wise
    policy._target_kl = 1e9
    policy._dp_batch = 256
    policy._ensure_update_state(256, batch.n, 1)
    u = policy._descriptor(batch, torch.zeros(batch.n, dtype=torch.int32, device=f"cuda:{rank}"))
    active = int(_lib.lib.fsrl_ppo_persist_active(ctypes.byref(u), batch.n, 256))
    start = (policy.arena.theta.clone(), policy.optim.m.clone(), policy.optim.v.clone(), policy.optim.step_count)
    out = []
    for off in (False, True):
        policy.arena.theta.copy_(start[0]); policy.optim.m.copy_(start[1]); policy.optim.v.copy_(start[2])
        policy.optim.step_count = start[3]
        policy._mirror_dirty = True
        policy._persist_off = off
        np.random.seed(200 + rank)
        policy.learn(batch, batch_size=256, repeat=1)
        torch.cuda.synchronize()
        out.append(policy.arena.theta.cpu().numpy().copy())
    moved = float(np.abs(out[0] - start[0].cpu().numpy()).max())
    return active, out[0], out[1], moved


def _worker_persistent(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{rank}"))
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    q.put((rank,) + _persistent_update(rank, dist))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("direct", ["1", "0"])
def test_two_rank_persistent_update_matches_chain_exchange(direct, monkeypatch):
    # direct = 1: W2 gradient tiles in one hop (the default for 2 ranks); 0: the two-hop owner scheme used beyond 2 ranks
    monkeypatch.setenv("FSRL_PPO_DP_DIRECT", direct)
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29700 + (os.getpid() % 1000)
    procs = [ctx.Process(target=_worker_persistent, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted((q.get(timeout=300) for _ in range(2)), key=lambda t: t[0])
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    (_, act0, pers0, chain0, moved0), (_, act1, pers1, chain1, moved1) = res
    assert act0 == 1 and act1 == 1                       # the gate selected the persistent launch on both ranks
    assert np.array_equal(pers0, pers1), np.abs(pers0 - pers1).max()      # lock-step: bit-identical parameters
    assert np.array_equal(chain0, chain1)
    assert moved0 > 0 and np.isfinite(pers0).all()
    # same global-minibatch update as the chain's exchange kernel, up to fp32 summation order (8 Adam steps)
    d = np.abs(pers0 - chain0)
    assert (d > 2e-5).mean() <= 1e-3 and d.max() <= 2 * 5e-4 * 8, (d.max(), (d > 2e-5).mean())   # (an element can move lr per step either way)


# ---------------------------------------------------------------------------------------------------
# CPO / TRPO-Lag / SAC-Lag / DDPG-Lag under data parallelism (SURVEY.md 8e)
# ---------------------------------------------------------------------------------------------------
def _build_algo(algo, device, seed=10, n_env=4):
    from fsrl_b200 import envs
    from fsrl_b200.agent import CPOAgent, DDPGLagAgent, SACLagAgent, TRPOLagAgent
    from fsrl_b200.data import FastCollector, VectorReplayBuffer
    task = "SafetyCarRun-v0" if algo in ("sac", "ddpg") else "SafetyCarCircle-v0"
    env = envs.make(task)
    hs = (64, 64)
    if algo == "cpo":
        agent = CPOAgent(env, seed=seed, hidden_sizes=hs, device=device, optim_critic_iters=3)
    elif algo == "trpo":
        agent = TRPOLagAgent(env, seed=seed, hidden_sizes=hs, device=device, optim_critic_iters=3, target_kl=0.001)
    elif algo == "sac":
        agent = SACLagAgent(env, seed=seed, hidden_sizes=hs, device=device, unbounded=True, n_step=2, tau=0.05)
    else:
        agent = DDPGLagAgent(env, seed=seed, hidden_sizes=hs, device=device, n_step=2, tau=0.05)
    venv = envs.DeviceVectorEnv(task, n_env, seed=seed + 2, device=device)
    buf = VectorReplayBuffer(n_env * env.spec.max_episode_steps, n_env, device=device)
    col = FastCollector(agent.policy, venv, buf, exploration_noise=True)
    return agent.policy, venv, buf, col


def _run_update(algo, policy, buf, col, env_seed, act_seed):
    col.env.seed(env_seed); col.reset_env()
    policy.set_action_seed(act_seed)
    stats = col.collect(n_episode=4)
    policy.pre_update_fn(stats_train=stats)
    np.random.seed(77)
    if algo in ("sac", "ddpg"):
        policy.update_many(6, 64, buf)
    else:
        idx = buf.sample_indices(0)
        batch = policy.process_fn(None, buf, idx)
        policy.learn(batch, batch_size=99999, repeat=1)
    torch.cuda.synchronize()
    return policy.arena.theta.detach().cpu().numpy().copy()


def _algo_worker(rank, world, port, q, algo, replicated):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dev = f"cuda:{rank}"
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(dev))
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from fsrl_b200 import parallel
    policy, venv, buf, col = _build_algo(algo, dev)
    theta_init = policy.arena.theta.detach().cpu().numpy().copy()
    base_upd = getattr(policy, "_upd_seed", 0)
    parallel.attach(policy, dist, device=dev)
    if replicated:
        # both ranks see IDENTICAL data and noise: the union-batch update must equal the single-GPU one
        if hasattr(policy, "_upd_seed"):
            policy._upd_seed = base_upd
        theta = _run_update(algo, policy, buf, col, 12, 11)
        ref_policy, _, rbuf, rcol = _build_algo(algo, dev)
        theta_ref = _run_update(algo, ref_policy, rbuf, rcol, 12, 11)
        q.put((rank, theta, theta_ref, theta_init))
    else:
        theta = _run_update(algo, policy, buf, col, parallel.shard_seed(12, rank), parallel.shard_seed(11, rank))
        q.put((rank, theta, None, theta_init))
    dist.barrier()
    dist.destroy_process_group()


def _spawn(algo, replicated):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29700 + (os.getpid() % 1000) + (hash((algo, replicated)) % 50)
    procs = [ctx.Process(target=_algo_worker, args=(r, 2, port, q, algo, replicated)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted((q.get(timeout=300) for _ in range(2)), key=lambda t: t[0])
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    return res


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("algo", ["cpo", "trpo", "sac", "ddpg"])
def test_two_rank_sharded_update_stays_in_lock_step(algo):
    (_, t0, _, init), (_, t1, _, _) = _spawn(algo, replicated=False)
    assert np.isfinite(t0).all()
    assert np.array_equal(t0, t1), np.abs(t0 - t1).max()      # bit-identical parameters on both ranks
    assert np.abs(t0 - init).max() > 0


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("algo", ["cpo", "trpo", "sac", "ddpg"])
def test_two_rank_replicated_data_equals_single_gpu_update(algo):
    (_, t0, ref0, init), (_, t1, _, _) = _spawn(algo, replicated=True)
    assert np.array_equal(t0, t1)
    moved = np.abs(ref0 - init).max()
    assert moved > 0
    # averaging two identical shards = the single-GPU update (only the reduction order differs)
    assert np.abs(t0 - ref0).max() <= 2e-2 * moved + 2e-6, (np.abs(t0 - ref0).max(), moved)
