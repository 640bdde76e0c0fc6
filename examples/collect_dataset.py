"""Collect an offline safe-RL dataset through the REFERENCE'S import names (fsrl / tianshou / gymnasium,
resolved by ``fsrl_b200.compat`` to the device engine) -- the flow of the reference's
``examples/customized/collect_dataset.py``: a TRPO-Lagrangian agent trains while its cost limit moves
from ``cost_start`` to ``cost_end`` (``cost_limit_scheduler``), every finished trajectory whose return
and cost lie in ``[rmin, rmax] x [cmin, cmax]`` is kept in a ``TrajectoryBuffer`` (grid filter,
``filter_interval=1.5``, ``max_traj_len`` trajectories), and the buffer is saved at the end or on an
interrupt.

``--training_num 1`` trains through ``BasicCollector`` like the reference; ``--training_num N`` (N > 1)
collects with ``FastCollector(..., traj_buffer=...)`` over N device envs.  Test episodes always go
through ``BasicCollector`` and also feed the buffer.  The dataset is written as
``<logdir>/<name>/dataset.npz`` (see TrajectoryBuffer.save).

``--user_env True`` collects the dataset of a user-written gymnasium-style env instead of a registered task
(``HazardReach`` of ``examples/train_host_env.py``): ``DummyVectorEnv`` over its constructors for N > 1 and
``BasicCollector`` over one instance otherwise, both stepping it on the host while the actor, the ring and the
trajectory copies stay on the GPU.

  python examples/collect_dataset.py --task SafetyCarCircle-v0 --epoch 20 --training_num 64
  python examples/collect_dataset.py --user_env True --epoch 20 --training_num 16
"""
import ast
import os
import signal
import sys
from dataclasses import asdict, dataclass
from typing import Optional, Tuple

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import fsrl_b200.compat  # noqa: E402

fsrl_b200.compat.install()

import bullet_safety_gym  # noqa: E402,F401  (task registration side effect in the reference)
import gymnasium as gym  # noqa: E402
import torch  # noqa: E402
from tianshou.data import ReplayBuffer, VectorReplayBuffer  # noqa: E402
from tianshou.env import DummyVectorEnv, ShmemVectorEnv, SubprocVectorEnv  # noqa: E402,F401
from tianshou.utils.net.common import Net  # noqa: E402
from tianshou.utils.net.continuous import ActorProb, Critic  # noqa: E402
from torch.distributions import Independent, Normal  # noqa: E402

from fsrl.data import BasicCollector, FastCollector, TrajectoryBuffer  # noqa: E402
from fsrl.policy import TRPOLagrangian  # noqa: E402
from fsrl.trainer import OnpolicyTrainer  # noqa: E402
from fsrl.utils import DummyLogger  # noqa: E402
from fsrl.utils.exp_util import seed_all  # noqa: E402
from fsrl.utils.net.common import ActorCritic  # noqa: E402
from train_host_env import HazardReach  # noqa: E402


@dataclass
class TrainCfg:
    task: str = "SafetyCarCircle-v0"
    user_env: bool = False            # HazardReach, a user env stepped on the host, instead of `task`
    cost_start: float = 5
    cost_end: float = 100
    epoch_start: int = 100
    epoch_end: int = 900
    epoch: int = 1000
    max_traj_len: int = 1500          # trajectories the buffer keeps
    rmin: float = -9999
    rmax: float = 9999
    cmin: float = 0
    cmax: float = 300
    device: str = "cuda"
    seed: int = 10
    lr: float = 5e-4
    hidden_sizes: Tuple[int, ...] = (128, 128)
    unbounded: bool = False
    target_kl: float = 0.001
    backtrack_coeff: float = 0.8
    max_backtracks: int = 10
    optim_critic_iters: int = 20
    gae_lambda: float = 0.95
    norm_adv: bool = True
    use_lagrangian: bool = True
    lagrangian_pid: Tuple[float, ...] = (0.05, 0.005, 0.1)
    rescaling: bool = True
    gamma: float = 0.99
    max_batchsize: int = 100000
    deterministic_eval: bool = False
    action_scaling: bool = True
    action_bound_method: str = "clip"
    episode_per_collect: int = 10
    step_per_epoch: int = 10000
    repeat_per_collect: int = 4
    buffer_size: int = 100000
    worker: str = "ShmemVectorEnv"
    training_num: int = 1
    testing_num: int = 2
    batch_size: int = 99999
    verbose: bool = False
    logdir: str = "logs"
    name: Optional[str] = "trpol-dataset"


def cost_limit_scheduler(epoch, epoch_start, epoch_end, cost_start, cost_end):
    """linear from cost_start at epoch_start to cost_end at epoch_end, constant outside"""
    x = min(max(0, epoch - epoch_start), epoch_end - epoch_start)
    return cost_start - x * (cost_start - cost_end) / (epoch_end - epoch_start)


def main(argv=None):
    cfg = asdict(TrainCfg())
    it = iter(sys.argv[1:] if argv is None else argv)
    for tok in it:                                   # `--field value` overrides, like pyrallis
        key, val = tok.lstrip("-"), next(it)
        try:
            cfg[key] = ast.literal_eval(val)
        except (ValueError, SyntaxError):
            cfg[key] = val
    args = TrainCfg(**cfg)
    seed_all(args.seed)

    if args.user_env:
        def make_env(i=0):
            return HazardReach(seed=args.seed + i)
    else:
        def make_env(i=0):
            return gym.make(args.task)
    env = make_env()
    state_shape, action_shape = env.observation_space.shape, env.action_space.shape
    max_action = env.action_space.high[0]
    net = Net(state_shape, hidden_sizes=args.hidden_sizes, device=args.device)
    actor = ActorProb(net, action_shape, max_action=max_action, unbounded=args.unbounded, device=args.device)
    critic = [Critic(Net(state_shape, hidden_sizes=args.hidden_sizes, device=args.device), device=args.device)
              for _ in range(2)]
    torch.nn.init.constant_(actor.sigma_param, -0.5)
    actor_critic = ActorCritic(actor, critic)
    for m in actor_critic.modules():
        if isinstance(m, torch.nn.Linear):
            torch.nn.init.orthogonal_(m.weight)
            torch.nn.init.zeros_(m.bias)
    optim = torch.optim.Adam(actor_critic.parameters(), lr=args.lr)
    policy = TRPOLagrangian(
        actor, critic, optim, lambda *logits: Independent(Normal(*logits), 1), logger=DummyLogger(),
        target_kl=args.target_kl, backtrack_coeff=args.backtrack_coeff, max_backtracks=args.max_backtracks,
        optim_critic_iters=args.optim_critic_iters, gae_lambda=args.gae_lambda,
        advantage_normalization=args.norm_adv, use_lagrangian=args.use_lagrangian,
        lagrangian_pid=args.lagrangian_pid, cost_limit=args.cost_start, rescaling=args.rescaling, gamma=args.gamma,
        max_batchsize=args.max_batchsize, deterministic_eval=args.deterministic_eval,
        action_scaling=args.action_scaling, action_bound_method=args.action_bound_method,
        observation_space=env.observation_space, action_space=env.action_space, lr_scheduler=None)

    traj_buffer = TrajectoryBuffer(args.max_traj_len, filter_interval=1.5, rmin=args.rmin, rmax=args.rmax,
                                   cmin=args.cmin, cmax=args.cmax)
    if args.training_num == 1:
        train_collector = BasicCollector(policy, env, ReplayBuffer(args.buffer_size), traj_buffer=traj_buffer)
    else:
        worker = DummyVectorEnv if args.user_env else eval(args.worker)
        train_envs = worker([lambda i=i: make_env(i) for i in range(args.training_num)])
        train_collector = FastCollector(policy, train_envs, VectorReplayBuffer(args.buffer_size, len(train_envs)),
                                        exploration_noise=True, traj_buffer=traj_buffer)
    test_collector = BasicCollector(policy, make_env(1000), traj_buffer=traj_buffer)
    trainer = OnpolicyTrainer(
        policy=policy, train_collector=train_collector, test_collector=test_collector, max_epoch=args.epoch,
        batch_size=args.batch_size, cost_limit=args.cost_end, step_per_epoch=args.step_per_epoch,
        repeat_per_collect=args.repeat_per_collect, episode_per_test=args.testing_num,
        episode_per_collect=args.episode_per_collect, stop_fn=lambda reward, cost: False, logger=DummyLogger(),
        verbose=args.verbose, show_progress=False)

    dataset_dir = os.path.join(args.logdir, args.name)

    def saving_dataset():
        traj_buffer.save(dataset_dir)

    def term_handler(signum, frame):
        print("Sig term handler, saving the dataset...")
        saving_dataset()
        sys.exit(0)

    previous = signal.signal(signal.SIGTERM, term_handler)
    try:
        for epoch, epoch_stat, info in trainer:
            print(f"Trajs: {len(traj_buffer.buffer)}, transitions: {len(traj_buffer)}")
            cost = cost_limit_scheduler(epoch, args.epoch_start, args.epoch_end, args.cost_start, args.cost_end)
            policy.update_cost_limit(cost)
    except KeyboardInterrupt:
        print("keyboardinterrupt detected, saving the dataset...")
    finally:
        signal.signal(signal.SIGTERM, previous)
    saving_dataset()
    return traj_buffer, os.path.join(dataset_dir, "dataset.npz")


if __name__ == "__main__":
    main()
