"""Watch an agent on the device envs: the flow of the reference's ``examples/mlp/eval_*_agent.py`` with ``render=True``.
Build the agent for ``--task``, load ``--path`` (a checkpoint ``train_agent.py`` wrote) or keep the fresh
initialisation, step ``DeviceVectorEnv(task, --envs, render_mode="rgb_array")`` with the policy in eval mode
(deterministic actions) until every env has finished one episode, drawing a frame after every vector step, and write
``<out>.gif`` (the envs tiled into one frame) or ``<out>.npz`` (the raw frames, ``[steps][envs][H][W][3]``).

  python examples/render_agent.py --task SafetyPointButton2Gymnasium-v0 --envs 4 --out /tmp/button2
  python examples/render_agent.py --task SafetyCarCircle-v0 --path logs/.../checkpoint/model.pt --out /tmp/circle

A user-defined device env renders when its struct defines ``draw`` (DESIGN §7): ``--header`` builds the plugin of the
header, registers it as ``--task_name`` and watches the agent on it instead of ``--task``.

  python examples/render_agent.py --header my_env.h --path logs/.../checkpoint/model.pt --out /tmp/mine
"""
import argparse
import math
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from fsrl_b200 import agent as agents  # noqa: E402
from fsrl_b200 import envs  # noqa: E402
from fsrl_b200.data import Batch  # noqa: E402

ALGOS = {"ppol": agents.PPOLagAgent, "cpo": agents.CPOAgent, "trpol": agents.TRPOLagAgent,
         "focops": agents.FOCOPSAgent, "sacl": agents.SACLagAgent, "ddpgl": agents.DDPGLagAgent,
         "cvpo": agents.CVPOAgent}


def tile(frames: np.ndarray) -> np.ndarray:
    """(n, H, W, 3) -> one (rows * H, cols * W, 3) image, row-major, unused tiles black."""
    n, H, W, _ = frames.shape
    cols = math.ceil(math.sqrt(n))
    rows = math.ceil(n / cols)
    out = np.zeros((rows * H, cols * W, 3), np.uint8)
    for k in range(n):
        r, c = divmod(k, cols)
        out[r * H:(r + 1) * H, c * W:(c + 1) * W] = frames[k]
    return out


def rollout(policy, venv, max_steps=None):
    """Step every env with the policy's deterministic action until each has finished one episode (finished envs are
    reset and keep moving); returns the frames [steps][envs][H][W][3] and each env's first-episode return and cost."""
    E = len(venv)
    obs, _ = venv.reset()
    ret, cost = np.zeros(E), np.zeros(E)
    done = np.zeros(E, bool)
    frames = []
    with torch.no_grad():
        while not done.all() and (max_steps is None or len(frames) < max_steps):
            act = policy(Batch(obs=obs)).act
            act = policy.map_action(act.cpu().numpy() if isinstance(act, torch.Tensor) else np.asarray(act))
            obs, rew, term, trunc, info = venv.step(act)
            frames.append(venv.render().cpu().numpy())
            live = ~done
            ret[live] += rew.cpu().numpy()[live]
            cost[live] += info.cost.cpu().numpy()[live]
            end = (term | trunc).cpu().numpy()
            done |= end
            if end.any():
                ids = np.nonzero(end)[0]
                obs = obs.clone()
                obs[torch.from_numpy(ids).to(obs.device)] = venv.reset(ids)[0]
    return np.stack(frames), ret, cost, done


def write(frames, out, fmt, fps):
    """<out>.gif through PIL (one frame per vector step; PIL merges identical consecutive frames into one longer
    frame), else <out>.npz of the raw frames.  Returns the path written."""
    if fmt == "gif":
        try:
            from PIL import Image
        except ImportError:
            print("PIL is not installed: writing .npz")
            fmt = "npz"
    if fmt == "npz":
        path = out + ".npz"
        np.savez_compressed(path, frames=frames)
        return path
    path = out + ".gif"
    images = [Image.fromarray(tile(f)) for f in frames]
    images[0].save(path, save_all=True, append_images=images[1:], duration=round(1000 / fps), loop=0)
    return path


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--task", default="SafetyCarCircle-v0", choices=sorted(envs.KINDS))
    ap.add_argument("--header", default=None, help="a header defining UserEnv with draw: render its plugin, not --task")
    ap.add_argument("--task_name", default=None, help="the task name of the --header plugin (default: <stem>-v0)")
    ap.add_argument("--plugin_dir", default=None, help="where --header's plugin is built and cached "
                                                       "(default: build_device_env's)")
    ap.add_argument("--algo", default="ppol", choices=sorted(ALGOS))
    ap.add_argument("--hidden_sizes", type=int, nargs="+", default=[128, 128])
    ap.add_argument("--path", default=None, help="checkpoint written by train_agent.py ({'model': state_dict, ...})")
    ap.add_argument("--envs", type=int, default=4)
    ap.add_argument("--size", type=int, nargs=2, default=[256, 256], metavar=("HEIGHT", "WIDTH"))
    ap.add_argument("--out", default="render")
    ap.add_argument("--format", default="gif", choices=["gif", "npz"])
    ap.add_argument("--fps", type=float, default=20.0)
    ap.add_argument("--max_steps", type=int, default=None, help="stop after this many vector steps")
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args(argv)

    task = args.task
    if args.header is not None:
        task = args.task_name or os.path.splitext(os.path.basename(args.header))[0] + "-v0"
        envs.register_device_env(task, envs.build_device_env(args.header, out=args.plugin_dir))
    demo_env = envs.make(task)
    agent = ALGOS[args.algo](env=demo_env, hidden_sizes=tuple(args.hidden_sizes), seed=args.seed)
    policy = agent.policy
    venv = envs.DeviceVectorEnv(task, args.envs, seed=args.seed, render_mode="rgb_array",
                                render_size=tuple(args.size))
    if args.path is not None:
        ckpt = torch.load(args.path, map_location="cuda")
        policy.load_state_dict(ckpt["model"])
        if "obs_rms" in ckpt:           # trained behind VectorEnvNormObs: normalize with its statistics, frozen
            venv = envs.VectorEnvNormObs(venv, update_obs_rms=False)
            rms = envs.ObsRunningMeanStd(demo_env.observation_space.shape[0])
            rms.load_state_dict(ckpt["obs_rms"])
            venv.set_obs_rms(rms)
    policy.eval()
    frames, ret, cost, done = rollout(policy, venv, args.max_steps)
    path = write(frames, args.out, args.format, args.fps)
    print(f"frames: {len(frames)} ({frames.shape[1]} envs, {frames.shape[2]} x {frames.shape[3]}) -> {path}")
    for e in range(len(ret)):
        print(f"env {e}: return {ret[e]:.2f} cost {cost[e]:.1f}" + ("" if done[e] else " (episode unfinished)"))
    print(f"mean return {ret.mean():.2f} cost {cost.mean():.2f}")


if __name__ == "__main__":
    main()
