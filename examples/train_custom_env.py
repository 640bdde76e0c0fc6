"""Train PPO-Lagrangian on a device env of your own: a short C++ header defines the env, `build_device_env` compiles it
into a plugin of the library (cached: the same header never compiles twice), `register_device_env` names it, and from
then on the task steps inside the one-launch fused collect like a built-in one (DESIGN §7).

  python examples/train_custom_env.py --epoch 1
"""
import argparse
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from fsrl_b200 import envs  # noqa: E402
from fsrl_b200.agent import PPOLagAgent  # noqa: E402

# A point mass kept inside a disc of radius 1.5: the reward pays for tangential speed (circling), the cost is 1 on
# every step faster than the speed limit, and leaving the disc ends the episode.
HEADER = r'''
#include "envs.cuh"

struct UserEnv {
    static constexpr int D = 5, A = 2, S = 4, T = 200;      // obs width, action width, state size, horizon
    static constexpr float DT = 0.05f, R = 1.5f, VLIM = 0.8f;

    __device__ static void reset(float* st, uint32_t seed, uint32_t env, uint32_t ep) {
        uint32_t r[4];
        fsrl::Philox::gen(env, ep, 0u, 0u, seed, fsrl::KEY_RESET, r);   // stream (env, episode)
        st[0] = fsrl::xm(fsrl::usym(r[0]), 0.5f);
        st[1] = fsrl::xm(fsrl::usym(r[1]), 0.5f);
        st[2] = 0.0f; st[3] = 0.0f;
    }
    __device__ static void observe(const float* st, float* o, uint32_t, uint32_t, uint32_t) {
        using namespace fsrl;
        o[0] = xd(st[0], R); o[1] = xd(st[1], R); o[2] = st[2]; o[3] = st[3];
        o[4] = xd(xq(xa(xm(st[0], st[0]), xm(st[1], st[1]))), R);
    }
    __device__ static void step(float* st, const float* a, uint32_t, uint32_t, uint32_t,
                                float& rew, float& cost, bool& term) {
        using namespace fsrl;
        st[2] = xa(xm(st[2], 0.95f), xm(a[0], DT));
        st[3] = xa(xm(st[3], 0.95f), xm(a[1], DT));
        st[0] = xa(st[0], xm(st[2], DT));
        st[1] = xa(st[1], xm(st[3], DT));
        const float r2 = xa(xm(st[0], st[0]), xm(st[1], st[1]));
        const float speed2 = xa(xm(st[2], st[2]), xm(st[3], st[3]));
        rew = xs(xm(st[0], st[3]), xm(st[1], st[2]));              // x vy - y vx
        cost = speed2 > VLIM * VLIM ? 1.0f : 0.0f;
        term = r2 > R * R;
    }
};
'''


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--task", default="PointInDisc-v0")
    ap.add_argument("--epoch", type=int, default=1)
    ap.add_argument("--training_num", type=int, default=64)
    ap.add_argument("--step_per_epoch", type=int, default=20000)
    ap.add_argument("--cost_limit", type=float, default=10.0)
    ap.add_argument("--plugin_dir", default=None, help="plugin cache (default: ~/.cache/fsrl_b200/env_plugins)")
    args = ap.parse_args()

    with tempfile.TemporaryDirectory() as tmp:
        header = os.path.join(tmp, "point_in_disc.h")
        with open(header, "w") as f:
            f.write(HEADER)
        plugin = envs.build_device_env(header, out=args.plugin_dir)
    envs.register_device_env(args.task, plugin)
    print(f"{args.task}: plugin {plugin}, (D, A, S, T) = {envs.plugin_dims(plugin)}")

    agent = PPOLagAgent(envs.make(args.task), cost_limit=args.cost_limit, hidden_sizes=(64, 64), seed=1)
    train = envs.DeviceVectorEnv(args.task, args.training_num, seed=2)
    test = envs.DeviceVectorEnv(args.task, 8, seed=3)
    agent.learn(train, test, epoch=args.epoch, episode_per_collect=args.training_num, step_per_epoch=args.step_per_epoch,
                repeat_per_collect=4, buffer_size=args.training_num * 200, testing_num=8, batch_size=512,
                save_ckpt=False, verbose=False, show_progress=False)
    rew, length, cost = agent.evaluate(test, eval_episodes=8)
    print(f"after {args.epoch} epoch(s): reward {rew:.2f}, length {length:.1f}, cost {cost:.2f}")


if __name__ == "__main__":
    main()
