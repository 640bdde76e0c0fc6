// HazardDash: a test env that is not in the library.  A point mass with a finite energy budget dashes to a goal
// through 12 hazards, all drawn from the reset's Philox stream.  A = 3 (thrust x, thrust y, boost), D = 19 (odd),
// S = 32 (= ENV_MAX_S).  Terminates on reaching the goal, running out of energy or leaving the arena; truncates at
// T = 200.  Exact-op arithmetic only, so tests/env_plugin_twin.py replays it bit for bit.
#include "envs.cuh"

namespace hazard_dash {
constexpr float DT = 0.1f, DAMP = 0.9f, ARENA = 2.0f, GOAL_R = 0.25f, HAZ_R = 0.3f, LIDAR = 2.0f, ECOST = 0.005f;
constexpr int NHAZ = 12;
}

struct UserEnv {
    // state: x, y, vx, vy, gx, gy, energy, steps in hazards, hazards (hx, hy) x 12
    static constexpr int D = 19, A = 3, S = 32, T = 200;

    __device__ static void reset(float* st, uint32_t seed, uint32_t env, uint32_t ep) {
        using namespace fsrl;
        using namespace hazard_dash;
        uint32_t r[4];
        Philox::gen(env, ep, 0u, 0u, seed, KEY_RESET, r);
        st[0] = xm(usym(r[0]), 0.5f);
        st[1] = xm(usym(r[1]), 0.5f);
        st[2] = 0.0f; st[3] = 0.0f;
        st[4] = xm(usym(r[2]), 1.5f);
        st[5] = xm(usym(r[3]), 1.5f);
        Philox::gen(env, ep, 1u, 0u, seed, KEY_RESET, r);
        st[6] = xa(1.0f, xm(usym(r[0]), 0.5f));   // energy in [0.5, 1.5)
        st[7] = 0.0f;
        for (int c = 0; c < NHAZ / 2; ++c) {
            Philox::gen(env, ep, 2u + (uint32_t)c, 0u, seed, KEY_RESET, r);
            for (int j = 0; j < 4; ++j) st[8 + 4 * c + j] = xm(usym(r[j]), ARENA);
        }
    }

    __device__ static void observe(const float* st, float* o, uint32_t, uint32_t, uint32_t) {
        using namespace fsrl;
        using namespace hazard_dash;
        const float x = st[0], y = st[1];
        o[0] = xd(x, ARENA); o[1] = xd(y, ARENA);
        o[2] = st[2]; o[3] = st[3];
        o[4] = xd(xs(st[4], x), ARENA); o[5] = xd(xs(st[5], y), ARENA);
        o[6] = st[6];
        for (int h = 0; h < NHAZ; ++h) {
            const float dx = xs(st[8 + 2 * h], x), dy = xs(st[9 + 2 * h], y);
            o[7 + h] = xd(fminf(xq(xa(xm(dx, dx), xm(dy, dy))), LIDAR), LIDAR);
        }
    }

    __device__ static void step(float* st, const float* a, uint32_t, uint32_t, uint32_t, float& rew, float& cost,
                                bool& term) {
        using namespace fsrl;
        using namespace hazard_dash;
        float x = st[0], y = st[1], vx = st[2], vy = st[3];
        const float gx = st[4], gy = st[5];
        const float d0 = xq(xa(xm(xs(gx, x), xs(gx, x)), xm(xs(gy, y), xs(gy, y))));
        const float k = xa(1.0f, xm(0.5f, a[2]));
        vx = xa(xm(vx, DAMP), xm(xm(a[0], k), DT));
        vy = xa(xm(vy, DAMP), xm(xm(a[1], k), DT));
        x = xa(x, xm(vx, DT));
        y = xa(y, xm(vy, DT));
        const float e = xs(st[6], xm(xa(fabsf(a[0]), fabsf(a[1])), xm(fabsf(k), ECOST)));
        const float d = xq(xa(xm(xs(gx, x), xs(gx, x)), xm(xs(gy, y), xs(gy, y))));
        cost = 0.0f;
        for (int h = 0; h < NHAZ; ++h) {
            const float dx = xs(st[8 + 2 * h], x), dy = xs(st[9 + 2 * h], y);
            if (xa(xm(dx, dx), xm(dy, dy)) < xm(HAZ_R, HAZ_R)) cost = 1.0f;
        }
        const bool goal = d < GOAL_R;
        rew = xm(xs(d0, d), 10.0f);
        if (goal) rew = xa(rew, 1.0f);
        term = goal || e <= 0.0f || fabsf(x) > ARENA || fabsf(y) > ARENA;
        st[0] = x; st[1] = y; st[2] = vx; st[3] = vy; st[6] = e;
        st[7] = xa(st[7], cost);
    }
};
