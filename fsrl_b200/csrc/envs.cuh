// Batched on-device safe-RL environments (the "env.step" the reference delegates to
// pybullet / mujoco worker processes: fsrl/data/fast_collector.py:286, tianshou vector envs).
//
// The reference's physics engines are absent and irreproducible (SURVEY.md F5), so these are
// OUR documented analytic models with the task structure of Bullet-Safety-Gym's Circle / Run
// tasks and Safety-Gymnasium's Point / Car Circle, Goal, Button and Push tasks and its velocity tasks (dense
// reward, binary cost, fixed horizon; the Drone tasks also terminate on a crash or a flip, Hopper, Walker2d and
// Ant on an unhealthy pose, every other task is truncation only).  Every arithmetic step
// uses only IEEE-exact operations (+ - * / sqrt, no FMA contraction, polynomial sin/cos), so
// the CPU twin in oracle/envs.py reproduces trajectories BIT-EXACTLY from the same actions.
//
// State lives in registers of the thread that owns the env; SoA [S][E] in HBM between steps.
// step() and observe() also receive the env's Philox key (seed, env, episode), so a model may
// regenerate data drawn at reset instead of storing it (the Goal2 layouts).
#pragma once
#include "common.cuh"

namespace fsrl {

// Kinds 0-8 are the Bullet-Safety-Gym tasks and PointGoal1; the Safety-Gymnasium navigation family
// starts at 16, its velocity family at 33.  Ids 9-15, 23 and 32 are unassigned.
enum EnvKind { ENV_CAR_CIRCLE = 0, ENV_CAR_RUN = 1, ENV_BALL_CIRCLE = 2, ENV_BALL_RUN = 3,
               ENV_ANT_CIRCLE = 4, ENV_POINT_GOAL = 5, ENV_ANT_RUN = 6, ENV_DRONE_CIRCLE = 7,
               ENV_DRONE_RUN = 8, ENV_POINT_CIRCLE1 = 16, ENV_POINT_CIRCLE2 = 17, ENV_CAR_CIRCLE1 = 18,
               ENV_CAR_CIRCLE2 = 19, ENV_POINT_GOAL2 = 20, ENV_CAR_GOAL1 = 21, ENV_CAR_GOAL2 = 22,
               ENV_POINT_BUTTON1 = 24, ENV_POINT_BUTTON2 = 25, ENV_CAR_BUTTON1 = 26, ENV_CAR_BUTTON2 = 27,
               ENV_POINT_PUSH1 = 28, ENV_POINT_PUSH2 = 29, ENV_CAR_PUSH1 = 30, ENV_CAR_PUSH2 = 31,
               ENV_HALF_CHEETAH_VEL = 33, ENV_HOPPER_VEL = 34, ENV_SWIMMER_VEL = 35, ENV_WALKER2D_VEL = 36,
               ENV_ANT_VEL = 37 };

// The built-in kinds, X(K) for each, in the three groups whose launchers compile in translation units of their own:
// rollout.cu, rollout_bp.cu (Button, Push) and rollout_vel.cu (velocity).  One file for all of them would make the
// library's build well over a third slower (DESIGN §5).
#define ENV_KINDS_CORE(X)                                                                                              \
    X(ENV_CAR_CIRCLE) X(ENV_CAR_RUN) X(ENV_BALL_CIRCLE) X(ENV_BALL_RUN) X(ENV_ANT_CIRCLE) X(ENV_POINT_GOAL)           \
    X(ENV_ANT_RUN) X(ENV_DRONE_CIRCLE) X(ENV_DRONE_RUN) X(ENV_POINT_CIRCLE1) X(ENV_POINT_CIRCLE2) X(ENV_CAR_CIRCLE1) \
    X(ENV_CAR_CIRCLE2) X(ENV_POINT_GOAL2) X(ENV_CAR_GOAL1) X(ENV_CAR_GOAL2)
#define ENV_KINDS_BP(X)                                                                                                \
    X(ENV_POINT_BUTTON1) X(ENV_POINT_BUTTON2) X(ENV_CAR_BUTTON1) X(ENV_CAR_BUTTON2) X(ENV_POINT_PUSH1)                \
    X(ENV_POINT_PUSH2) X(ENV_CAR_PUSH1) X(ENV_CAR_PUSH2)
#define ENV_KINDS_VEL(X) X(ENV_HALF_CHEETAH_VEL) X(ENV_HOPPER_VEL) X(ENV_SWIMMER_VEL) X(ENV_WALKER2D_VEL) X(ENV_ANT_VEL)
#define ENV_KINDS(X) ENV_KINDS_CORE(X) ENV_KINDS_BP(X) ENV_KINDS_VEL(X)

constexpr int ENV_MAX_A = 8;
constexpr int ENV_MAX_S = 32;

// exact-op helpers (never contracted into FMA)
__device__ __forceinline__ float xm(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float xa(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float xs(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float xd(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float xq(float a) { return __fsqrt_rn(a); }

// map_action (base_policy.py:244-256): the policy's action -> what the env receives.  Bound to
// [-1, 1] by clipping or tanh (bound = FSRL_BOUND_*), then stretch onto [lo, hi].  The rollout
// kernel steps the env with it and the trajectory copy stores it, so both must call this one.
__device__ __forceinline__ float map_action(float v, int bound, int scaling, float lo, float hi) {
    if (bound == 1) v = fminf(1.0f, fmaxf(-1.0f, v));
    else if (bound == 2) v = tanhf(v);
    if (scaling) v = xa(lo, xd(xm(xs(hi, lo), xa(v, 1.0f)), 2.0f));
    return v;
}

// rotate the unit heading (c, s) by a small angle d with polynomial sin/cos, renormalise
__device__ __forceinline__ void rotate_heading(float& c, float& s, float d) {
    const float d2 = xm(d, d);
    // sn = d * (1 - d2/6 * (1 - d2/20));  cs = 1 - d2/2 * (1 - d2/12 * (1 - d2/30))
    const float sn = xm(d, xs(1.0f, xm(xd(d2, 6.0f), xs(1.0f, xd(d2, 20.0f)))));
    const float cs = xs(1.0f, xm(xd(d2, 2.0f), xs(1.0f, xm(xd(d2, 12.0f), xs(1.0f, xd(d2, 30.0f))))));
    const float c2 = xs(xm(c, cs), xm(s, sn));
    const float s2 = xa(xm(s, cs), xm(c, sn));
    const float n = xq(xa(xm(c2, c2), xm(s2, s2)));
    c = xd(c2, n);
    s = xd(s2, n);
}

// uniform in [-1, 1): 2*u - 1 with u = (x >> 8) * 2^-24  (exact)
__device__ __forceinline__ float usym(uint32_t x) {
    return xs(xm((float)(x >> 8), 2.0f / 16777216.0f), 1.0f);
}

constexpr uint32_t KEY_RESET = 0x52534554u;  // 'RSET'
constexpr uint32_t KEY_ACT = 0x4143544Eu;    // 'ACTN'
constexpr uint32_t KEY_GOAL = 0x474F414Cu;   // 'GOAL'

// ---- model constants (mirrored in oracle/envs.py) -------------------------------------------
namespace carc {
constexpr float DT = 0.05f, R = 1.5f, XLIM = 1.125f, VMAX = 1.5f, WMAX = 3.0f, AV = 0.2f, AW = 0.3f;
}
namespace carr {
constexpr float DT = 0.05f, YLIM = 0.6f, VLIM = 1.2f, VMAX = 1.5f, WMAX = 3.0f, AV = 0.2f, AW = 0.3f, RSCALE = 2.0f;
}
namespace ball {
constexpr float DT = 0.05f, R = 1.5f, XLIM = 1.125f, ACC = 4.0f, DRAG = 2.0f, YLIM = 0.6f, VLIM = 1.5f, RSCALE = 2.5f;
}
namespace ant {
constexpr float DT = 0.05f, R = 3.0f, XLIM = 2.25f, VMAX = 2.0f, WMAX = 2.0f, AV = 0.1f, AW = 0.15f;
constexpr float KA = 20.0f, KQ = 10.0f, KD = 4.0f;
}
namespace antr {
constexpr float YLIM = 1.0f, VLIM = 0.8f, RSCALE = 1.0f;
}
namespace drone {
constexpr float DT = 0.05f, G = 9.8f, TM = 4.9f, KM = 0.3f, KT = 20.0f, KP = 25.0f, KD = 6.0f;
constexpr float KY = 4.0f, KDY = 2.0f, DRAG = 0.5f, Z0 = 1.0f, FLIP = 0.8f;
constexpr float R = 1.5f, XLIM = 1.125f, YLIM = 0.6f, VLIM = 1.0f, RSCALE = 1.0f;
}
namespace pgoal {
constexpr float DT = 0.05f, VMAX = 1.0f, WMAX = 3.0f, AV = 0.2f, AW = 0.3f, ARENA = 2.0f;
constexpr float GOAL_R = 0.3f, HAZ_R = 0.2f, LIDAR_MAX = 3.0f;
constexpr int NHAZ = 8, NBIN = 16;
}
namespace nav {   // the Safety-Gymnasium family beyond PointGoal1 (the Point body uses pgoal's constants)
constexpr float CAR_VW = 1.0f, CAR_AL = 0.2f, TRACK = 0.5f;    // Car: top wheel speed, wheel lag, track width
constexpr float CIRC_R = 1.5f, WALL = 1.125f, START = 0.8f;    // Circle: circle radius, walls, reset box
constexpr float VASE_R = 0.25f;                                // Goal2: robot-vase contact distance
}
namespace button {   // Button1 / Button2; hazards use pgoal::HAZ_R
constexpr float BUTTON_R = 0.2f, GREM_R = 0.2f;     // robot-button and robot-gremlin contact distances
constexpr float GREM_W = 1.0f, GREM_TRAVEL = 0.35f; // gremlin orbit: angular speed (rad/s) and radius
constexpr int DELAY = 10;                           // steps the buttons stay hidden and inert after a press
}
namespace push {     // Push1 / Push2; the goal uses pgoal::GOAL_R
constexpr float PUSH_D = 0.3f;                      // robot-box centre distance on contact (robot + box radius)
constexpr float HAZ_R = 0.3f, PILLAR_R = 0.4f;      // robot-hazard and robot-pillar contact distances
constexpr float BOX_START = 1.0f;                   // the box starts in [-BOX_START, BOX_START]^2
}

struct EnvDims { int D, A, S, T; };

// host: the widths of a built-in kind or of a registered plugin kind, from its launcher table (rollout.cu); false for
// an unknown kind
bool env_kind_dims(int kind, EnvDims& d);

// ---------------------------------------------------------------------------------------------
// Car (unicycle with first-order actuator lag).  state: x, y, c, s, v, w [, x0 (run)]
// ---------------------------------------------------------------------------------------------
template <int KIND>
struct Env;

__device__ __forceinline__ void heading_from_box(float a, float b, float& c, float& s) {
    // direction of a uniform point of the square (documented: not a uniform angle)
    float n2 = xa(xm(a, a), xm(b, b));
    if (n2 < 1e-12f) { c = 1.0f; s = 0.0f; return; }
    const float n = xq(n2);
    c = xd(a, n);
    s = xd(b, n);
}

__device__ __forceinline__ void car_advance(float* st, float a0, float a1, float vmax, float wmax,
                                            float av, float aw, float dt) {
    float x = st[0], y = st[1], c = st[2], s = st[3], v = st[4], w = st[5];
    v = xa(v, xm(xs(xm(a0, vmax), v), av));
    w = xa(w, xm(xs(xm(a1, wmax), w), aw));
    rotate_heading(c, s, xm(w, dt));
    x = xa(x, xm(xm(v, c), dt));
    y = xa(y, xm(xm(v, s), dt));
    st[0] = x; st[1] = y; st[2] = c; st[3] = s; st[4] = v; st[5] = w;
}

template <>
struct Env<ENV_CAR_CIRCLE> {
    static constexpr int D = 8, A = 2, S = 6, T = 300;
    __device__ static void reset(float* st, uint32_t seed, uint32_t env, uint32_t ep) {
        uint32_t r[4];
        Philox::gen(env, ep, 0u, 0u, seed, KEY_RESET, r);
        st[0] = xm(usym(r[0]), 0.3f);
        st[1] = xm(usym(r[1]), 0.3f);
        heading_from_box(usym(r[2]), usym(r[3]), st[2], st[3]);
        st[4] = 0.0f; st[5] = 0.0f;
    }
    __device__ static void observe(const float* st, float* o, uint32_t, uint32_t, uint32_t) {
        using namespace carc;
        const float x = st[0], y = st[1], c = st[2], s = st[3], v = st[4], w = st[5];
        const float r = xq(xa(xm(x, x), xm(y, y)));
        o[0] = xd(x, R); o[1] = xd(y, R); o[2] = xm(v, c); o[3] = xm(v, s);
        o[4] = c; o[5] = s; o[6] = xd(w, WMAX); o[7] = xd(xs(r, R), R);
    }
    __device__ static void step(float* st, const float* a, uint32_t, uint32_t, uint32_t,
                                float& rew, float& cost, bool& term) {
        using namespace carc;
        car_advance(st, a[0], a[1], VMAX, WMAX, AV, AW, DT);
        const float x = st[0], y = st[1], vx = xm(st[4], st[2]), vy = xm(st[4], st[3]);
        const float r = xq(xa(xm(x, x), xm(y, y)));
        // reward = (x*vy - y*vx) / (R * (1 + |r - R|))
        rew = xd(xs(xm(x, vy), xm(y, vx)), xm(R, xa(1.0f, fabsf(xs(r, R)))));
        cost = (fabsf(x) > XLIM) ? 1.0f : 0.0f;
        term = false;
    }
};

template <>
struct Env<ENV_CAR_RUN> {
    static constexpr int D = 7, A = 2, S = 7, T = 200;
    __device__ static void reset(float* st, uint32_t seed, uint32_t env, uint32_t ep) {
        uint32_t r[4];
        Philox::gen(env, ep, 0u, 0u, seed, KEY_RESET, r);
        st[0] = 0.0f;
        st[1] = xm(usym(r[0]), 0.2f);
        heading_from_box(1.0f, xm(usym(r[1]), 0.3f), st[2], st[3]);
        st[4] = 0.0f; st[5] = 0.0f; st[6] = 0.0f;
    }
    __device__ static void observe(const float* st, float* o, uint32_t, uint32_t, uint32_t) {
        using namespace carr;
        o[0] = st[1]; o[1] = xm(st[4], st[2]); o[2] = xm(st[4], st[3]); o[3] = st[2]; o[4] = st[3];
        o[5] = xd(st[5], WMAX); o[6] = xd(st[4], VLIM);
    }
    __device__ static void step(float* st, const float* a, uint32_t, uint32_t, uint32_t,
                                float& rew, float& cost, bool& term) {
        using namespace carr;
        const float x_old = st[0];
        car_advance(st, a[0], a[1], VMAX, WMAX, AV, AW, DT);
        rew = xm(xd(xs(st[0], x_old), DT), RSCALE);
        cost = (fabsf(st[1]) > YLIM || st[4] > VLIM) ? 1.0f : 0.0f;
        st[6] = xa(st[6], cost);
        term = false;
    }
};

// ---------------------------------------------------------------------------------------------
// Ball (force-controlled point mass with linear drag).  state: x, y, vx, vy [, x0]
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void ball_advance(float* st, float a0, float a1) {
    using namespace ball;
    float x = st[0], y = st[1], vx = st[2], vy = st[3];
    vx = xa(vx, xm(xs(xm(a0, ACC), xm(DRAG, vx)), DT));
    vy = xa(vy, xm(xs(xm(a1, ACC), xm(DRAG, vy)), DT));
    x = xa(x, xm(vx, DT));
    y = xa(y, xm(vy, DT));
    st[0] = x; st[1] = y; st[2] = vx; st[3] = vy;
}

template <>
struct Env<ENV_BALL_CIRCLE> {
    static constexpr int D = 8, A = 2, S = 4, T = 200;
    __device__ static void reset(float* st, uint32_t seed, uint32_t env, uint32_t ep) {
        uint32_t r[4];
        Philox::gen(env, ep, 0u, 0u, seed, KEY_RESET, r);
        st[0] = xm(usym(r[0]), 0.3f); st[1] = xm(usym(r[1]), 0.3f); st[2] = 0.0f; st[3] = 0.0f;
    }
    __device__ static void observe(const float* st, float* o, uint32_t, uint32_t, uint32_t) {
        using namespace ball;
        const float x = st[0], y = st[1], vx = st[2], vy = st[3];
        const float r = xq(xa(xm(x, x), xm(y, y)));
        const float rg = xa(r, 1e-6f);
        o[0] = xd(x, R); o[1] = xd(y, R); o[2] = vx; o[3] = vy; o[4] = xd(xs(r, R), R);
        o[5] = xq(xa(xm(vx, vx), xm(vy, vy))); o[6] = xd(x, rg); o[7] = xd(y, rg);
    }
    __device__ static void step(float* st, const float* a, uint32_t, uint32_t, uint32_t,
                                float& rew, float& cost, bool& term) {
        using namespace ball;
        ball_advance(st, a[0], a[1]);
        const float x = st[0], y = st[1], vx = st[2], vy = st[3];
        const float r = xq(xa(xm(x, x), xm(y, y)));
        rew = xd(xs(xm(x, vy), xm(y, vx)), xm(R, xa(1.0f, fabsf(xs(r, R)))));
        cost = (fabsf(x) > XLIM) ? 1.0f : 0.0f;
        term = false;
    }
};

template <>
struct Env<ENV_BALL_RUN> {
    static constexpr int D = 7, A = 2, S = 5, T = 100;
    __device__ static void reset(float* st, uint32_t seed, uint32_t env, uint32_t ep) {
        uint32_t r[4];
        Philox::gen(env, ep, 0u, 0u, seed, KEY_RESET, r);
        st[0] = 0.0f; st[1] = xm(usym(r[0]), 0.2f); st[2] = 0.0f; st[3] = 0.0f; st[4] = 0.0f;
    }
    __device__ static void observe(const float* st, float* o, uint32_t, uint32_t, uint32_t) {
        using namespace ball;
        const float y = st[1], vx = st[2], vy = st[3];
        const float sp = xq(xa(xm(vx, vx), xm(vy, vy)));
        o[0] = y; o[1] = vx; o[2] = vy; o[3] = sp; o[4] = xs(sp, VLIM); o[5] = xs(fabsf(y), YLIM);
        o[6] = xd(st[0], 10.0f);
    }
    __device__ static void step(float* st, const float* a, uint32_t, uint32_t, uint32_t,
                                float& rew, float& cost, bool& term) {
        using namespace ball;
        const float x_old = st[0];
        ball_advance(st, a[0], a[1]);
        const float vx = st[2], vy = st[3];
        const float sp = xq(xa(xm(vx, vx), xm(vy, vy)));
        rew = xm(xd(xs(st[0], x_old), DT), RSCALE);
        cost = (fabsf(st[1]) > YLIM || sp > VLIM) ? 1.0f : 0.0f;
        st[4] = xa(st[4], cost);
        term = false;
    }
};

// ---------------------------------------------------------------------------------------------
// Ant-Circle (D = 34, A = 8): a torso that moves like the car, driven by 8 actuated joints
// modelled as damped oscillators.  Joints 0-3 contribute thrust, 4-7 contribute turning.
// state: x, y, c, s, v, w, q[8], qd[8], a_prev[8]
// ---------------------------------------------------------------------------------------------
// the 8 joints (shared with Ant-Run): integrate, remember the action, sum thrust / turn / a.a
__device__ __forceinline__ void ant_joints(float* st, const float* a, float& thrust, float& turn, float& ctrl) {
    using namespace ant;
    thrust = 0.0f; turn = 0.0f; ctrl = 0.0f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        float q = st[6 + j], qd = st[14 + j];
        // qd += (KA*a - KQ*q - KD*qd) * dt ; q += qd * dt
        qd = xa(qd, xm(xs(xs(xm(KA, a[j]), xm(KQ, q)), xm(KD, qd)), DT));
        q = xa(q, xm(qd, DT));
        st[6 + j] = q; st[14 + j] = qd; st[22 + j] = a[j];
        if (j < 4) thrust = xa(thrust, q); else turn = xa(turn, q);
        ctrl = xa(ctrl, xm(a[j], a[j]));
    }
}

template <>
struct Env<ENV_ANT_CIRCLE> {
    static constexpr int D = 34, A = 8, S = 30, T = 500;
    __device__ static void reset(float* st, uint32_t seed, uint32_t env, uint32_t ep) {
        uint32_t r[4];
        Philox::gen(env, ep, 0u, 0u, seed, KEY_RESET, r);
        st[0] = xm(usym(r[0]), 0.5f);
        st[1] = xm(usym(r[1]), 0.5f);
        heading_from_box(usym(r[2]), usym(r[3]), st[2], st[3]);
        st[4] = 0.0f; st[5] = 0.0f;
        uint32_t q[4];
        Philox::gen(env, ep, 1u, 0u, seed, KEY_RESET, q);
        uint32_t q2[4];
        Philox::gen(env, ep, 2u, 0u, seed, KEY_RESET, q2);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            st[6 + j] = xm(usym(q[j]), 0.1f);
            st[10 + j] = xm(usym(q2[j]), 0.1f);
        }
#pragma unroll
        for (int j = 0; j < 16; ++j) st[14 + j] = 0.0f;
    }
    __device__ static void observe(const float* st, float* o, uint32_t, uint32_t, uint32_t) {
        using namespace ant;
        const float x = st[0], y = st[1], c = st[2], s = st[3], v = st[4], w = st[5];
        const float r = xq(xa(xm(x, x), xm(y, y)));
        o[0] = xd(x, R); o[1] = xd(y, R); o[2] = xm(v, c); o[3] = xm(v, s);
        o[4] = c; o[5] = s; o[6] = xd(w, WMAX); o[7] = xd(xs(r, R), R);
        float aq = 0.0f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            o[8 + j] = st[6 + j];
            o[16 + j] = xm(st[14 + j], 0.1f);
            o[24 + j] = st[22 + j];
            aq = xa(aq, fabsf(st[6 + j]));
        }
        o[32] = xd(v, VMAX);
        o[33] = xa(0.5f, xm(aq, 0.0125f));
    }
    __device__ static void step(float* st, const float* a, uint32_t, uint32_t, uint32_t,
                                float& rew, float& cost, bool& term) {
        using namespace ant;
        float thrust, turn, ctrl;
        ant_joints(st, a, thrust, turn, ctrl);
        // joint deflection (bounded to [-1,1]) commands the torso
        float f = fminf(1.0f, fmaxf(-1.0f, xm(thrust, 0.25f)));
        float g = fminf(1.0f, fmaxf(-1.0f, xm(turn, 0.25f)));
        car_advance(st, f, g, VMAX, WMAX, AV, AW, DT);
        const float x = st[0], y = st[1], vx = xm(st[4], st[2]), vy = xm(st[4], st[3]);
        const float r = xq(xa(xm(x, x), xm(y, y)));
        rew = xs(xd(xs(xm(x, vy), xm(y, vx)), xm(R, xa(1.0f, fabsf(xs(r, R))))), xm(0.005f, ctrl));
        cost = (fabsf(x) > XLIM) ? 1.0f : 0.0f;
        term = false;
    }
};

// ---------------------------------------------------------------------------------------------
// 16-bin pseudo-lidar of the Safety-Gymnasium tasks, computed with exact ops (sector membership by
// cross products against constant bin-edge directions, no atan2).  The tasks follow the drones.
// ---------------------------------------------------------------------------------------------
__device__ __constant__ float LIDAR_EDGE_C[16] = {
    1.0f, 0.92387953f, 0.70710678f, 0.38268343f, 0.0f, -0.38268343f, -0.70710678f, -0.92387953f,
    -1.0f, -0.92387953f, -0.70710678f, -0.38268343f, 0.0f, 0.38268343f, 0.70710678f, 0.92387953f};
__device__ __constant__ float LIDAR_EDGE_S[16] = {
    0.0f, 0.38268343f, 0.70710678f, 0.92387953f, 1.0f, 0.92387953f, 0.70710678f, 0.38268343f,
    0.0f, -0.38268343f, -0.70710678f, -0.92387953f, -1.0f, -0.92387953f, -0.70710678f, -0.38268343f};

// rx, ry: object position in the robot frame.  Returns its sector; val = its closeness.
__device__ __forceinline__ int lidar_bin(float rx, float ry, float& val) {
    using namespace pgoal;
    const float d = xq(xa(xm(rx, rx), xm(ry, ry)));
    val = fmaxf(0.0f, xs(1.0f, xd(d, LIDAR_MAX)));
    int bin = 0;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        const int k1 = (k + 1) & 15;
        const float c0 = xs(xm(LIDAR_EDGE_C[k], ry), xm(LIDAR_EDGE_S[k], rx));     // cross(edge_k, r)
        const float c1 = xs(xm(LIDAR_EDGE_C[k1], ry), xm(LIDAR_EDGE_S[k1], rx));   // cross(edge_k+1, r)
        if (c0 >= 0.0f && c1 < 0.0f) bin = k;
    }
    return bin;
}

// Writes max(closeness) into the object's sector.
__device__ __forceinline__ void lidar_add(float* bins, float rx, float ry) {
    float val;
    const int bin = lidar_bin(rx, ry, val);
    bins[bin] = fmaxf(bins[bin], val);
}


// ---------------------------------------------------------------------------------------------
// Ant-Run (D = 34, A = 8, T = 300): Ant-Circle's joints and torso on the Run task.  Reward is the
// forward progress in x per second minus Ant-Circle's control cost; cost 1 when |y| leaves the
// corridor or the torso speed exceeds VLIM.
// state: x, y, c, s, v, w, q[8], qd[8], a_prev[8], cost_sum
// ---------------------------------------------------------------------------------------------
template <>
struct Env<ENV_ANT_RUN> {
    static constexpr int D = 34, A = 8, S = 31, T = 300;
    __device__ static void reset(float* st, uint32_t seed, uint32_t env, uint32_t ep) {
        uint32_t r[4];
        Philox::gen(env, ep, 0u, 0u, seed, KEY_RESET, r);
        st[0] = 0.0f;
        st[1] = xm(usym(r[0]), 0.2f);
        heading_from_box(1.0f, xm(usym(r[1]), 0.3f), st[2], st[3]);
        st[4] = 0.0f; st[5] = 0.0f;
        uint32_t q[4];
        Philox::gen(env, ep, 1u, 0u, seed, KEY_RESET, q);
        uint32_t q2[4];
        Philox::gen(env, ep, 2u, 0u, seed, KEY_RESET, q2);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            st[6 + j] = xm(usym(q[j]), 0.1f);
            st[10 + j] = xm(usym(q2[j]), 0.1f);
        }
#pragma unroll
        for (int j = 0; j < 17; ++j) st[14 + j] = 0.0f;
    }
    __device__ static void observe(const float* st, float* o, uint32_t, uint32_t, uint32_t) {
        using namespace ant;
        const float y = st[1], c = st[2], s = st[3], v = st[4], w = st[5];
        o[0] = y; o[1] = xm(v, c); o[2] = xm(v, s); o[3] = c; o[4] = s;
        o[5] = xd(w, WMAX); o[6] = xd(v, antr::VLIM); o[7] = xd(st[0], 10.0f);
        float aq = 0.0f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            o[8 + j] = st[6 + j];
            o[16 + j] = xm(st[14 + j], 0.1f);
            o[24 + j] = st[22 + j];
            aq = xa(aq, fabsf(st[6 + j]));
        }
        o[32] = xs(fabsf(y), antr::YLIM);
        o[33] = xa(0.5f, xm(aq, 0.0125f));
    }
    __device__ static void step(float* st, const float* a, uint32_t, uint32_t, uint32_t,
                                float& rew, float& cost, bool& term) {
        using namespace ant;
        const float x_old = st[0];
        float thrust, turn, ctrl;
        ant_joints(st, a, thrust, turn, ctrl);
        float f = fminf(1.0f, fmaxf(-1.0f, xm(thrust, 0.25f)));
        float g = fminf(1.0f, fmaxf(-1.0f, xm(turn, 0.25f)));
        car_advance(st, f, g, VMAX, WMAX, AV, AW, DT);
        rew = xs(xm(xd(xs(st[0], x_old), DT), antr::RSCALE), xm(0.005f, ctrl));
        cost = (fabsf(st[1]) > antr::YLIM || st[4] > antr::VLIM) ? 1.0f : 0.0f;
        st[30] = xa(st[30], cost);
        term = false;
    }
};

// ---------------------------------------------------------------------------------------------
// Quadrotor (A = 4), shared by Drone-Circle and Drone-Run.
//   motors   m_j += ((a_j + 1)/2 - m_j) * KM         (first-order lag; a = 0 is hover, m = 1/2)
//   mix      thrust = TM * sum m  (TM * 2 = G);  roll = m0+m3-m1-m2, pitch = m0+m1-m2-m3,
//            yaw = m0+m2-m1-m3
//   attitude roll / pitch are small angles with an attitude-hold spring and damped rates:
//            p += (KT*roll - KP*phi - KD*p) * dt ; phi += p * dt   (same for pitch)
//            the yaw rate is damped (KY, KDY) and turns the unit heading (c, s) by rotate_heading
//   forces   body-frame (thrust*sin(pitch), thrust*sin(roll)) rotated into the world by the
//            heading, vertical thrust*cos(roll)*cos(pitch) - G, linear drag DRAG on every axis;
//            sin / cos are the polynomials of rotate_heading
//   termination: altitude z <= 0 (crash), or |roll| or |pitch| > FLIP
// state: x, y, z, c, s, vx, vy, vz, phi, theta, p, q, r, m[4] [, cost_sum (run)]
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void poly_sincos(float d, float& sn, float& cs) {
    const float d2 = xm(d, d);
    sn = xm(d, xs(1.0f, xm(xd(d2, 6.0f), xs(1.0f, xd(d2, 20.0f)))));
    cs = xs(1.0f, xm(xd(d2, 2.0f), xs(1.0f, xm(xd(d2, 12.0f), xs(1.0f, xd(d2, 30.0f))))));
}

// reset: hover at Z0 with the motors at hover thrust, small random x, y (x = 0 for Run) and tilt,
// random heading
__device__ __forceinline__ void drone_reset(float* st, bool run, uint32_t seed, uint32_t env, uint32_t ep) {
    uint32_t r[4];
    Philox::gen(env, ep, 0u, 0u, seed, KEY_RESET, r);
    st[0] = run ? 0.0f : xm(usym(r[0]), 0.3f);
    st[1] = xm(usym(r[1]), 0.3f);
    st[2] = drone::Z0;
    heading_from_box(usym(r[2]), usym(r[3]), st[3], st[4]);
    uint32_t q[4];
    Philox::gen(env, ep, 1u, 0u, seed, KEY_RESET, q);
    st[5] = 0.0f; st[6] = 0.0f; st[7] = 0.0f;
    st[8] = xm(usym(q[0]), 0.1f);
    st[9] = xm(usym(q[1]), 0.1f);
    st[10] = 0.0f; st[11] = 0.0f; st[12] = 0.0f;
#pragma unroll
    for (int j = 0; j < 4; ++j) st[13 + j] = 0.5f;
}

// one step of the body; returns terminated
__device__ __forceinline__ bool drone_advance(float* st, const float* a) {
    using namespace drone;
    float m[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        m[j] = xa(st[13 + j], xm(xs(xm(xa(a[j], 1.0f), 0.5f), st[13 + j]), KM));
        st[13 + j] = m[j];
    }
    const float thr = xm(TM, xa(xa(m[0], m[1]), xa(m[2], m[3])));
    const float tr = xs(xa(m[0], m[3]), xa(m[1], m[2]));
    const float tp = xs(xa(m[0], m[1]), xa(m[2], m[3]));
    const float ty = xs(xa(m[0], m[2]), xa(m[1], m[3]));
    float x = st[0], y = st[1], z = st[2], c = st[3], s = st[4], vx = st[5], vy = st[6], vz = st[7];
    float phi = st[8], th = st[9], p = st[10], q = st[11], r = st[12];
    p = xa(p, xm(xs(xs(xm(KT, tr), xm(KP, phi)), xm(KD, p)), DT));
    phi = xa(phi, xm(p, DT));
    q = xa(q, xm(xs(xs(xm(KT, tp), xm(KP, th)), xm(KD, q)), DT));
    th = xa(th, xm(q, DT));
    r = xa(r, xm(xs(xm(KY, ty), xm(KDY, r)), DT));
    rotate_heading(c, s, xm(r, DT));
    float sp, cp, sth, cth;
    poly_sincos(phi, sp, cp);
    poly_sincos(th, sth, cth);
    const float axb = xm(thr, sth), ayb = xm(thr, sp);
    const float ax = xs(xm(c, axb), xm(s, ayb));
    const float ay = xa(xm(s, axb), xm(c, ayb));
    const float az = xs(xm(xm(thr, cp), cth), G);
    vx = xa(vx, xm(xs(ax, xm(DRAG, vx)), DT));
    vy = xa(vy, xm(xs(ay, xm(DRAG, vy)), DT));
    vz = xa(vz, xm(xs(az, xm(DRAG, vz)), DT));
    x = xa(x, xm(vx, DT));
    y = xa(y, xm(vy, DT));
    z = xa(z, xm(vz, DT));
    st[0] = x; st[1] = y; st[2] = z; st[3] = c; st[4] = s; st[5] = vx; st[6] = vy; st[7] = vz;
    st[8] = phi; st[9] = th; st[10] = p; st[11] = q; st[12] = r;
    return z <= 0.0f || fabsf(phi) > FLIP || fabsf(th) > FLIP;
}

// the 15 body channels of both Drone tasks
__device__ __forceinline__ void drone_body_obs(const float* st, float* o) {
    o[0] = xs(st[2], drone::Z0);
    o[1] = st[5]; o[2] = st[6]; o[3] = st[7];
    o[4] = st[3]; o[5] = st[4];
    o[6] = st[8]; o[7] = st[9];
    o[8] = st[10]; o[9] = st[11]; o[10] = st[12];
#pragma unroll
    for (int j = 0; j < 4; ++j) o[11 + j] = xm(xs(st[13 + j], 0.5f), 2.0f);
}

// Drone-Circle (D = 18, T = 300): Car/Ball-Circle's reward and cost on the quadrotor
template <>
struct Env<ENV_DRONE_CIRCLE> {
    static constexpr int D = 18, A = 4, S = 17, T = 300;
    __device__ static void reset(float* st, uint32_t seed, uint32_t env, uint32_t ep) {
        drone_reset(st, false, seed, env, ep);
    }
    __device__ static void observe(const float* st, float* o, uint32_t, uint32_t, uint32_t) {
        using namespace drone;
        const float x = st[0], y = st[1];
        const float r = xq(xa(xm(x, x), xm(y, y)));
        o[0] = xd(x, R); o[1] = xd(y, R);
        drone_body_obs(st, o + 2);
        o[17] = xd(xs(r, R), R);
    }
    __device__ static void step(float* st, const float* a, uint32_t, uint32_t, uint32_t,
                                float& rew, float& cost, bool& term) {
        using namespace drone;
        term = drone_advance(st, a);
        const float x = st[0], y = st[1], vx = st[5], vy = st[6];
        const float r = xq(xa(xm(x, x), xm(y, y)));
        rew = xd(xs(xm(x, vy), xm(y, vx)), xm(R, xa(1.0f, fabsf(xs(r, R)))));
        cost = (fabsf(x) > XLIM) ? 1.0f : 0.0f;
    }
};

// Drone-Run (D = 19, T = 200): Car/Ball-Run's reward and cost on the quadrotor
template <>
struct Env<ENV_DRONE_RUN> {
    static constexpr int D = 19, A = 4, S = 18, T = 200;
    __device__ static void reset(float* st, uint32_t seed, uint32_t env, uint32_t ep) {
        drone_reset(st, true, seed, env, ep);
        st[17] = 0.0f;
    }
    __device__ static void observe(const float* st, float* o, uint32_t, uint32_t, uint32_t) {
        using namespace drone;
        const float vx = st[5], vy = st[6];
        const float sp = xq(xa(xm(vx, vx), xm(vy, vy)));
        o[0] = st[1];
        drone_body_obs(st, o + 1);
        o[16] = xs(sp, VLIM); o[17] = xs(fabsf(st[1]), YLIM); o[18] = xd(st[0], 10.0f);
    }
    __device__ static void step(float* st, const float* a, uint32_t, uint32_t, uint32_t,
                                float& rew, float& cost, bool& term) {
        using namespace drone;
        const float x_old = st[0];
        term = drone_advance(st, a);
        const float vx = st[5], vy = st[6];
        const float sp = xq(xa(xm(vx, vx), xm(vy, vy)));
        rew = xm(xd(xs(st[0], x_old), DT), RSCALE);
        cost = (fabsf(st[1]) > YLIM || sp > VLIM) ? 1.0f : 0.0f;
        st[17] = xa(st[17], cost);
    }
};

// ---------------------------------------------------------------------------------------------
// Safety-Gymnasium navigation: the Point and Car robots on the Circle and Goal tasks.
//
// Bodies (state x, y, c, s, v, w: forward speed and yaw rate):
//   Point  PointGoal1's unicycle (car_advance, pgoal constants)
//   Car    differential drive: the two actions command the left / right wheel speeds vl, vr, which
//          follow them through a first-order lag; v = (vl + vr) / 2, w = (vr - vl) / TRACK.  Safety-
//          Gymnasium's Car also carries rear-ball sensors; they are not modelled.
// Both expose the same 12 proprioceptive channels (accelerometer, velocimeter, gyro, magnetometer).
// ---------------------------------------------------------------------------------------------
// The Car's wheel lag is linear, so it is the same lag on v and w: v follows (cl + cr) / 2 * CAR_VW and
// w follows (cr - cl) / TRACK * CAR_VW for the wheel commands cl = a[0], cr = a[1].
template <bool CAR>
__device__ __forceinline__ void nav_advance(float* st, const float* a) {
    using namespace nav;
    if constexpr (CAR)
        car_advance(st, xm(xa(a[0], a[1]), 0.5f), xm(xs(a[1], a[0]), 0.5f), CAR_VW, xd(xm(2.0f, CAR_VW), TRACK),
                    CAR_AL, CAR_AL, pgoal::DT);
    else
        car_advance(st, a[0], a[1], pgoal::VMAX, pgoal::WMAX, pgoal::AV, pgoal::AW, pgoal::DT);
}

// the 12 proprioceptive channels from forward speed v, yaw rate w, the speed before the step, heading
__device__ __forceinline__ void nav_sensors(float* o, float v, float w, float v_prev, float c, float s) {
    o[0] = xd(xs(v, v_prev), pgoal::DT); o[1] = xm(v, w); o[2] = 9.81f;   // accelerometer
    o[3] = v; o[4] = 0.0f; o[5] = 0.0f;                                    // velocimeter (body frame)
    o[6] = 0.0f; o[7] = 0.0f; o[8] = w;                                    // gyro
    o[9] = c; o[10] = xs(0.0f, s); o[11] = 0.0f;                           // magnetometer
}

// the world point (ox, oy) into a lidar of the robot at (x, y) with heading (c, s):
// robot frame rx = c*dx + s*dy ; ry = -s*dx + c*dy
__device__ __forceinline__ void lidar_world(float* bins, float ox, float oy, float x, float y, float c, float s) {
    const float dx = xs(ox, x), dy = xs(oy, y);
    lidar_add(bins, xa(xm(c, dx), xm(s, dy)), xs(xm(c, dy), xm(s, dx)));
}

// the robot's pose at reset on the Goal, Button and Push tasks: position in [-0.5, 0.5]^2, heading towards a
// point of the square, at rest (x, y, c, s, v, w = draw 0 of the reset's Philox stream)
__device__ __forceinline__ void nav_reset_pose(float* st, uint32_t seed, uint32_t env, uint32_t ep) {
    uint32_t r[4];
    Philox::gen(env, ep, 0u, 0u, seed, KEY_RESET, r);
    st[0] = xm(usym(r[0]), 0.5f);
    st[1] = xm(usym(r[1]), 0.5f);
    heading_from_box(usym(r[2]), usym(r[3]), st[2], st[3]);
    st[4] = 0.0f; st[5] = 0.0f;
}

// the squared distance from the robot (x, y) to the point (ox, oy)
__device__ __forceinline__ float nav_dist2(float ox, float oy, float x, float y) {
    const float dx = xs(ox, x), dy = xs(oy, y);
    return xa(xm(dx, dx), xm(dy, dy));
}

// Circle (D = 28, A = 2, T = 500): the 12 channels, then a 16-bin lidar towards the circle's centre.
// Reward is Safety-Gymnasium's 0.1 * (x*vy - y*vx) / (r * (1 + |r - R|)), with r kept away from 0.
// Cost 1 outside the walls: |x| > WALL at level 1, |x| or |y| > WALL at level 2.  The walls do not
// stop the robot.  Resets start inside the walls.
// state: x, y, c, s, v, w, v_prev
template <bool CAR, int LEVEL>
struct NavCircle {
    static constexpr int D = 28, A = 2, S = 7, T = 500;
    __device__ static void reset(float* st, uint32_t seed, uint32_t env, uint32_t ep) {
        uint32_t r[4];
        Philox::gen(env, ep, 0u, 0u, seed, KEY_RESET, r);
        st[0] = xm(usym(r[0]), nav::START);
        st[1] = xm(usym(r[1]), nav::START);
        heading_from_box(usym(r[2]), usym(r[3]), st[2], st[3]);
        st[4] = 0.0f; st[5] = 0.0f; st[6] = 0.0f;
    }
    __device__ static void observe(const float* st, float* o, uint32_t, uint32_t, uint32_t) {
        const float x = st[0], y = st[1], c = st[2], s = st[3];
        nav_sensors(o, st[4], st[5], st[6], c, s);
        // one object: its sector holds its closeness and the others 0, written without a dynamic index
        // so that o stays in registers
        const float dx = xs(0.0f, x), dy = xs(0.0f, y);
        float val;
        const int bin = lidar_bin(xa(xm(c, dx), xm(s, dy)), xs(xm(c, dy), xm(s, dx)), val);
#pragma unroll
        for (int k = 0; k < 16; ++k) o[12 + k] = k == bin ? val : 0.0f;
    }
    __device__ static void step(float* st, const float* a, uint32_t, uint32_t, uint32_t,
                                float& rew, float& cost, bool& term) {
        using namespace nav;
        st[6] = st[4];
        nav_advance<CAR>(st, a);
        const float x = st[0], y = st[1], vx = xm(st[4], st[2]), vy = xm(st[4], st[3]);
        const float r = xq(xa(xm(x, x), xm(y, y)));
        rew = xm(xd(xs(xm(x, vy), xm(y, vx)), xm(fmaxf(r, 1e-6f), xa(1.0f, fabsf(xs(r, CIRC_R))))), 0.1f);
        cost = (fabsf(x) > WALL || (LEVEL == 2 && fabsf(y) > WALL)) ? 1.0f : 0.0f;
        term = false;
    }
};

// Goal (D = 60, A = 2, T = 1000): one goal, re-sampled when reached (+1 and the distance progress as
// reward); three 16-bin lidars (goal, hazards, vases).  Level 1: 8 hazards and 1 vase, the layout
// stored in the state; cost 1 inside a hazard.  Level 2: 10 hazards and 10 vases; the 40 floats do
// not fit ENV_MAX_S, so step / observe regenerate them from the reset's Philox stream.  Vases are
// static discs: touching one (distance <= VASE_R) costs 1 like a hazard, and Safety-Gymnasium's
// vase-velocity cost has no counterpart.  The arena walls clamp the robot.
// state, level 1: x, y, c, s, v, w, gx, gy, goal_count, haz[8][2], vase[2], v_prev
// state, level 2: x, y, c, s, v, w, gx, gy, goal_count, v_prev
template <bool CAR, int LEVEL>
struct NavGoal {
    static constexpr int D = 60, A = 2, S = LEVEL == 1 ? 28 : 10, T = 1000;
    static constexpr int VPREV = S - 1;
    static_assert(S <= ENV_MAX_S, "env state too large");

    // f(vase, x, y) for every hazard, then every vase.  Reset draws them with counters 1, 2, ... of
    // its Philox stream, two (x, y) pairs per draw.
    template <typename F>
    __device__ static void layout(const float* st, uint32_t seed, uint32_t env, uint32_t ep, F&& f) {
        using namespace pgoal;
        if constexpr (LEVEL == 1) {
#pragma unroll
            for (int h = 0; h < NHAZ; ++h) f(false, st[9 + 2 * h], st[10 + 2 * h]);
            f(true, st[25], st[26]);
        } else {
#pragma unroll
            for (int h = 0; h < 10; ++h) {   // draws 0-4: 10 hazards, draws 5-9: 10 vases
                uint32_t q[4];
                Philox::gen(env, ep, 1u + h, 0u, seed, KEY_RESET, q);
                f(h >= 5, xm(usym(q[0]), ARENA), xm(usym(q[1]), ARENA));
                f(h >= 5, xm(usym(q[2]), ARENA), xm(usym(q[3]), ARENA));
            }
        }
    }
    __device__ static void sample_goal(float* st, uint32_t seed, uint32_t env, uint32_t ep, uint32_t k) {
        uint32_t r[4];
        Philox::gen(env, ep, k, 0u, seed, KEY_GOAL, r);
        st[6] = xm(usym(r[0]), pgoal::ARENA);
        st[7] = xm(usym(r[1]), pgoal::ARENA);
    }
    __device__ static void reset(float* st, uint32_t seed, uint32_t env, uint32_t ep) {
        using namespace pgoal;
        nav_reset_pose(st, seed, env, ep);
        sample_goal(st, seed, env, ep, 0u);
        st[8] = 0.0f;
        if constexpr (LEVEL == 1) {
#pragma unroll
            for (int h = 0; h < 5; ++h) {   // 5 Philox calls -> 10 (x, y) pairs: 8 hazards, vase, spare
                uint32_t q[4];
                Philox::gen(env, ep, 1u + h, 0u, seed, KEY_RESET, q);
                if (h < 4) {
                    st[9 + 4 * h] = xm(usym(q[0]), ARENA); st[10 + 4 * h] = xm(usym(q[1]), ARENA);
                    st[11 + 4 * h] = xm(usym(q[2]), ARENA); st[12 + 4 * h] = xm(usym(q[3]), ARENA);
                } else {
                    st[25] = xm(usym(q[0]), ARENA); st[26] = xm(usym(q[1]), ARENA);
                }
            }
        }
        st[VPREV] = 0.0f;
    }
    __device__ static void observe(const float* st, float* o, uint32_t seed, uint32_t env, uint32_t ep) {
        const float x = st[0], y = st[1], c = st[2], s = st[3];
        nav_sensors(o, st[4], st[5], st[VPREV], c, s);
        float* gl = o + 12; float* hl = o + 28; float* vl = o + 44;
#pragma unroll
        for (int k = 0; k < 16; ++k) { gl[k] = 0.0f; hl[k] = 0.0f; vl[k] = 0.0f; }
        lidar_world(gl, st[6], st[7], x, y, c, s);
        layout(st, seed, env, ep, [&](bool vase, float ox, float oy) { lidar_world(vase ? vl : hl, ox, oy, x, y, c, s); });
    }
    __device__ static void step(float* st, const float* a, uint32_t seed, uint32_t env, uint32_t ep,
                                float& rew, float& cost, bool& term) {
        using namespace pgoal;
        const float dxo = xs(st[6], st[0]), dyo = xs(st[7], st[1]);
        const float dist_old = xq(xa(xm(dxo, dxo), xm(dyo, dyo)));
        st[VPREV] = st[4];
        nav_advance<CAR>(st, a);
        st[0] = fminf(ARENA, fmaxf(-ARENA, st[0]));
        st[1] = fminf(ARENA, fmaxf(-ARENA, st[1]));
        const float dxn = xs(st[6], st[0]), dyn = xs(st[7], st[1]);
        const float dist = xq(xa(xm(dxn, dxn), xm(dyn, dyn)));
        rew = xs(dist_old, dist);
        if (dist <= GOAL_R) {
            rew = xa(rew, 1.0f);
            st[8] = xa(st[8], 1.0f);
            sample_goal(st, seed, env, ep, 16u + (uint32_t)st[8]);
        }
        float c = 0.0f;
        layout(st, seed, env, ep, [&](bool vase, float ox, float oy) {
            const float dx = xs(ox, st[0]), dy = xs(oy, st[1]);
            const float d2 = xa(xm(dx, dx), xm(dy, dy));
            if (vase ? (LEVEL == 2 && d2 <= nav::VASE_R * nav::VASE_R) : d2 <= HAZ_R * HAZ_R) c = 1.0f;
        });
        cost = c;
        term = false;
    }
};

// Button (D = 76, A = 2, T = 1000): 4 buttons, one of them the goal; hazards and gremlins (level 1: 4 and 4,
// level 2: 8 and 6), all drawn in the arena at reset.  The layout does not fit ENV_MAX_S beside the dynamic
// state, so step / observe regenerate it from the reset's Philox stream at both levels: draws 1-2 hold the
// buttons, draws 3, 4, ... the hazards and then the gremlins' orbit centres, two (x, y) pairs per draw.
//   Gremlins orbit their centre at radius GREM_TRAVEL.  One unit phase (pc, ps) advances by GREM_W * DT per step
//   (rotate_heading); gremlin k sits at the phase turned by (k mod 4) quarter-turns, gremlins 4-5 use the
//   mirrored phase (pc, -ps) and orbit the other way.
//   Step: reward = the distance progress towards the goal button.  A live step (timer 0) with the robot within
//   BUTTON_R of the goal presses it: +1, the count goes up, the buttons go hidden and inert for DELAY steps and
//   the goal moves to one of the other three buttons, (goal + 1 + r % 3) % 4 with r from the goal stream at
//   16 + count.  While the timer runs it counts down and nothing presses.  Then the gremlins move.
//   Cost 1 within pgoal::HAZ_R of a hazard, within GREM_R of a gremlin, or, on a live step, within BUTTON_R
//   of a button other than the step's goal.
//   Observation: the 12 channels, then 16-bin lidars of the goal button | all buttons (zero while the timer
//   runs) | gremlins | hazards.  The arena walls clamp the robot; gremlins may orbit past them.
// state: x, y, c, s, v, w, v_prev, goal, count, timer, pc, ps
template <bool CAR, int LEVEL>
struct NavButton {
    static constexpr int D = 76, A = 2, S = 12, T = 1000;
    static constexpr int NHAZ = LEVEL == 1 ? 4 : 8, NGREM = LEVEL == 1 ? 4 : 6;
    static_assert((NHAZ + NGREM) % 2 == 0, "two objects per Philox draw");

    __device__ static void buttons(uint32_t seed, uint32_t env, uint32_t ep, float (&bx)[4], float (&by)[4]) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            uint32_t q[4];
            Philox::gen(env, ep, 1u + h, 0u, seed, KEY_RESET, q);
            bx[2 * h] = xm(usym(q[0]), pgoal::ARENA); by[2 * h] = xm(usym(q[1]), pgoal::ARENA);
            bx[2 * h + 1] = xm(usym(q[2]), pgoal::ARENA); by[2 * h + 1] = xm(usym(q[3]), pgoal::ARENA);
        }
    }
    // f(gremlin, x, y) for every hazard, then every gremlin at the phase held in the state
    template <typename F>
    __device__ static void hazards_gremlins(const float* st, uint32_t seed, uint32_t env, uint32_t ep, F&& f) {
        const float pc = st[10], ps = st[11];
#pragma unroll
        for (int h = 0; h < (NHAZ + NGREM) / 2; ++h) {
            uint32_t q[4];
            Philox::gen(env, ep, 3u + h, 0u, seed, KEY_RESET, q);
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const int k = 2 * h + j;
                const float ox = xm(usym(q[2 * j]), pgoal::ARENA), oy = xm(usym(q[2 * j + 1]), pgoal::ARENA);
                if (k < NHAZ) {
                    f(false, ox, oy);
                    continue;
                }
                const int g = k - NHAZ;
                const float qs = g >= 4 ? -ps : ps;
                const float ux = (g & 3) == 0 ? pc : (g & 3) == 1 ? -qs : (g & 3) == 2 ? -pc : qs;
                const float uy = (g & 3) == 0 ? qs : (g & 3) == 1 ? pc : (g & 3) == 2 ? -qs : -pc;
                f(true, xa(ox, xm(button::GREM_TRAVEL, ux)), xa(oy, xm(button::GREM_TRAVEL, uy)));
            }
        }
    }
    __device__ static void reset(float* st, uint32_t seed, uint32_t env, uint32_t ep) {
        nav_reset_pose(st, seed, env, ep);
        st[6] = 0.0f;
        uint32_t g[4];
        Philox::gen(env, ep, 0u, 0u, seed, KEY_GOAL, g);
        st[7] = (float)(g[0] % 4u);
        st[8] = 0.0f; st[9] = 0.0f;
        heading_from_box(usym(g[1]), usym(g[2]), st[10], st[11]);
    }
    __device__ static void observe(const float* st, float* o, uint32_t seed, uint32_t env, uint32_t ep) {
        const float x = st[0], y = st[1], c = st[2], s = st[3];
        nav_sensors(o, st[4], st[5], st[6], c, s);
        float* gl = o + 12; float* bl = o + 28; float* ml = o + 44; float* hl = o + 60;
#pragma unroll
        for (int k = 0; k < 16; ++k) { gl[k] = 0.0f; bl[k] = 0.0f; ml[k] = 0.0f; hl[k] = 0.0f; }
        float bx[4], by[4];
        buttons(seed, env, ep, bx, by);
        const int goal = (int)st[7];
        const bool live = st[9] == 0.0f;
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            if (b == goal) lidar_world(gl, bx[b], by[b], x, y, c, s);
            if (live) lidar_world(bl, bx[b], by[b], x, y, c, s);
        }
        hazards_gremlins(st, seed, env, ep, [&](bool grem, float ox, float oy) { lidar_world(grem ? ml : hl, ox, oy, x, y, c, s); });
    }
    __device__ static void step(float* st, const float* a, uint32_t seed, uint32_t env, uint32_t ep,
                                float& rew, float& cost, bool& term) {
        using namespace button;
        float bx[4], by[4];
        buttons(seed, env, ep, bx, by);
        const int goal = (int)st[7];
        float gx = bx[0], gy = by[0];
#pragma unroll
        for (int b = 1; b < 4; ++b)
            if (b == goal) { gx = bx[b]; gy = by[b]; }
        const float dist_old = xq(nav_dist2(gx, gy, st[0], st[1]));
        st[6] = st[4];
        nav_advance<CAR>(st, a);
        st[0] = fminf(pgoal::ARENA, fmaxf(-pgoal::ARENA, st[0]));
        st[1] = fminf(pgoal::ARENA, fmaxf(-pgoal::ARENA, st[1]));
        const float dist = xq(nav_dist2(gx, gy, st[0], st[1]));
        rew = xs(dist_old, dist);
        const bool live = st[9] == 0.0f;
        if (!live) {
            st[9] = xs(st[9], 1.0f);
        } else if (dist <= BUTTON_R) {
            rew = xa(rew, 1.0f);
            st[8] = xa(st[8], 1.0f);
            st[9] = (float)DELAY;
            uint32_t r[4];
            Philox::gen(env, ep, 16u + (uint32_t)st[8], 0u, seed, KEY_GOAL, r);
            st[7] = (float)((goal + 1 + (int)(r[0] % 3u)) & 3);
        }
        rotate_heading(st[10], st[11], GREM_W * pgoal::DT);
        float c = 0.0f;
#pragma unroll
        for (int b = 0; b < 4; ++b)
            if (live && b != goal && nav_dist2(bx[b], by[b], st[0], st[1]) <= BUTTON_R * BUTTON_R) c = 1.0f;
        hazards_gremlins(st, seed, env, ep, [&](bool grem, float ox, float oy) {
            const float d2 = nav_dist2(ox, oy, st[0], st[1]);
            if (grem ? d2 <= GREM_R * GREM_R : d2 <= pgoal::HAZ_R * pgoal::HAZ_R) c = 1.0f;
        });
        cost = c;
        term = false;
    }
};

// Push (D = 76, A = 2, T = 1000): one box, one goal, hazards and pillars (level 1: 2 and 1, level 2: 4 and 4).
// The layout fits the state: reset draws the box in [-BOX_START, BOX_START]^2 and the hazards and pillars in
// the arena from draws 1, 2, ... of its Philox stream, two (x, y) pairs per draw; the goal comes from the goal
// stream as on the Goal tasks.
//   The box is pushed kinematically: after the robot moves (and is clamped), a box closer than PUSH_D to it
//   moves along the unit vector robot -> box (the robot's heading at zero distance) until it is PUSH_D away,
//   then is clamped to the arena.  The robot is not slowed; pillars block neither the robot nor the box.
//   Reward = the robot-box distance progress + the box-goal distance progress; a box centre within
//   pgoal::GOAL_R of the goal adds +1 and re-draws the goal (goal stream, 16 + count).
//   Cost 1 within HAZ_R of a hazard and, at level 2 only, within PILLAR_R of a pillar.
//   Observation: the 12 channels, then 16-bin lidars of the goal | box | hazards | pillars.
// state: x, y, c, s, v, w, gx, gy, goal_count, bx, by, haz[NHAZ][2], pillar[NPIL][2], v_prev
template <bool CAR, int LEVEL>
struct NavPush {
    static constexpr int NHAZ = LEVEL == 1 ? 2 : 4, NPIL = LEVEL == 1 ? 1 : 4;
    static constexpr int HAZ0 = 11, PIL0 = HAZ0 + 2 * NHAZ, VPREV = PIL0 + 2 * NPIL;
    static constexpr int D = 76, A = 2, S = VPREV + 1, T = 1000;
    static_assert(S <= ENV_MAX_S, "env state too large");

    __device__ static void reset(float* st, uint32_t seed, uint32_t env, uint32_t ep) {
        nav_reset_pose(st, seed, env, ep);
        NavGoal<CAR, LEVEL>::sample_goal(st, seed, env, ep, 0u);
        st[8] = 0.0f;
        // object k (0: the box, then the hazards, then the pillars) at st[9 + 2k], st[10 + 2k]
        constexpr int NOBJ = 1 + NHAZ + NPIL;
#pragma unroll
        for (int h = 0; h < (NOBJ + 1) / 2; ++h) {
            uint32_t q[4];
            Philox::gen(env, ep, 1u + h, 0u, seed, KEY_RESET, q);
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const int k = 2 * h + j;
                if (k >= NOBJ) continue;
                const float sc = k == 0 ? push::BOX_START : pgoal::ARENA;
                st[9 + 2 * k] = xm(usym(q[2 * j]), sc);
                st[10 + 2 * k] = xm(usym(q[2 * j + 1]), sc);
            }
        }
        st[VPREV] = 0.0f;
    }
    __device__ static void observe(const float* st, float* o, uint32_t, uint32_t, uint32_t) {
        const float x = st[0], y = st[1], c = st[2], s = st[3];
        nav_sensors(o, st[4], st[5], st[VPREV], c, s);
        float* gl = o + 12; float* bl = o + 28; float* hl = o + 44; float* pl = o + 60;
#pragma unroll
        for (int k = 0; k < 16; ++k) { gl[k] = 0.0f; bl[k] = 0.0f; hl[k] = 0.0f; pl[k] = 0.0f; }
        lidar_world(gl, st[6], st[7], x, y, c, s);
        lidar_world(bl, st[9], st[10], x, y, c, s);
#pragma unroll
        for (int h = 0; h < NHAZ; ++h) lidar_world(hl, st[HAZ0 + 2 * h], st[HAZ0 + 2 * h + 1], x, y, c, s);
#pragma unroll
        for (int p = 0; p < NPIL; ++p) lidar_world(pl, st[PIL0 + 2 * p], st[PIL0 + 2 * p + 1], x, y, c, s);
    }
    __device__ static void step(float* st, const float* a, uint32_t seed, uint32_t env, uint32_t ep,
                                float& rew, float& cost, bool& term) {
        using namespace push;
        const float rb_old = xq(nav_dist2(st[9], st[10], st[0], st[1]));
        const float bg_old = xq(nav_dist2(st[6], st[7], st[9], st[10]));
        st[VPREV] = st[4];
        nav_advance<CAR>(st, a);
        const float x = fminf(pgoal::ARENA, fmaxf(-pgoal::ARENA, st[0]));
        const float y = fminf(pgoal::ARENA, fmaxf(-pgoal::ARENA, st[1]));
        st[0] = x; st[1] = y;
        const float dx = xs(st[9], x), dy = xs(st[10], y);
        const float d = xq(xa(xm(dx, dx), xm(dy, dy)));
        if (d < PUSH_D) {
            const float ux = d == 0.0f ? st[2] : xd(dx, d), uy = d == 0.0f ? st[3] : xd(dy, d);
            st[9] = fminf(pgoal::ARENA, fmaxf(-pgoal::ARENA, xa(x, xm(PUSH_D, ux))));
            st[10] = fminf(pgoal::ARENA, fmaxf(-pgoal::ARENA, xa(y, xm(PUSH_D, uy))));
        }
        const float rb = xq(nav_dist2(st[9], st[10], x, y));
        const float bg = xq(nav_dist2(st[6], st[7], st[9], st[10]));
        rew = xa(xs(rb_old, rb), xs(bg_old, bg));
        if (bg <= pgoal::GOAL_R) {
            rew = xa(rew, 1.0f);
            st[8] = xa(st[8], 1.0f);
            NavGoal<CAR, LEVEL>::sample_goal(st, seed, env, ep, 16u + (uint32_t)st[8]);
        }
        float c = 0.0f;
#pragma unroll
        for (int h = 0; h < NHAZ; ++h)
            if (nav_dist2(st[HAZ0 + 2 * h], st[HAZ0 + 2 * h + 1], x, y) <= HAZ_R * HAZ_R) c = 1.0f;
        if constexpr (LEVEL == 2) {
#pragma unroll
            for (int p = 0; p < NPIL; ++p)
                if (nav_dist2(st[PIL0 + 2 * p], st[PIL0 + 2 * p + 1], x, y) <= PILLAR_R * PILLAR_R) c = 1.0f;
        }
        cost = c;
        term = false;
    }
};

// ---------------------------------------------------------------------------------------------
// Safety-Gymnasium velocity tasks (T = 1000): HalfCheetah, Hopper, Swimmer, Walker2d and Ant, with the observation
// widths of gymnasium's MuJoCo v4 robots minus the x (x, y) position.  Our models, not MuJoCo:
//   Joints   N damped, driven joints: qd += (KA*a - KQ*q - KD*qd) * DT ; q += qd * DT  (vel_joints).
//   Gait     forward force F = clamp(GK * sum over the robot's joint pairs (i, k) of q_i*qd_k - q_k*qd_i, -1, 1):
//            the signed area the pairs sweep.  A constant action (qd -> 0) or in-phase motion sweeps none; two
//            joints driven by sinusoids a quarter period apart sweep a constant area.  The forward speed moves the
//            fraction RDT of the way to VMAX * F per step (linear drag).
//   Pitch    (HalfCheetah, Hopper, Walker2d) wd += (PU*th - PT*tq - PD*wd) * DT ; th += wd * DT, with tq the
//            thigh angle (Hopper q0, Walker2d (q0 + q3) / 2, HalfCheetah q0 - q3).  PU > 0 (Hopper, Walker2d)
//            is an inverted pendulum that only thigh feedback holds up; HalfCheetah's PU < 0 is a restoring
//            spring, and the model has no flips.  |th| is clamped to FALL (lying on the ground).
//   Height   z follows zt through a spring-damper (ZK, ZD): planar zt = (Z0 - ZQ * sum knee^2) * cos th, Ant
//            zt = Z0 + ANT_ZA * (sum of the 4 ankles).
//   Swimmer  the plane with a heading: the yaw rate follows SW_KW * (q0 + q1) (the body's bend).
//   Ant      Ant-Circle's joint layout; the gait pairs are (hip j, ankle j + 4), the speed runs along the heading,
//            the yaw rate follows ANT_KW * (area of legs 0-1 - area of legs 2-3), small roll / pitch angles with
//            spring-dampers are driven by the hips, and the quaternion observation is built from half-angles.
//   Reward   vx + HEALTHY - WCTRL * |a|^2 (a: the action the env receives).  Cost 1 when the speed (vx; the
//            planar speed for Ant) exceeds VCOST.  Terminated, checked after the step: Hopper z <= 0.7 or
//            |th| >= 0.2; Walker2d z <= 0.8, z >= 2 or |th| >= 1; Ant z < 0.2 or z > 1.
//   Reset    from the reset's Philox stream: draw 0 the body, draws 1-2 the joint angles (4 per draw, +-0.05).
// observation  HalfCheetah / Hopper / Walker2d: z, th, q[N], vx, vz, wd, qd[N]
//              Swimmer: th, q0, q1, vx, vy, wd, qd0, qd1
//              Ant: z, quaternion (w, x, y, z), q[8], vx, vy, vz, roll rate, pitch rate, yaw rate, qd[8]
// state        planar: z, vz, th, wd, vx, q[N], qd[N];  Swimmer: th, c, s, u, wd, q[2], qd[2]
//              Ant: z, vz, c, s, u, w, roll, roll rate, pitch, pitch rate, q[8], qd[8]
// ---------------------------------------------------------------------------------------------
namespace vel {
constexpr float DT = 0.05f, KA = 20.0f, KQ = 10.0f, KD = 4.0f;   // joints
constexpr float RDT = 0.1f;                                       // forward-speed relaxation per step
constexpr float ZK = 40.0f, ZD = 10.0f, ZQ = 0.05f, FALL = 1.5f;  // height spring-damper, knee crouch, pitch clamp
constexpr float SW_KW = 0.5f, SW_YD = 2.0f;                       // Swimmer yaw
constexpr float ANT_KW = 0.02f, ANT_YD = 2.0f;                    // Ant yaw
constexpr float ANT_AT = 0.5f, ANT_AS = 20.0f, ANT_AD = 6.0f;     // Ant roll / pitch: hip drive, spring, damping
constexpr float ANT_ZA = 0.1f;                                    // Ant height per unit of ankle angle
}

// per robot: N joints, state offset of q, the saturated speed, gait gain, cost threshold, control weight, healthy
// reward, standing height and pitch constants
template <int KIND> struct VelCfg;
template <> struct VelCfg<ENV_HALF_CHEETAH_VEL> {
    static constexpr int N = 6, Q0 = 5, D = 17, S = 17;
    static constexpr float VMAX = 4.0f, GK = 0.05f, VCOST = 2.8f, WCTRL = 0.1f, HEALTHY = 0.0f, Z0 = 0.6f;
    static constexpr float PU = -20.0f, PT = 0.5f, PD = 2.0f;
};
template <> struct VelCfg<ENV_HOPPER_VEL> {
    static constexpr int N = 3, Q0 = 5, D = 11, S = 11;
    static constexpr float VMAX = 0.5f, GK = 0.2f, VCOST = 0.35f, WCTRL = 1e-3f, HEALTHY = 1.0f, Z0 = 1.25f;
    static constexpr float PU = 2.0f, PT = 2.0f, PD = 1.0f;
};
template <> struct VelCfg<ENV_SWIMMER_VEL> {
    static constexpr int N = 2, Q0 = 5, D = 8, S = 9;
    static constexpr float VMAX = 0.07f, GK = 0.2f, VCOST = 0.05f, WCTRL = 1e-4f, HEALTHY = 0.0f;
};
template <> struct VelCfg<ENV_WALKER2D_VEL> {
    static constexpr int N = 6, Q0 = 5, D = 17, S = 17;
    static constexpr float VMAX = 2.5f, GK = 0.1f, VCOST = 1.7f, WCTRL = 1e-3f, HEALTHY = 1.0f, Z0 = 1.25f;
    static constexpr float PU = 2.0f, PT = 2.0f, PD = 1.0f;
};
template <> struct VelCfg<ENV_ANT_VEL> {
    static constexpr int N = 8, Q0 = 10, D = 27, S = 26;
    static constexpr float VMAX = 3.5f, GK = 0.05f, VCOST = 2.5f, WCTRL = 0.5f, HEALTHY = 1.0f, Z0 = 0.6f;
};

// the N joints q = st[0..N), qd = st[N..2N), integrated in place; returns sum a_j^2
template <int N>
__device__ __forceinline__ float vel_joints(float* st, const float* a) {
    using namespace vel;
    float ctrl = 0.0f;
#pragma unroll
    for (int j = 0; j < N; ++j) {
        const float q = st[j];
        const float qd = xa(st[N + j], xm(xs(xs(xm(KA, a[j]), xm(KQ, q)), xm(KD, st[N + j])), DT));
        st[j] = xa(q, xm(qd, DT));
        st[N + j] = qd;
        ctrl = xa(ctrl, xm(a[j], a[j]));
    }
    return ctrl;
}

// the area joints i and k sweep per unit time: q_i * qd_k - q_k * qd_i (q = st[0..N), qd = st[N..2N))
template <int N>
__device__ __forceinline__ float vel_area(const float* st, int i, int k) {
    return xs(xm(st[i], st[N + k]), xm(st[k], st[N + i]));
}

template <int KIND>
struct Velocity {
    using C = VelCfg<KIND>;
    static constexpr int N = C::N, Q0 = C::Q0, D = C::D, A = N, S = C::S, T = 1000;
    static constexpr bool PLANAR = KIND != ENV_SWIMMER_VEL && KIND != ENV_ANT_VEL;
    static_assert(S <= ENV_MAX_S && A <= ENV_MAX_A, "env too large");

    // the saturated gait force of the joints q = st[0..N), qd = st[N..2N)
    __device__ static float gait(const float* j) {
        float g = 0.0f;
        if constexpr (KIND == ENV_HOPPER_VEL) {
            g = xa(g, vel_area<N>(j, 0, 1)); g = xa(g, vel_area<N>(j, 1, 2));
        } else if constexpr (KIND == ENV_SWIMMER_VEL) {
            g = xa(g, vel_area<N>(j, 0, 1));
        } else if constexpr (KIND == ENV_ANT_VEL) {
#pragma unroll
            for (int k = 0; k < 4; ++k) g = xa(g, vel_area<N>(j, k, k + 4));
        } else {
            g = xa(g, vel_area<N>(j, 0, 1)); g = xa(g, vel_area<N>(j, 1, 2));
            g = xa(g, vel_area<N>(j, 3, 4)); g = xa(g, vel_area<N>(j, 4, 5));
        }
        return fminf(1.0f, fmaxf(-1.0f, xm(g, C::GK)));
    }
    __device__ static void reset(float* st, uint32_t seed, uint32_t env, uint32_t ep) {
        uint32_t r[4];
        Philox::gen(env, ep, 0u, 0u, seed, KEY_RESET, r);
#pragma unroll
        for (int i = 0; i < S; ++i) st[i] = 0.0f;
        if constexpr (PLANAR) {
            st[0] = xa(C::Z0, xm(usym(r[0]), 0.005f));
            st[2] = xm(usym(r[1]), 0.02f);
            st[3] = xm(usym(r[2]), 0.02f);
        } else if constexpr (KIND == ENV_SWIMMER_VEL) {
            st[0] = xm(usym(r[0]), 0.05f);
            poly_sincos(st[0], st[2], st[1]);
        } else {
            st[0] = xa(C::Z0, xm(usym(r[0]), 0.005f));
            float sn, cs;
            poly_sincos(xm(usym(r[1]), 0.05f), sn, cs);
            const float n = xq(xa(xm(cs, cs), xm(sn, sn)));
            st[2] = xd(cs, n); st[3] = xd(sn, n);
            st[6] = xm(usym(r[2]), 0.02f);
            st[8] = xm(usym(r[3]), 0.02f);
        }
#pragma unroll
        for (int h = 0; h < (N + 3) / 4; ++h) {
            uint32_t q[4];
            Philox::gen(env, ep, 1u + h, 0u, seed, KEY_RESET, q);
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (4 * h + j < N) st[Q0 + 4 * h + j] = xm(usym(q[j]), 0.05f);
        }
    }
    __device__ static void observe(const float* st, float* o, uint32_t, uint32_t, uint32_t) {
        if constexpr (PLANAR) {
            o[0] = st[0]; o[1] = st[2];
#pragma unroll
            for (int j = 0; j < N; ++j) { o[2 + j] = st[Q0 + j]; o[5 + N + j] = st[Q0 + N + j]; }
            o[2 + N] = st[4]; o[3 + N] = st[1]; o[4 + N] = st[3];
        } else if constexpr (KIND == ENV_SWIMMER_VEL) {
            o[0] = st[0]; o[1] = st[5]; o[2] = st[6];
            o[3] = xm(st[3], st[1]); o[4] = xm(st[3], st[2]); o[5] = st[4];
            o[6] = st[7]; o[7] = st[8];
        } else {
            const float c = st[2], s = st[3];
            const float ch = xq(fmaxf(0.0f, xm(xa(1.0f, c), 0.5f)));
            float sh = xq(fmaxf(0.0f, xm(xs(1.0f, c), 0.5f)));
            if (s < 0.0f) sh = -sh;
            float sr, cr, sp, cp;
            poly_sincos(xm(st[6], 0.5f), sr, cr);
            poly_sincos(xm(st[8], 0.5f), sp, cp);
            o[0] = st[0];
            o[1] = xa(xm(xm(ch, cp), cr), xm(xm(sh, sp), sr));
            o[2] = xs(xm(xm(ch, cp), sr), xm(xm(sh, sp), cr));
            o[3] = xa(xm(xm(ch, sp), cr), xm(xm(sh, cp), sr));
            o[4] = xs(xm(xm(sh, cp), cr), xm(xm(ch, sp), sr));
#pragma unroll
            for (int j = 0; j < 8; ++j) { o[5 + j] = st[Q0 + j]; o[19 + j] = st[Q0 + 8 + j]; }
            o[13] = xm(st[4], c); o[14] = xm(st[4], s); o[15] = st[1];
            o[16] = st[7]; o[17] = st[9]; o[18] = st[5];
        }
    }
    __device__ static void step(float* st, const float* a, uint32_t, uint32_t, uint32_t,
                                float& rew, float& cost, bool& term) {
        using namespace vel;
        float* j = st + Q0;
        const float ctrl = vel_joints<N>(j, a);
        const float F = gait(j);
        float vx, speed;
        term = false;
        if constexpr (PLANAR) {
            st[4] = xa(st[4], xm(xs(xm(C::VMAX, F), st[4]), RDT));
            float tq, kn;
            if constexpr (KIND == ENV_HOPPER_VEL) {
                tq = j[0]; kn = xm(j[1], j[1]);
            } else if constexpr (KIND == ENV_WALKER2D_VEL) {
                tq = xm(xa(j[0], j[3]), 0.5f); kn = xa(xm(j[1], j[1]), xm(j[4], j[4]));
            } else {
                tq = xs(j[0], j[3]); kn = xa(xm(j[1], j[1]), xm(j[4], j[4]));
            }
            float th = st[2], wd = st[3];
            wd = xa(wd, xm(xs(xs(xm(C::PU, th), xm(C::PT, tq)), xm(C::PD, wd)), DT));
            th = xa(th, xm(wd, DT));
            if (fabsf(th) > FALL) { th = th > 0.0f ? FALL : -FALL; wd = 0.0f; }
            st[2] = th; st[3] = wd;
            float sth, cth;
            poly_sincos(th, sth, cth);
            const float zt = xm(xs(C::Z0, xm(ZQ, kn)), cth);
            st[1] = xa(st[1], xm(xs(xm(ZK, xs(zt, st[0])), xm(ZD, st[1])), DT));
            st[0] = xa(st[0], xm(st[1], DT));
            vx = st[4];
            speed = vx;
            const float z = st[0];
            if constexpr (KIND == ENV_HOPPER_VEL) term = z <= 0.7f || fabsf(th) >= 0.2f;
            if constexpr (KIND == ENV_WALKER2D_VEL) term = z <= 0.8f || z >= 2.0f || fabsf(th) >= 1.0f;
        } else if constexpr (KIND == ENV_SWIMMER_VEL) {
            st[3] = xa(st[3], xm(xs(xm(C::VMAX, F), st[3]), RDT));
            st[4] = xa(st[4], xm(xs(xm(SW_KW, xa(j[0], j[1])), xm(SW_YD, st[4])), DT));
            const float d = xm(st[4], DT);
            st[0] = xa(st[0], d);
            rotate_heading(st[1], st[2], d);
            vx = xm(st[3], st[1]);
            speed = vx;
        } else {
            st[4] = xa(st[4], xm(xs(xm(C::VMAX, F), st[4]), RDT));
            const float lft = xa(vel_area<N>(j, 0, 4), vel_area<N>(j, 1, 5));
            const float rgt = xa(vel_area<N>(j, 2, 6), vel_area<N>(j, 3, 7));
            st[5] = xa(st[5], xm(xs(xm(ANT_KW, xs(lft, rgt)), xm(ANT_YD, st[5])), DT));
            rotate_heading(st[2], st[3], xm(st[5], DT));
            st[7] = xa(st[7], xm(xs(xs(xm(ANT_AT, xs(xa(j[0], j[1]), xa(j[2], j[3]))), xm(ANT_AS, st[6])),
                                    xm(ANT_AD, st[7])), DT));
            st[6] = xa(st[6], xm(st[7], DT));
            st[9] = xa(st[9], xm(xs(xs(xm(ANT_AT, xs(xa(j[0], j[3]), xa(j[1], j[2]))), xm(ANT_AS, st[8])),
                                    xm(ANT_AD, st[9])), DT));
            st[8] = xa(st[8], xm(st[9], DT));
            const float zt = xa(C::Z0, xm(ANT_ZA, xa(xa(j[4], j[5]), xa(j[6], j[7]))));
            st[1] = xa(st[1], xm(xs(xm(ZK, xs(zt, st[0])), xm(ZD, st[1])), DT));
            st[0] = xa(st[0], xm(st[1], DT));
            vx = xm(st[4], st[2]);
            const float vy = xm(st[4], st[3]);
            speed = xq(xa(xm(vx, vx), xm(vy, vy)));
            term = st[0] < 0.2f || st[0] > 1.0f;
        }
        rew = xs(xa(vx, C::HEALTHY), xm(C::WCTRL, ctrl));
        cost = speed > C::VCOST ? 1.0f : 0.0f;
    }
};

template <> struct Env<ENV_HALF_CHEETAH_VEL> : Velocity<ENV_HALF_CHEETAH_VEL> {};
template <> struct Env<ENV_HOPPER_VEL> : Velocity<ENV_HOPPER_VEL> {};
template <> struct Env<ENV_SWIMMER_VEL> : Velocity<ENV_SWIMMER_VEL> {};
template <> struct Env<ENV_WALKER2D_VEL> : Velocity<ENV_WALKER2D_VEL> {};
template <> struct Env<ENV_ANT_VEL> : Velocity<ENV_ANT_VEL> {};

template <> struct Env<ENV_POINT_GOAL> : NavGoal<false, 1> {};
template <> struct Env<ENV_POINT_CIRCLE1> : NavCircle<false, 1> {};
template <> struct Env<ENV_POINT_CIRCLE2> : NavCircle<false, 2> {};
template <> struct Env<ENV_CAR_CIRCLE1> : NavCircle<true, 1> {};
template <> struct Env<ENV_CAR_CIRCLE2> : NavCircle<true, 2> {};
template <> struct Env<ENV_POINT_GOAL2> : NavGoal<false, 2> {};
template <> struct Env<ENV_CAR_GOAL1> : NavGoal<true, 1> {};
template <> struct Env<ENV_CAR_GOAL2> : NavGoal<true, 2> {};
template <> struct Env<ENV_POINT_BUTTON1> : NavButton<false, 1> {};
template <> struct Env<ENV_POINT_BUTTON2> : NavButton<false, 2> {};
template <> struct Env<ENV_CAR_BUTTON1> : NavButton<true, 1> {};
template <> struct Env<ENV_CAR_BUTTON2> : NavButton<true, 2> {};
template <> struct Env<ENV_POINT_PUSH1> : NavPush<false, 1> {};
template <> struct Env<ENV_POINT_PUSH2> : NavPush<false, 2> {};
template <> struct Env<ENV_CAR_PUSH1> : NavPush<true, 1> {};
template <> struct Env<ENV_CAR_PUSH2> : NavPush<true, 2> {};

}  // namespace fsrl
