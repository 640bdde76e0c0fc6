// The scenes of the built-in device envs (fsrl_env_render).  The rasterizer, the primitives and the palette are in
// render.cuh; this file defines scene<K> for every built-in kind: a top-down or side view per env family, decoded
// from env_state (and, where step / observe regenerate a layout from the reset's Philox stream, through the same
// envs.cuh functions).  Only the exact helpers of envs.cuh are used, so tests/render_twin.py reproduces every pixel.
// The scenes of every family are documented in DESIGN §7.
#include "render.cuh"

namespace fsrl {
namespace render {

// sin / cos of an angle up to a few radians: the polynomial of poly_sincos at a / 4, doubled twice
__device__ __forceinline__ void wide_sincos(float a, float& sn, float& cs) {
    float s, c;
    poly_sincos(xm(a, 0.25f), s, c);
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const float s2 = xm(xm(s, c), 2.0f), c2 = xs(xm(c, c), xm(s, s));
        s = s2; c = c2;
    }
    sn = s; cs = c;
}

// (c, s) turned by the unit (ck, sk)
__device__ __forceinline__ void turn(float& c, float& s, float ck, float sk) {
    const float c2 = xs(xm(c, ck), xm(s, sk)), s2 = xa(xm(s, ck), xm(c, sk));
    c = c2; s = s2;
}

// Bullet-Safety-Gym Circle (kinds 0, 2, 4, 7) and Run (1, 3, 6, 8)
template <int K>
__device__ void scene_bullet(Builder& b, const float* st, bool cost) {
    constexpr bool RUN = K == ENV_CAR_RUN || K == ENV_BALL_RUN || K == ENV_ANT_RUN || K == ENV_DRONE_RUN;
    constexpr bool ANT = K == ENV_ANT_CIRCLE || K == ENV_ANT_RUN;
    constexpr bool BALL = K == ENV_BALL_CIRCLE || K == ENV_BALL_RUN;
    constexpr bool DRONE = K == ENV_DRONE_CIRCLE || K == ENV_DRONE_RUN;
    constexpr float RR = ANT ? 0.2f : 0.1f;                     // robot radius
    const float x = st[0], y = st[1];
    float c, s, hl;
    if constexpr (BALL) {   // the ball has no heading: its velocity, 0.25 s ahead
        c = st[2]; s = st[3]; hl = 0.25f;
    } else {
        c = DRONE ? st[3] : st[2]; s = DRONE ? st[4] : st[3]; hl = 2.0f * RR;
    }
    if constexpr (!RUN) {
        constexpr float R = ANT ? ant::R : carc::R, XLIM = ANT ? ant::XLIM : carc::XLIM;
        b.window(0.0f, 0.0f, 1.3f * R, 1.3f * R);
        b.box(b.sc.x0, b.sc.y0, -XLIM, b.sc.y1, C_WALL);
        b.box(XLIM, b.sc.y0, b.sc.x1, b.sc.y1, C_WALL);
        b.ring(0.0f, 0.0f, 0.98f * R, 1.02f * R, C_CIRCLE);
        b.robot(x, y, c, s, RR, hl, 0.35f * RR, cost);
        if constexpr (DRONE) b.gauge(st[2], drone::Z0, true);   // altitude, the mark at the hover height
    } else {
        constexpr float YLIM = ANT ? antr::YLIM : K == ENV_BALL_RUN ? ball::YLIM : K == ENV_DRONE_RUN ? drone::YLIM
                                                                                                        : carr::YLIM;
        constexpr float VLIM = ANT ? antr::VLIM : K == ENV_BALL_RUN ? ball::VLIM : K == ENV_DRONE_RUN ? drone::VLIM
                                                                                                        : carr::VLIM;
        b.window(x, 0.0f, 2.0f * YLIM, 2.0f * YLIM);
        b.box(b.sc.x0, YLIM, b.sc.x1, b.sc.y1, C_WALL);
        b.box(b.sc.x0, b.sc.y0, b.sc.x1, -YLIM, C_WALL);
        // a tick across the corridor at every whole x in the window, so the window's motion shows
        const float tw = 0.01f * YLIM;
        for (float k = ceilf(b.sc.x0); k <= b.sc.x1; k = xa(k, 1.0f)) b.box(xs(k, tw), -YLIM, xa(k, tw), YLIM, C_TICK);
        b.robot(x, y, c, s, RR, hl, 0.35f * RR, cost);
        float v;
        if constexpr (BALL) v = xq(xa(xm(st[2], st[2]), xm(st[3], st[3])));
        else if constexpr (DRONE) v = xq(xa(xm(st[5], st[5]), xm(st[6], st[6])));
        else v = st[4];
        b.gauge(v, VLIM, false);
    }
}

// Safety-Gymnasium navigation: Circle, Goal, Button, Push (kinds 5, 16-31)
template <int K>
__device__ void scene_nav(Builder& b, float* st, uint32_t seed, uint32_t env, uint32_t ep, bool cost) {
    using E_ = Env<K>;
    constexpr float RR = 0.15f;
    constexpr bool CIRCLE = K >= ENV_POINT_CIRCLE1 && K <= ENV_CAR_CIRCLE2;
    constexpr bool GOAL = K == ENV_POINT_GOAL || (K >= ENV_POINT_GOAL2 && K <= ENV_CAR_GOAL2);
    constexpr bool BUTTON = K >= ENV_POINT_BUTTON1 && K <= ENV_CAR_BUTTON2;
    if constexpr (CIRCLE) {
        constexpr bool L2 = K == ENV_POINT_CIRCLE2 || K == ENV_CAR_CIRCLE2;
        b.window(0.0f, 0.0f, 1.3f * nav::CIRC_R, 1.3f * nav::CIRC_R);
        b.box(b.sc.x0, b.sc.y0, -nav::WALL, b.sc.y1, C_WALL);
        b.box(nav::WALL, b.sc.y0, b.sc.x1, b.sc.y1, C_WALL);
        if constexpr (L2) {
            b.box(b.sc.x0, nav::WALL, b.sc.x1, b.sc.y1, C_WALL);
            b.box(b.sc.x0, b.sc.y0, b.sc.x1, -nav::WALL, C_WALL);
        }
        b.ring(0.0f, 0.0f, 0.98f * nav::CIRC_R, 1.02f * nav::CIRC_R, C_CIRCLE);
    } else {
        constexpr float A = pgoal::ARENA;
        b.window(0.0f, 0.0f, 1.1f * A, 1.1f * A);
        b.box(-A, -A, A, A, C_FLOOR);
        if constexpr (GOAL) {
            b.disc(st[6], st[7], pgoal::GOAL_R, C_GOAL);
            E_::layout(st, seed, env, ep, [&](bool vase, float ox, float oy) {
                if (vase) b.box(xs(ox, 0.1f), xs(oy, 0.1f), xa(ox, 0.1f), xa(oy, 0.1f), C_VASE);
                else b.disc(ox, oy, pgoal::HAZ_R, C_HAZARD);
            });
        } else if constexpr (BUTTON) {
            if (st[9] == 0.0f) {   // hidden while the timer runs, as their lidar is
                float bx[4], by[4];
                E_::buttons(seed, env, ep, bx, by);
                const int goal = (int)st[7];
#pragma unroll
                for (int k = 0; k < 4; ++k) b.disc(bx[k], by[k], 0.1f, k == goal ? C_GOAL : C_BUTTON);
            }
            E_::hazards_gremlins(st, seed, env, ep, [&](bool grem, float ox, float oy) {
                if (grem) b.box(xs(ox, 0.1f), xs(oy, 0.1f), xa(ox, 0.1f), xa(oy, 0.1f), C_GREMLIN);
                else b.disc(ox, oy, pgoal::HAZ_R, C_HAZARD);
            });
        } else {
            b.disc(st[6], st[7], pgoal::GOAL_R, C_GOAL);
#pragma unroll
            for (int h = 0; h < E_::NHAZ; ++h) b.disc(st[E_::HAZ0 + 2 * h], st[E_::HAZ0 + 2 * h + 1], push::HAZ_R, C_HAZARD);
#pragma unroll
            for (int p = 0; p < E_::NPIL; ++p) b.disc(st[E_::PIL0 + 2 * p], st[E_::PIL0 + 2 * p + 1], 0.25f, C_PILLAR);
            b.box(xs(st[9], 0.15f), xs(st[10], 0.15f), xa(st[9], 0.15f), xa(st[10], 0.15f), C_BOX);
        }
    }
    b.robot(st[0], st[1], st[2], st[3], RR, 2.0f * RR, 0.35f * RR, cost);
}

// a chain of limbs from (x, y): link k points along (c, s) turned by the sum of q[0..k], length len[k]
template <int N>
__device__ void limbs(Builder& b, float x, float y, float c, float s, const float* q, const float (&len)[N], float hw) {
#pragma unroll
    for (int k = 0; k < N; ++k) {
        float sn, cs;
        wide_sincos(q[k], sn, cs);
        turn(c, s, cs, sn);
        const float x2 = xa(x, xm(len[k], c)), y2 = xa(y, xm(len[k], s));
        b.seg(x, y, x2, y2, hw, C_LIMB);
        x = x2; y = y2;
    }
}

// Safety-Gymnasium velocity tasks (kinds 33-37)
template <int K>
__device__ void scene_velocity(Builder& b, const float* st, bool cost) {
    using C = VelCfg<K>;
    constexpr int Q0 = C::Q0;
    const int col = cost ? C_COST : C_ROBOT;
    if constexpr (K == ENV_SWIMMER_VEL) {   // top-down: the head along the heading, the two links behind it
        b.window(0.0f, 0.0f, 1.0f, 1.0f);
        const float c = st[1], s = st[2];
        b.seg(0.0f, 0.0f, xm(0.35f, c), xm(0.35f, s), 0.06f, col);
        const float len[2] = {0.35f, 0.35f};
        limbs<2>(b, 0.0f, 0.0f, -c, -s, st + Q0, len, 0.05f);
        b.gauge(xm(st[3], c), C::VCOST, false);
    } else if constexpr (K == ENV_ANT_VEL) {   // top-down: the torso, its heading and four two-link legs
        b.window(0.0f, 0.0f, 1.2f, 1.2f);
        const float c = st[2], s = st[3];
        constexpr float H = 0.70710678f;
        const float dc[4] = {H, -H, -H, H}, ds[4] = {H, H, -H, -H};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            float lc = c, ls = s;
            turn(lc, ls, dc[k], ds[k]);
            const float q[2] = {st[Q0 + k], st[Q0 + 4 + k]};
            const float len[2] = {0.35f, 0.35f};
            limbs<2>(b, 0.0f, 0.0f, lc, ls, q, len, 0.05f);
        }
        b.robot(0.0f, 0.0f, c, s, 0.2f, 0.4f, 0.06f, cost);
        const float vx = xm(st[4], c), vy = xm(st[4], s);
        b.gauge(xq(xa(xm(vx, vx), xm(vy, vy))), C::VCOST, false);
    } else {   // side view following the torso: ground, torso at its height and pitch, the legs
        constexpr bool CHEETAH = K == ENV_HALF_CHEETAH_VEL;
        const float z = st[0];
        float sn, cs;
        wide_sincos(st[2], sn, cs);
        b.window(0.0f, CHEETAH ? 0.7f : 1.0f, CHEETAH ? 1.5f : 1.3f, CHEETAH ? 1.0f : 1.3f);
        b.box(b.sc.x0, b.sc.y0, b.sc.x1, 0.0f, C_GROUND);
        const float len[3] = {0.45f, 0.5f, 0.2f};
        if constexpr (CHEETAH) {   // a horizontal torso, the back leg (q0-2) at its rear, the front leg (q3-5) at its front
            const float hx = xm(0.5f, cs), hy = xm(0.5f, sn);
            const float bx = xs(0.0f, hx), by = xs(z, hy), fx = hx, fy = xa(z, hy);
            const float clen[3] = {0.3f, 0.3f, 0.2f};
            limbs<3>(b, bx, by, sn, xs(0.0f, cs), st + Q0, clen, 0.04f);
            limbs<3>(b, fx, fy, sn, xs(0.0f, cs), st + Q0 + 3, clen, 0.04f);
            b.seg(bx, by, fx, fy, 0.06f, col);
        } else {   // an upright torso; Hopper's leg (q0-2), Walker2d's right (q0-2) and left (q3-5) legs from its hip
            const float hx = xm(0.2f, sn), hy = xm(0.2f, cs);
            const float px = hx, py = xs(z, hy);
            limbs<3>(b, px, py, sn, xs(0.0f, cs), st + Q0, len, 0.04f);
            if constexpr (K == ENV_WALKER2D_VEL) limbs<3>(b, px, py, sn, xs(0.0f, cs), st + Q0 + 3, len, 0.04f);
            b.seg(px, py, xs(0.0f, hx), xa(z, hy), 0.06f, col);
        }
        b.gauge(st[4], C::VCOST, false);
    }
}

// the built-in kinds' scenes (declared in render.cuh)
template <int K>
__device__ void scene(Builder& b, float* st, uint32_t seed, uint32_t env, uint32_t ep, bool cost) {
    if constexpr (K <= ENV_DRONE_RUN && K != ENV_POINT_GOAL) scene_bullet<K>(b, st, cost);
    else if constexpr (K < ENV_HALF_CHEETAH_VEL) scene_nav<K>(b, st, seed, env, ep, cost);
    else scene_velocity<K>(b, st, cost);
}

}  // namespace render

// the renderer of a known kind: a built-in kind's table, or the launcher registered for a plugin kind
// (fsrl_env_register_renderer), NULL when it has none
static const fsrl_env_renderer_t* env_renderer(int kind) {
    switch (kind) {
#define RENDER_TABLE_CASE(K)                                          \
    case K: {                                                         \
        static constexpr fsrl_env_renderer_t t = render_table<K>();   \
        return &t;                                                    \
    }
        ENV_KINDS(RENDER_TABLE_CASE)
#undef RENDER_TABLE_CASE
        default: return env_plugin_renderer(kind);
    }
}

}  // namespace fsrl

using namespace fsrl;

extern "C" int fsrl_env_render(const fsrl_rollout_t* r, const int32_t* ids, int n, int height, int width,
                               const float* last_cost, uint8_t* out, void* stream) {
    FSRL_REQUIRE(r != nullptr, "fsrl_env_render: null descriptor");
    FSRL_REQUIRE(env_table(r->kind) != nullptr, "fsrl_env_render: unknown env kind %d", r->kind);
    FSRL_REQUIRE(r->E > 0, "fsrl_env_render: E must be positive");
    FSRL_REQUIRE(n >= 1, "fsrl_env_render: n = %d must be at least 1", n);
    int rc = check_ids("fsrl_env_render", r, ids, n);
    if (rc) return rc;
    FSRL_REQUIRE(height >= 16 && height <= 1024 && width >= 16 && width <= 1024,
                 "fsrl_env_render: frame size %d x %d outside [16, 1024]", height, width);
    FSRL_REQUIRE(out != nullptr, "fsrl_env_render: null output");
    FSRL_REQUIRE(r->env_state && r->env_t && r->ep_idx, "fsrl_env_render: null state pointer");
    const fsrl_env_renderer_t* t = env_renderer(r->kind);
    FSRL_REQUIRE(t != nullptr,
                 "fsrl_env_render: env kind %d is a user-defined env whose struct has no draw: it has no renderer",
                 r->kind);
    return t->render(r, ids, n, height, width, last_cost, out, stream);
}
