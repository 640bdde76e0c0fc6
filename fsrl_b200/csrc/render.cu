// RGB frames of the device envs (fsrl_env_render): E * H * W independent coverage tests against a per-env scene.
//
// One CTA draws one env's frame over a band of rows.  Thread 0 decodes the env's scene from env_state (and, where
// step / observe regenerate a layout from the reset's Philox stream, through the same envs.cuh functions) into a
// list of at most MAX_PRIM primitives in shared memory: axis-aligned boxes, discs / rings and capsule segments, each
// with a palette colour.  Then every thread shades pixels: pixel (i, j) samples the world point at its centre,
// (x0 + (j + 0.5) sx, y1 - (i + 0.5) sy), and takes the colour of the LAST primitive covering it (painter's order;
// walked backwards, the first hit wins).  No antialiasing.  Coverage uses only the exact helpers of envs.cuh and
// compares squared distances, so tests/render_twin.py reproduces every pixel bit for bit in numpy float32.
// The band is staged in shared memory with the alignment the global bytes have mod 16 and stored as 16-byte words.
// Read-only on the env: nothing but `out` is written.  The scenes of every family are documented in DESIGN §7.
#include "rollout.cuh"

namespace fsrl {
namespace render {

constexpr int TPB = 256;
constexpr int MAX_PRIM = 32;   // Goal2 uses 25
constexpr int BAND_BYTES = 12288;   // staged bytes per CTA: rows = clamp(BAND_BYTES / (3 W), 1, H)

enum PrimType { PRIM_BOX = 0, PRIM_DISC = 1, PRIM_SEG = 2 };

// the palette (mirrored in tests/render_twin.py)
enum Colour { C_BG, C_FLOOR, C_WALL, C_CIRCLE, C_ROBOT, C_HEADING, C_COST, C_HAZARD, C_VASE, C_GOAL, C_BUTTON,
              C_GREMLIN, C_BOX, C_PILLAR, C_GROUND, C_LIMB, C_GAUGE_BG, C_GAUGE, C_MARK, C_TICK, N_COLOUR };
__constant__ uint8_t PALETTE[N_COLOUR][3] = {
    {24, 24, 32},    {54, 58, 70},   {120, 40, 40},  {70, 160, 90},  {70, 130, 230}, {250, 250, 250}, {240, 60, 40},
    {150, 60, 170},  {90, 200, 220}, {60, 210, 80},  {230, 190, 50}, {240, 120, 30}, {200, 150, 90},  {140, 140, 150},
    {90, 80, 60},    {180, 200, 240}, {60, 60, 60},  {80, 200, 120}, {250, 250, 250}, {80, 84, 100}};

// box: x in [a, c], y in [b, d].  disc: (x - a)^2 + (y - b)^2 in [c, d].
// seg: p = (x - a, y - b), t = clamp(p.(c, d) / e, 0, 1) (0 when e = 0), |p - t (c, d)|^2 <= f.
struct Prim { int type, colour; float a, b, c, d, e, f; };

struct Scene {
    float x0, x1, y0, y1;   // the view window
    int n;
    Prim p[MAX_PRIM];
};

struct Builder {
    Scene& sc;
    __device__ void put(int type, int colour, float a, float b, float c, float d, float e, float f) {
        if (sc.n < MAX_PRIM) sc.p[sc.n++] = Prim{type, colour, a, b, c, d, e, f};
    }
    __device__ void box(float x0, float y0, float x1, float y1, int col) { put(PRIM_BOX, col, x0, y0, x1, y1, 0.0f, 0.0f); }
    __device__ void disc(float cx, float cy, float r, int col) { put(PRIM_DISC, col, cx, cy, 0.0f, xm(r, r), 0.0f, 0.0f); }
    __device__ void ring(float cx, float cy, float r0, float r1, int col) {
        put(PRIM_DISC, col, cx, cy, xm(r0, r0), xm(r1, r1), 0.0f, 0.0f);
    }
    __device__ void seg(float ax, float ay, float bx, float by, float hw, int col) {
        const float dx = xs(bx, ax), dy = xs(by, ay);
        put(PRIM_SEG, col, ax, ay, dx, dy, xa(xm(dx, dx), xm(dy, dy)), xm(hw, hw));
    }
    // the window centred on (cx, cy) with half-extents (hx, hy)
    __device__ void window(float cx, float cy, float hx, float hy) {
        sc.x0 = xs(cx, hx); sc.x1 = xa(cx, hx); sc.y0 = xs(cy, hy); sc.y1 = xa(cy, hy);
    }
    // the robot: a disc of radius r and a heading segment of length hl from its centre
    __device__ void robot(float x, float y, float c, float s, float r, float hl, float hw, bool cost) {
        disc(x, y, r, cost ? C_COST : C_ROBOT);
        seg(x, y, xa(x, xm(hl, c)), xa(y, xm(hl, s)), hw, C_HEADING);
    }
    // a gauge along the bottom edge (a speed; its bar takes the cost colour past the mark) or the left edge (the
    // drone's altitude): value v on a scale [0, 2 * lim] with the mark at lim
    __device__ void gauge(float v, float lim, bool vertical) {
        const float L = xs(sc.x1, sc.x0), H = xs(sc.y1, sc.y0);
        const float frac = fminf(1.0f, fmaxf(0.0f, xd(v, xm(2.0f, lim))));
        const int col = !vertical && v > lim ? C_COST : C_GAUGE;
        if (!vertical) {
            const float g0 = xa(sc.x0, xm(L, 0.05f)), g1 = xs(sc.x1, xm(L, 0.05f));
            const float h0 = xa(sc.y0, xm(H, 0.03f)), h1 = xa(sc.y0, xm(H, 0.07f));
            const float gl = xs(g1, g0), m = xa(g0, xm(0.5f, gl)), mw = xm(L, 0.004f);
            box(g0, h0, g1, h1, C_GAUGE_BG);
            box(g0, h0, xa(g0, xm(frac, gl)), h1, col);
            box(xs(m, mw), xs(h0, xm(H, 0.01f)), xa(m, mw), xa(h1, xm(H, 0.01f)), C_MARK);
        } else {
            const float g0 = xa(sc.y0, xm(H, 0.05f)), g1 = xs(sc.y1, xm(H, 0.05f));
            const float h0 = xa(sc.x0, xm(L, 0.03f)), h1 = xa(sc.x0, xm(L, 0.07f));
            const float gl = xs(g1, g0), m = xa(g0, xm(0.5f, gl)), mw = xm(H, 0.004f);
            box(h0, g0, h1, g1, C_GAUGE_BG);
            box(h0, g0, h1, xa(g0, xm(frac, gl)), col);
            box(xs(h0, xm(L, 0.01f)), xs(m, mw), xa(h1, xm(L, 0.01f)), xa(m, mw), C_MARK);
        }
    }
    // the episode's progress t / T as a thin bar along the top edge
    __device__ void progress(int t, int T) {
        const float L = xs(sc.x1, sc.x0), H = xs(sc.y1, sc.y0);
        const float frac = fminf(1.0f, xd((float)t, (float)T));
        box(sc.x0, xs(sc.y1, xm(H, 0.015f)), xa(sc.x0, xm(frac, L)), sc.y1, C_MARK);
    }
};

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

// the scene of env e into sc (one thread; kept out of line so the pixel loop's registers stay its own)
template <int K>
__device__ __noinline__ void decode(Scene& sc, const float* env_state, int E, int e, uint32_t seed, uint32_t ep, int t,
                                    bool cost) {
    float st[ENV_MAX_S];
#pragma unroll
    for (int i = 0; i < Env<K>::S; ++i) st[i] = env_state[(size_t)i * E + e];
    Builder b{sc};
    sc.n = 0;
    if constexpr (K <= ENV_DRONE_RUN && K != ENV_POINT_GOAL) scene_bullet<K>(b, st, cost);
    else if constexpr (K < ENV_HALF_CHEETAH_VEL) scene_nav<K>(b, st, seed, (uint32_t)e, ep, cost);
    else scene_velocity<K>(b, st, cost);
    b.progress(t, Env<K>::T);
}

__device__ __forceinline__ bool covers(const Prim& p, float x, float y) {
    if (p.type == PRIM_BOX) return x >= p.a && x <= p.c && y >= p.b && y <= p.d;
    const float ux = xs(x, p.a), uy = xs(y, p.b);
    if (p.type == PRIM_DISC) {
        const float d2 = xa(xm(ux, ux), xm(uy, uy));
        return d2 >= p.c && d2 <= p.d;
    }
    float t = 0.0f;
    if (p.e > 0.0f) t = fminf(1.0f, fmaxf(0.0f, xd(xa(xm(ux, p.c), xm(uy, p.d)), p.e)));
    const float ex = xs(ux, xm(t, p.c)), ey = xs(uy, xm(t, p.d));
    return xa(xm(ex, ex), xm(ey, ey)) <= p.f;
}

// grid (bands, images): CTA (b, k) draws rows [b * rows, ...) of the frames k, k + gridDim.y, ...
template <int K>
__global__ void __launch_bounds__(TPB) render_kernel(const fsrl_rollout_t r, const __grid_constant__ EnvIds ids, int H,
                                                     int W, int rows, const float* __restrict__ last_cost,
                                                     uint8_t* __restrict__ out) {
    __shared__ Scene sc;
    __shared__ __align__(16) uint8_t band[BAND_BYTES + 16];
    const int r0 = blockIdx.x * rows;
    const int nr = min(rows, H - r0);
    const int npx = nr * W;
    for (int k = blockIdx.y; k < ids.n; k += gridDim.y) {
        if (threadIdx.x == 0) {
            const int e = env_of_row(ids, k);
            decode<K>(sc, r.env_state, r.E, e, r.seed_env, r.ep_idx[e] - 1u, r.env_t[e],
                      last_cost != nullptr && last_cost[e] > 0.0f);
        }
        uint8_t* g = out + ((size_t)(ids.i0 + k) * H + r0) * W * 3;
        const int pad = (int)(reinterpret_cast<uintptr_t>(g) & 15u);
        __syncthreads();
        const float sx = xd(xs(sc.x1, sc.x0), (float)W), sy = xd(xs(sc.y1, sc.y0), (float)H);
        for (int p = threadIdx.x; p < npx; p += TPB) {
            const int i = r0 + p / W, j = p % W;
            const float x = xa(sc.x0, xm((float)j + 0.5f, sx)), y = xs(sc.y1, xm((float)i + 0.5f, sy));
            int col = C_BG;
            for (int q = sc.n - 1; q >= 0; --q)
                if (covers(sc.p[q], x, y)) { col = sc.p[q].colour; break; }
            uint8_t* o = band + pad + 3 * p;
            o[0] = PALETTE[col][0]; o[1] = PALETTE[col][1]; o[2] = PALETTE[col][2];
        }
        __syncthreads();
        // the bytes [0, nb) of g: a head up to the first 16-byte boundary, 16-byte words, a tail
        const int nb = 3 * npx;
        const int head = min(nb, (16 - pad) & 15);
        const int nw = (nb - head) / 16;
        for (int q = threadIdx.x; q < head; q += TPB) g[q] = band[pad + q];
        for (int q = threadIdx.x; q < nw; q += TPB)
            reinterpret_cast<uint4*>(g + head)[q] = reinterpret_cast<const uint4*>(band + pad + head)[q];
        for (int q = head + 16 * nw + threadIdx.x; q < nb; q += TPB) g[q] = band[pad + q];
        __syncthreads();
    }
}

template <int K>
int launch(const fsrl_rollout_t& r, const int32_t* ids, int n, int H, int W, const float* last_cost, uint8_t* out,
           cudaStream_t s) {
    const int rows = max(1, min(H, BAND_BYTES / (3 * W)));
    return for_id_chunks(ids, n, [&](const EnvIds& c) {
        const dim3 grid((H + rows - 1) / rows, min(c.n, 65535));
        render_kernel<K><<<grid, TPB, 0, s>>>(r, c, H, W, rows, last_cost, out);
        FSRL_LAUNCH_CHECK();
        return FSRL_OK;
    });
}

}  // namespace render
}  // namespace fsrl

using namespace fsrl;

extern "C" int fsrl_env_render(const fsrl_rollout_t* r, const int32_t* ids, int n, int height, int width,
                               const float* last_cost, uint8_t* out, void* stream) {
    FSRL_REQUIRE(r != nullptr, "fsrl_env_render: null descriptor");
    FSRL_REQUIRE(!env_plugin(r->kind), "fsrl_env_render: env kind %d is a user-defined env, which has no renderer",
                 r->kind);
    FSRL_REQUIRE(env_kind_known(r->kind), "fsrl_env_render: unknown env kind %d", r->kind);
    FSRL_REQUIRE(r->E > 0, "fsrl_env_render: E must be positive");
    FSRL_REQUIRE(n >= 1, "fsrl_env_render: n = %d must be at least 1", n);
    FSRL_REQUIRE(ids != nullptr || n == r->E, "fsrl_env_render: without ids, n must be E = %d (got %d)", r->E, n);
    if (ids)
        for (int i = 0; i < n; ++i)
            FSRL_REQUIRE(ids[i] >= 0 && ids[i] < r->E, "fsrl_env_render: ids[%d] = %d outside [0, E = %d)", i, ids[i],
                         r->E);
    FSRL_REQUIRE(height >= 16 && height <= 1024 && width >= 16 && width <= 1024,
                 "fsrl_env_render: frame size %d x %d outside [16, 1024]", height, width);
    FSRL_REQUIRE(out != nullptr, "fsrl_env_render: null output");
    FSRL_REQUIRE(r->env_state && r->env_t && r->ep_idx, "fsrl_env_render: null state pointer");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    int rc = FSRL_OK;
    DISPATCH_KIND(r->kind, rc = render::launch<K>(*r, ids, n, height, width, last_cost, out, s));
    return rc;
}
