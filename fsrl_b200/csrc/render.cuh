// The rasterizer of fsrl_env_render: E * H * W independent coverage tests against a per-env scene.  Shared by the
// library (render.cu, the scenes of the built-in kinds) and the env plugins (env_plugin.cu, a UserEnv's draw).
//
// One CTA draws one env's frame over a band of rows.  Thread 0 decodes the env's scene from env_state (scene<K>:
// render.cu for the built-in kinds, env_plugin.cu for a plugin's) into a list of at most MAX_PRIM primitives in
// shared memory: axis-aligned boxes, discs / rings and capsule segments, each with a palette colour.  Then every
// thread shades pixels: pixel (i, j) samples the world point at its centre, (x0 + (j + 0.5) sx, y1 - (i + 0.5) sy),
// and takes the colour of the LAST primitive covering it (painter's order; walked backwards, the first hit wins).  No
// antialiasing.  Coverage uses only the exact helpers of envs.cuh and compares squared distances, so
// tests/render_twin.py reproduces every pixel bit for bit in numpy float32.
// The band is staged in shared memory with the alignment the global bytes have mod 16 and stored as 16-byte words.
// Read-only on the env: nothing but `out` is written.  The scenes and the drawing contract are documented in DESIGN §7.
#ifndef FSRL_RENDER_CUH
#define FSRL_RENDER_CUH

#include "rollout.cuh"

namespace fsrl {
namespace render {

constexpr int TPB = 256;
constexpr int MAX_PRIM = 32;   // Goal2 uses 25; a plugin's draw gets MAX_PRIM - 1, the progress bar takes the last
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

// The scene of kind K: the window and primitives of one env, from st (a local copy of its S state floats) and the
// (seed, env, ep) its reset / observe / step receive; cost is last_cost[e] > 0.  Defined for the built-in kinds in
// render.cu and for a plugin's ENV_USER in env_plugin.cu (through UserEnv::draw).
template <int K>
__device__ void scene(Builder& b, float* st, uint32_t seed, uint32_t env, uint32_t ep, bool cost);

// the scene of env e into sc and the progress bar (one thread; kept out of line so the pixel loop's registers stay
// its own)
template <int K>
__device__ __noinline__ void decode(Scene& sc, const float* env_state, int E, int e, uint32_t seed, uint32_t ep, int t,
                                    bool cost) {
    float st[ENV_MAX_S];
#pragma unroll
    for (int i = 0; i < Env<K>::S; ++i) st[i] = env_state[(size_t)i * E + e];
    Builder b{sc};
    sc.n = 0;
    scene<K>(b, st, seed, (uint32_t)e, ep, cost);
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

// the frames of kind K (fsrl_env_render after its argument checks)
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

// The renderer table of kind K: render::launch<K> behind the C signature of fsrl_env_renderer_t.  fsrl_env_render
// reaches a kind through such a table: render.cu defines the built-in kinds', env_plugin.cu a drawing plugin's.
template <int K>
constexpr fsrl_env_renderer_t render_table() {
    return {FSRL_ABI_VERSION, 0,
            [](const fsrl_rollout_t* r, const int32_t* ids, int n, int height, int width, const float* last_cost,
               uint8_t* out, void* s) {
                return render::launch<K>(*r, ids, n, height, width, last_cost, out, static_cast<cudaStream_t>(s));
            }};
}

}  // namespace fsrl

#endif  // FSRL_RENDER_CUH
