// A tiny env (D = A = S = 1) whose draw never sets a window and emits 40 discs in a row at the height st[0]: the
// frame shows the default window [-1, 1] x [-1, 1] and only the first MAX_PRIM - 1 = 31 discs.
#include "envs.cuh"
#include "render.cuh"

struct UserEnv {
    static constexpr int D = 1, A = 1, S = 1, T = 20;

    __device__ static void reset(float* st, uint32_t seed, uint32_t env, uint32_t ep) {
        uint32_t r[4];
        fsrl::Philox::gen(env, ep, 0u, 0u, seed, fsrl::KEY_RESET, r);
        st[0] = fsrl::xm(fsrl::usym(r[0]), 0.5f);
    }
    __device__ static void observe(const float* st, float* o, uint32_t, uint32_t, uint32_t) { o[0] = st[0]; }
    __device__ static void step(float* st, const float* a, uint32_t, uint32_t, uint32_t, float& rew, float& cost,
                                bool& term) {
        st[0] = fminf(0.9f, fmaxf(-0.9f, fsrl::xa(st[0], fsrl::xm(a[0], 0.1f))));
        rew = 0.0f;
        cost = st[0] > 0.5f ? 1.0f : 0.0f;
        term = false;
    }
    __device__ static void draw(const float* st, uint32_t, uint32_t, uint32_t, bool cost, fsrl::render::Builder& b) {
        using namespace fsrl::render;
        for (int k = 0; k < 40; ++k)
            b.disc(fsrl::xa(-0.975f, fsrl::xm(0.05f, (float)k)), st[0], 0.024f,
                   k == 0 && cost ? C_COST : k % 2 ? C_GOAL : C_HAZARD);
    }
};
