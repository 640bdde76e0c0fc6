// The built-in SafetyCarCircle-v0 struct with a draw that restates the library's Car Circle scene through the
// drawing contract: its frames must be bit-identical to the built-in kind's.
#include "envs.cuh"
#include "render.cuh"

struct UserEnv : fsrl::Env<fsrl::ENV_CAR_CIRCLE> {
    __device__ static void draw(const float* st, uint32_t, uint32_t, uint32_t, bool cost, fsrl::render::Builder& b) {
        using namespace fsrl::render;
        constexpr float R = fsrl::carc::R, XLIM = fsrl::carc::XLIM, RR = 0.1f;
        b.window(0.0f, 0.0f, 1.3f * R, 1.3f * R);
        b.box(b.sc.x0, b.sc.y0, -XLIM, b.sc.y1, C_WALL);
        b.box(XLIM, b.sc.y0, b.sc.x1, b.sc.y1, C_WALL);
        b.ring(0.0f, 0.0f, 0.98f * R, 1.02f * R, C_CIRCLE);
        b.robot(st[0], st[1], st[2], st[3], RR, 2.0f * RR, 0.35f * RR, cost);
    }
};
