// HazardDash (tests/envs/hazard_dash.h) with a scene: the arena floor, the goal, the 12 hazards, the robot with its
// velocity as the heading (0.5 s ahead) and the energy on a vertical gauge with the mark at 1.  19 primitives.
#define UserEnv HazardDashBase
#include "../envs/hazard_dash.h"
#undef UserEnv
#include "render.cuh"

struct UserEnv : HazardDashBase {
    __device__ static void draw(const float* st, uint32_t, uint32_t, uint32_t, bool cost, fsrl::render::Builder& b) {
        using namespace fsrl::render;
        using namespace hazard_dash;
        b.window(0.0f, 0.0f, 1.1f * ARENA, 1.1f * ARENA);
        b.box(-ARENA, -ARENA, ARENA, ARENA, C_FLOOR);
        b.disc(st[4], st[5], GOAL_R, C_GOAL);
        for (int h = 0; h < NHAZ; ++h) b.disc(st[8 + 2 * h], st[9 + 2 * h], HAZ_R, C_HAZARD);
        b.robot(st[0], st[1], st[2], st[3], 0.1f, 0.5f, 0.035f, cost);
        b.gauge(st[6], 1.0f, true);
    }
};
