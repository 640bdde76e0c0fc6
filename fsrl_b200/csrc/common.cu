// C-ABI plumbing shared by every entry point: thread-local error text, version, device info;
// the W2 mirror kernel of every learner.
#include "arena.cuh"
#include "fsrl_b200.h"
#include <stdarg.h>
#include <string.h>

namespace fsrl {
static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int sm_count() {
    static int cached[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (cached[dev] == 0) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        cached[dev] = n;
    }
    return cached[dev];
}

__global__ void w2_mirror_kernel(const W2Mirror mr, int H) {
    const float* src = mr.w2t[blockIdx.y];
    const int tt = blockIdx.x;
    w2_tile(mr.w2n[blockIdx.y], H, (tt / (H / 32)) * 32, (tt % (H / 32)) * 32,
            [&](int k, int o) { return src[(size_t)k * H + o]; });
}

int launch_w2_mirror(const W2Mirror& mr, int n_nets, int H, cudaStream_t s) {
    FSRL_REQUIRE(n_nets >= 1 && n_nets <= W2_MIRROR_MAX_NETS, "w2 mirror: %d nets in one launch", n_nets);
    w2_mirror_kernel<<<dim3((H / 32) * (H / 32), n_nets), 256, 0, s>>>(mr, H);
    FSRL_LAUNCH_CHECK();
    return FSRL_OK;
}
}  // namespace fsrl

extern "C" const char* fsrl_last_error(void) { return fsrl::g_err; }
extern "C" int fsrl_abi_version(void) { return FSRL_ABI_VERSION; }
namespace fsrl { unsigned long long g_launches = 0; }
extern "C" unsigned long long fsrl_launch_count(void) { return fsrl::g_launches; }
extern "C" int fsrl_sm_count(void) { return fsrl::sm_count(); }

// sizes of the descriptor structs, checked against the ctypes mirrors at import time
extern "C" size_t fsrl_abi_sizeof(int which) {
    switch (which) {
        case 0: return sizeof(fsrl_mlp3_t);
        case 1: return sizeof(fsrl_collect_stats_t);
        case 2: return sizeof(fsrl_rollout_t);
        case 3: return sizeof(fsrl_ppo_update_t);
        case 4: return sizeof(fsrl_netref_t);
        case 5: return sizeof(fsrl_netlist_t);
        case 6: return sizeof(fsrl_engine_t);
        case 7: return sizeof(fsrl_eng_input_t);
        case 8: return sizeof(fsrl_offpolicy_t);
        case 9: return sizeof(fsrl_cpo_t);
        case 10: return sizeof(fsrl_cvpo_t);
        case 11: return sizeof(fsrl_traj_row_t);
        case 12: return sizeof(fsrl_traj_scan_t);
        case 13: return sizeof(fsrl_traj_arena_t);
        case 14: return sizeof(fsrl_host_step_t);
        case 15: return sizeof(fsrl_obs_rms_t);
        case 16: return sizeof(fsrl_host_norm_t);
        case 17: return sizeof(fsrl_env_plugin_t);
        case 18: return sizeof(fsrl_env_renderer_t);
        default: return 0;
    }
}
