// The launcher tables of the velocity kinds (envs.cuh Velocity), in a translation unit of their own so that their
// kernels compile in parallel with rollout.cu, which looks the tables up here.
#include "rollout.cuh"

namespace fsrl {

const fsrl_env_plugin_t* env_table_vel(int kind) {
    switch (kind) {
        ENV_KINDS_VEL(ENV_TABLE_CASE)
        default: return nullptr;
    }
}

}  // namespace fsrl
