// The launcher tables of the Button and Push kinds (envs.cuh NavButton / NavPush), in a translation unit of their
// own so that their kernels compile in parallel with rollout.cu, which looks the tables up here.
#include "rollout.cuh"

namespace fsrl {

const fsrl_env_plugin_t* env_table_bp(int kind) {
    switch (kind) {
        ENV_KINDS_BP(ENV_TABLE_CASE)
        default: return nullptr;
    }
}

}  // namespace fsrl
