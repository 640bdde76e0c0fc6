// The rollout launchers of the velocity kinds (envs.cuh Velocity), instantiated in a translation unit of their own
// so that they compile in parallel with rollout.cu, which dispatches to them.
#include "rollout.cuh"

namespace fsrl {

ROLLOUT_VEL_KINDS(ROLLOUT_LAUNCHERS, )

}  // namespace fsrl
