// The rollout launchers of the Button and Push kinds (envs.cuh NavButton / NavPush), instantiated in a
// translation unit of their own so that they compile in parallel with rollout.cu, which dispatches to them.
#include "rollout.cuh"

namespace fsrl {

ROLLOUT_BP_KINDS(ROLLOUT_LAUNCHERS, )

}  // namespace fsrl
