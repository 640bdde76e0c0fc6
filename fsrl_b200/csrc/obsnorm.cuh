// Observation normalization on the device (obsnorm.cu): the launchers the collect paths compose with their
// own kernels.  See fsrl_obs_rms_t in fsrl_b200.h for the statistics and the normalization.
#pragma once
#include "common.cuh"
#include "fsrl_b200.h"

namespace fsrl {

// Which env ids a pass takes.  Collect passes read the rollout state, the others the mask of the workspace.
enum ObsNormSel : int {
    OBS_SEL_MASK = 0,       // mask[e]
    OBS_SEL_STEPPED = 1,    // mask[e] (the snapshot of active before the step) unless the collect had finished
    OBS_SEL_RESTARTED = 2,  // mask[e] && active[e] && env_t[e] == 0: reset by the resolve kernel; the pass then
                            // leaves mask[e] = active[e] && !finished, the snapshot of the next step
};

// One update + normalize pass over x[E][D].  ring: also write each normalized row to its env's ring slot
// b_ptr[e] - 1 (b_obs_next), when a.b_obs_next is set.
struct ObsNormPass {
    const fsrl_obs_rms_t* n;
    float* x;
    int E, sel, ring;
    const fsrl_rollout_t* a;   // the collect passes only
};

int launch_obs_norm(const ObsNormPass& p, cudaStream_t s);
// mask[e] = active[e] && !finished for every env: the snapshot before the first step of fsrl_rollout_norm_steps
int launch_obs_norm_snapshot(const fsrl_rollout_t& a, const fsrl_obs_rms_t& n, cudaStream_t s);
// The rows of the envs ids[0..count) (device ids; NULL: row k is env k): optionally copy rows_in[k] to
// x[ids[k]], update and normalize them in x, optionally copy x[ids[k]] to out[k].
int launch_obs_norm_rows(const fsrl_obs_rms_t& n, float* x, int E, const int* ids, int count, const float* rows_in,
                         float* out, cudaStream_t s);
// out[k] = x[ids[k]] (device ids) for k < count
int launch_obs_gather(const float* x, int D, const int* ids, int count, float* out, cudaStream_t s);
// the argument checks shared by the entry points
int check_obs_rms(const char* fn, const fsrl_obs_rms_t* n, int E, int D);

}  // namespace fsrl
