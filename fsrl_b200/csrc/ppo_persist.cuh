// Persistent wgmma PPO-Lagrangian update (csrc/ppo_persist.cu): one launch per repeat.
#pragma once
#include "common.cuh"
#include "fsrl_b200.h"

namespace fsrl {
// floats of workspace (operand images, partial buffers, flags) the persistent path needs
size_t ppo_persist_ws_floats(int n_nets, int D, int H);
// floats every peer-mapped exchange buffer needs (gradient tiles, small-parameter slices)
size_t ppo_persist_p2p_floats(int n_nets);
// shape / mode / co-residency gate: everything else takes the three-launch chain of csrc/ppo.cu
bool ppo_persist_supported(const fsrl_ppo_update_t& u, long long n_total, int batch_size);
// `ug` carries the gathered (contiguous) batch and the per-minibatch advantage statistics
int ppo_persist_run(const fsrl_ppo_update_t& ug, int n_mb, int stats_slot0, long long adam_t0, cudaStream_t s);
}  // namespace fsrl
