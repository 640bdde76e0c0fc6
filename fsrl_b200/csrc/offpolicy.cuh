// Pieces of the off-policy gradient step (offpolicy.cu) that CVPO's step (cvpo.cu) runs unchanged:
// the head-output stride of the engine scratch, the update's Philox key, engine inputs, and the
// launches of the n-step target and critic-regression kernels.
#pragma once
#include "common.cuh"
#include "fsrl_b200.h"

namespace fsrl {

constexpr int OD_LD = 16;    // row stride of the engine's out / dout scratch
constexpr uint32_t KEY_UPD = 0x55504454u;   // 'UPDT': noise stream of the update's rsample()

inline fsrl_eng_input_t mk_in(const float* xa, const int* ia, int Da, const float* xb, const int* ib, int Db) {
    fsrl_eng_input_t in;
    in.xa = xa; in.ia = ia; in.xb = xb; in.ib = ib; in.Da = Da; in.Db = Db;
    return in;
}

// w_target[i][b] = (min-over-heads Q'_i - alpha*logp') * vmask * gamma^k + partial_i (alpha only when d.use_alpha)
void launch_nstep_target(const fsrl_offpolicy_t& d, int B, cudaStream_t s);
// q_dout = d/dq of sum_i sum_heads mean((q - target_i)^2); stat[FSRL_OFF_ST_Q0 + i] += loss of stream i
void launch_critic_grad(const fsrl_offpolicy_t& d, int B, float* stat, cudaStream_t s);

}  // namespace fsrl
