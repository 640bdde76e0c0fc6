// The PPO-Lagrangian loss of one minibatch row, shared by the three-launch chain (ppo.cu) and the persistent
// launch (ppo_persist.cu): the gradient at the head outputs and the row's terms of the minibatch statistics.
// The callers differ only in where the head and its gradient live.
#pragma once
#include "common.cuh"
#include "fsrl_b200.h"

namespace fsrl {

// slots of one minibatch's statistics block (FSRL_PPO_STATS floats); critic i's value loss goes to ST_VF0 + i
constexpr int ST_ACTOR_REW = 0, ST_ACTOR_SAFETY = 1, ST_KL = 2, ST_VF0 = 3, ST_ENTROPY = 5, ST_GRADNORM = 6;

// Actor row (fsrl/policy/ppo_lag.py:173-212): out = head outputs (the first A are the Gaussian's mean before the
// optional tanh bound), act = the row's action, ls / rsg = log sigma and 1 / sigma per action dimension,
// adv_r / adv_c = the row's reward / cost advantage, mean / rstd = mean and 1 / std of the minibatch's reward [0]
// and cost [1] advantages (ppo_lag.py:178-182), invB = 1 / minibatch size.
// g_mu[j] = d loss / d out[j], g_ls[j] = d loss / d log sigma[j] (zero for j >= A); st_rew, st_saf, st_kl are the
// row's terms of loss/actor_rew, loss/actor_safety and approx_kl (already divided by the minibatch size).
__device__ __forceinline__ void ppo_actor_row(const fsrl_ppo_update_t& u, const float* out, const float* act,
                                              const float* ls, const float* rsg, float logp_old, float adv_r,
                                              float adv_c, const float* mean, const float* rstd, float invB,
                                              float (&g_mu)[8], float (&g_ls)[8], float& st_rew, float& st_saf,
                                              float& st_kl) {
    const int A = u.A;
    float logp = 0.f, zz[8], dmu[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        zz[j] = dmu[j] = 0.f;
        if (j < A) {
            const float tnh = tanhf(out[j]);
            const float mu = u.bounded ? u.max_action * tnh : out[j];
            dmu[j] = u.bounded ? u.max_action * (1.0f - tnh * tnh) : 1.0f;
            zz[j] = (act[j] - mu) * rsg[j];
            logp += -0.5f * zz[j] * zz[j] - ls[j] - LOG_SQRT_2PI;
        }
    }
    const float ratio = expf(logp - logp_old);
    const float ar = (adv_r - mean[0]) * rstd[0];
    const float surr1 = ratio * ar;
    const float rc = fminf(fmaxf(ratio, 1.0f - u.eps_clip), 1.0f + u.eps_clip);
    const float surr2 = rc * ar;
    // d(-min(surr1, surr2)) / d ratio; ties split evenly like torch.min's backward
    const bool inside = (ratio >= 1.0f - u.eps_clip) && (ratio <= 1.0f + u.eps_clip);
    float g_ratio, lrew;   // d loss_rew / d ratio (before the 1 / B of the mean), loss_rew
    if (surr1 < surr2) { g_ratio = -ar; lrew = -surr1; }
    else if (surr1 > surr2) { g_ratio = inside ? -ar : 0.f; lrew = -surr2; }
    else { g_ratio = inside ? -ar : -0.5f * ar; lrew = -surr1; }
    if (u.dual_clip > 0.f && ar < 0.f) {
        // clip2 = max(min(surr1, surr2), dual_clip * adv) for negative advantages (:188-191)
        const float c1 = fminf(surr1, surr2), c2 = u.dual_clip * ar;
        if (c2 > c1) { g_ratio = 0.f; lrew = -c2; }
        else if (c2 == c1) { g_ratio *= 0.5f; }
    }
    float g_saf = 0.f, lsaf = 0.f;
    if (u.use_lagrangian && u.C > 1) {
        const float ac = (adv_c - mean[1]) * rstd[1];
        g_saf = ac * u.lagrangian;          // d mean(ratio * adv_c * lambda) / d ratio
        lsaf = ratio * ac * u.lagrangian;
    }
    // d loss / d logp = rescaling * (g_ratio + g_saf) * ratio / B
    const float gl = u.rescaling * (g_ratio + g_saf) * ratio * invB;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        g_mu[j] = g_ls[j] = 0.f;
        if (j < A) {
            g_mu[j] = gl * (zz[j] * rsg[j]) * dmu[j];
            g_ls[j] = gl * (zz[j] * zz[j] - 1.0f);
        }
    }
    st_rew = lrew * invB; st_saf = lsaf * invB; st_kl = (logp_old - logp) * invB;
}

// Critic row (critics_loss, ppo_lag.py:152-171): v = head output, ret = return target, v_old = the value stored with
// the batch (read only with value_clip).  Returns d loss / d v including vf_coef and 1 / B; *loss = the row's term
// of loss/vf_i.
__device__ __forceinline__ float ppo_value_row(const fsrl_ppo_update_t& u, float v, float ret, float v_old, float invB,
                                               float& loss) {
    float lv, gv;
    if (u.value_clip) {
        const float dv = fminf(fmaxf(v - v_old, -u.eps_clip), u.eps_clip);
        const float vc = v_old + dv;
        const float vf1 = (ret - v) * (ret - v), vf2 = (ret - vc) * (ret - vc);
        const bool in_clip = (v - v_old > -u.eps_clip) && (v - v_old < u.eps_clip);
        // d max(vf1, vf2) / d v; ties split evenly like torch.max's backward
        if (vf1 > vf2) { lv = vf1; gv = 2.0f * (v - ret); }
        else if (vf1 < vf2) { lv = vf2; gv = in_clip ? 2.0f * (vc - ret) : 0.f; }
        else { lv = vf1; gv = in_clip ? 2.0f * (v - ret) : (v - ret); }
    } else {
        lv = (ret - v) * (ret - v);
        gv = 2.0f * (v - ret);
    }
    loss = lv * invB;
    return u.vf_coef * gv * invB;
}

// entropy of the diagonal Gaussian policy: sum over the A action dimensions of 1/2 + log sqrt(2 pi) + log sigma
__device__ __forceinline__ float ppo_entropy(const float* ls, int A) {
    float ent = 0.f;
    for (int j = 0; j < A; ++j) ent += 0.5f + LOG_SQRT_2PI + ls[j];
    return ent;
}

}  // namespace fsrl
