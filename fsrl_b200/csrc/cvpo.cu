// CVPO gradient steps on the device: the off-policy step's n-step targets and critic regression
// (offpolicy.cuh), then the E-step and M-step of Constrained Variational Policy Optimization on the
// generic MLP engine (engine.cu) plus the four small kernels below.
//
// Replaces (reference):
//   fsrl/policy/cvpo.py:206-222 _target_q / process_fn, :224-246 forward (unsquashed dist.sample()),
//       :248-276 critics_loss, :278-287 _estep_dual_loss, :289-317 gaussian_kl, :319-420 policy_loss,
//       :422-430 learn, :202-204 sync_weight
//
// Random draws come from the Philox stream KEY_CVPO (DESIGN.md §4): counter (row, step_lo,
// 8*step_hi + chunk, stream) with stream 0 = the next action of the n-step target (row = b) and
// stream 1 = the K particles of the E-step (row = k*B + b); chunk c covers action dims 4c..4c+3.
#include "arena.cuh"
#include "offpolicy.cuh"

namespace fsrl {

constexpr uint32_t KEY_CVPO = 0x4356504Fu;        // 'CVPO'
constexpr float CVPO_DUAL_EPS = 1.1920929e-06f;    // np.finfo(np.float32).eps * 10 (cvpo.py:163)
constexpr int ESTEP_T = 256, MSTEP_T = 256;

// mu / sigma of a Gaussian actor head row (ActorProb.forward): conditioned sigma from the head's
// second half, otherwise exp(sigma_param)
__device__ __forceinline__ void cvpo_head(const fsrl_cvpo_t& d, const float* o, const float* log_sigma, int j,
                                          float& mu, float& sig) {
    const int A = d.off.A;
    mu = d.off.bounded ? d.off.max_action * tanhf(o[j]) : o[j];
    sig = d.cond_sigma ? expf(fminf(fmaxf(o[A + j], d.off.sigma_min), d.off.sigma_max)) : expf(log_sigma[j]);
}

__device__ __forceinline__ void cvpo_noise(const fsrl_cvpo_t& d, uint32_t row, unsigned long long step, uint32_t stream,
                                           float (&eps)[8]) {
#pragma unroll
    for (int c = 0; c < 2; ++c) {
        if (4 * c < d.off.A) {
            uint32_t rr[4];
            Philox::gen(row, (uint32_t)step, (uint32_t)(step >> 32) * 8u + (uint32_t)c, stream, d.off.seed, KEY_CVPO, rr);
            gauss_pair(rr[0], rr[1], eps[4 * c], eps[4 * c + 1]);
            gauss_pair(rr[2], rr[3], eps[4 * c + 2], eps[4 * c + 3]);
        }
    }
}

// _target_q's action: dist.sample() of the CURRENT actor at obs_next[terminal] (no squash, no clip)
__global__ void cvpo_next_action_kernel(const fsrl_cvpo_t d, int B, unsigned long long step) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    float eps[8];
    cvpo_noise(d, (uint32_t)b, step, 0u, eps);
    const float* o = d.off.actor_out + (size_t)b * OD_LD;
    for (int j = 0; j < d.off.A; ++j) {
        float mu, sig;
        cvpo_head(d, o, d.log_sigma, j, mu, sig);
        d.off.w_act_next[(size_t)b * d.off.A + j] = fmaf(sig, eps[j], mu);
    }
}

// old_dist.sample((K,)) (cvpo.py:332-334): particle row r = k*B + b, its observation row
// part_idx[r] = idx[b] for the Q pass; the k = 0 rows also keep (mu_old, std_old) for the M-step
__global__ void cvpo_particle_kernel(const fsrl_cvpo_t d, const int* __restrict__ idx, int B, unsigned long long step) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= d.K * B) return;
    const int b = r % B, A = d.off.A;
    float eps[8];
    cvpo_noise(d, (uint32_t)r, step, 1u, eps);
    const float* o = d.off.actor_old_out + (size_t)b * OD_LD;
    for (int j = 0; j < A; ++j) {
        float mu, sig;
        cvpo_head(d, o, d.log_sigma_old, j, mu, sig);
        d.particles[(size_t)r * A + j] = fmaf(sig, eps[j], mu);
        if (r < B) { d.mu_old[(size_t)b * A + j] = mu; d.std_old[(size_t)b * A + j] = sig; }
    }
    d.part_idx[r] = idx[b];
}

__device__ __forceinline__ float cvpo_qmin(const fsrl_offpolicy_t& o, int i, int r) {
    if (o.twin) return fminf(o.q_out[2 * i][(size_t)r * OD_LD], o.q_out[2 * i + 1][(size_t)r * OD_LD]);
    return o.q_out[i][(size_t)r * OD_LD];
}

// E-step (cvpo.py:346-363), one CTA, fixed-order reductions.  comb starts as min-Q_r of every particle and,
// like the reference's in-place `combined_q -= lambda * q_c` on q_values[0], loses lambda*q_c once more in
// every dual iteration and once more for the weights.  Per iteration the dual gradients are closed-form:
//   d/d eta    = eps_kl + mean_b(lse_b - log K) - mean_b(sum_k p_kb c_kb) / eta,   lse_b = logsumexp_k(c_kb / eta)
//   d/d lambda = qc_thres - mean_b(sum_k p_kb q_c,kb),                              p = softmax_k(c / eta)
// Each row is shifted by its largest c before the division: with x_k = (c_k - cm_b) / eta the eta term's row is
// log(sum_k e^x_k) - sum_k p_k x_k, the entropy of the weights (at most log K), and the weights carry no exponent
// error of size |c| / eta.  Unshifted, both are differences of numbers of size |c| / eta.
__global__ void __launch_bounds__(ESTEP_T) cvpo_estep_kernel(const fsrl_cvpo_t d, int B, float* __restrict__ stat) {
    __shared__ double red[ESTEP_T / 32];
    __shared__ float s_dual[2];
    const fsrl_offpolicy_t& o = d.off;
    const int K = d.K, C = o.C, tid = threadIdx.x;
    float* st = d.estep_state;
    for (int i = 0; i < C; ++i) {                                   // estep/val_q{i}: mean of the n-step targets
        double v = 0.0;
        for (int b = tid; b < B; b += ESTEP_T) v += (double)o.w_target[(size_t)i * B + b];
        v = block_sum<ESTEP_T / 32>(v, red);
        if (tid == 0) stat[FSRL_CVPO_ST_VAL_Q0 + i] = (float)(v / B);
    }
    for (int r = tid; r < K * B; r += ESTEP_T) d.comb[r] = cvpo_qmin(o, 0, r);
    if (tid == 0) { s_dual[0] = st[0]; s_dual[1] = C > 1 ? st[1] : 0.f; }
    __syncthreads();
    const float logK = logf((float)K);
    for (int it = 0; it < d.estep_iters; ++it) {
        const float eta = s_dual[0], lam = s_dual[1];
        // Adam's bias corrections, in every thread before the rows: pow is a call, and few values are live here.
        // st[6] was last written by thread 0 before the barrier.
        const float t = st[6] + 1.0f;
        const double bc1 = 1.0 - pow(0.9, (double)t), bc2 = 1.0 - pow(0.999, (double)t);
        const AdamStep ad = {0.1f, 0.999f, 0.001f, (float)sqrt(bc2), 1e-8f, (float)(-(d.estep_dual_lr / bc1))};
        double s_lse = 0.0, s_ent = 0.0, s_pq = 0.0;
        for (int b = tid; b < B; b += ESTEP_T) {
            float cm = -INFINITY;
            for (int k = 0; k < K; ++k) {
                const int r = k * B + b;
                float c = d.comb[r];
                if (C > 1) c = __fsub_rn(c, __fmul_rn(lam, cvpo_qmin(o, 1, r)));
                d.comb[r] = c;
                cm = fmaxf(cm, c);
            }
            float se = 0.f, sx = 0.f, pq = 0.f;
            for (int k = 0; k < K; ++k) {
                const int r = k * B + b;
                const float x = (d.comb[r] - cm) / eta;
                const float e = expf(x);
                se += e; sx += e * x;
                if (C > 1) pq += e * cvpo_qmin(o, 1, r);
            }
            const float lse = logf(se);
            s_lse += (double)(cm / eta + lse - logK);
            s_ent += (double)(lse - sx / se - logK);
            s_pq += (double)(pq / se);
        }
        s_lse = block_sum<ESTEP_T / 32>(s_lse, red);
        s_ent = block_sum<ESTEP_T / 32>(s_ent, red);
        s_pq = block_sum<ESTEP_T / 32>(s_pq, red);
        if (tid == 0) {
            const float m_lse = (float)(s_lse / B), m_ent = (float)(s_ent / B), m_pq = (float)(s_pq / B);
            float loss = eta * d.estep_kl + eta * m_lse;
            const float g[2] = {d.estep_kl + m_ent, d.qc_thres - m_pq};
            if (C > 1) loss += lam * d.qc_thres;
            for (int i = 0; i < C; ++i) {
                float m = st[2 + i], v = st[4 + i];
                st[i] = adam_update(st[i], g[i], m, v, ad);
                st[2 + i] = m; st[4 + i] = v;
            }
            st[6] = t;
            stat[FSRL_CVPO_ST_ESTEP_LOSS] = loss;
            s_dual[0] = st[0]; s_dual[1] = C > 1 ? st[1] : 0.f;
        }
        __syncthreads();
    }
    if (tid == 0) {                                                 // estep_dual.data.clamp_ (cvpo.py:352)
        for (int i = 0; i < C; ++i) {
            st[i] = fminf(fmaxf(st[i], CVPO_DUAL_EPS), d.estep_dual_max);
            stat[FSRL_CVPO_ST_DUAL0 + i] = st[i];
        }
        s_dual[0] = st[0]; s_dual[1] = C > 1 ? st[1] : 0.f;
    }
    __syncthreads();
    const float eta = s_dual[0], lam = s_dual[1];
    for (int b = tid; b < B; b += ESTEP_T) {                        // optimal_q -= ...; softmax over k (:360-363)
        float cm = -INFINITY;
        for (int k = 0; k < K; ++k) {
            const int r = k * B + b;
            float c = d.comb[r];
            if (C > 1) c = __fsub_rn(c, __fmul_rn(lam, cvpo_qmin(o, 1, r)));
            d.comb[r] = c;
            cm = fmaxf(cm, c);
        }
        float se = 0.f;
        for (int k = 0; k < K; ++k) {
            const int r = k * B + b;
            const float e = expf((d.comb[r] - cm) / eta);
            d.weights[r] = e;
            se += e;
        }
        for (int k = 0; k < K; ++k) d.weights[k * B + b] /= se;
    }
}

// One M-step iteration (cvpo.py:373-418), one CTA: the KL / MLE / entropy sums of the batch, the Adam step of
// (dual_mu, dual_std) with the clip of their uses, then d loss / d actor head for every row:
//   loss = -mean_kb w [log N(a; mu, std_old) + log N(a; mu_old, std)] + dmu (kl_mu - thr_mu) + dstd (kl_std - thr_std)
// mu goes through dist1 and kl_mu, std through dist2 and kl_std; then the tanh of a bounded mean, the clamp
// gate of a conditioned sigma, or (state-independent sigma) the extra column of sigma_param.
__global__ void __launch_bounds__(MSTEP_T) cvpo_mstep_kernel(const fsrl_cvpo_t d, int B, float* __restrict__ stat) {
    __shared__ double red[MSTEP_T / 32];
    __shared__ float s_dmu, s_dstd;
    const fsrl_offpolicy_t& o = d.off;
    const int K = d.K, A = o.A, tid = threadIdx.x;
    double s_klm = 0.0, s_kls = 0.0, s_ent = 0.0, s_mle = 0.0;
    for (int b = tid; b < B; b += MSTEP_T) {
        const float* out = o.actor_out + (size_t)b * OD_LD;
        float klm = 0.f, kls = 0.f, ent = 0.f, mle = 0.f;
        for (int j = 0; j < A; ++j) {
            float mu, sig;
            cvpo_head(d, out, d.log_sigma, j, mu, sig);
            const float mo = d.mu_old[(size_t)b * A + j], so = d.std_old[(size_t)b * A + j];
            const float vo = fmaxf(so * so, 1e-6f), v = fmaxf(sig * sig, 1e-6f);
            klm += 0.5f * (mo - mu) * (mo - mu) / vo;
            kls += 0.5f * (logf(v / vo) + vo / v - 1.0f);
            ent += 1.0f + 2.0f * LOG_SQRT_2PI + logf(so) + logf(sig);
            const float lso = logf(so), ls = logf(sig);
            for (int k = 0; k < K; ++k) {
                const float a = d.particles[((size_t)k * B + b) * A + j];
                const float z1 = (a - mu) / so, z2 = (a - mo) / sig;
                mle += d.weights[k * B + b] * (-0.5f * z1 * z1 - lso - 0.5f * z2 * z2 - ls - 2.0f * LOG_SQRT_2PI);
            }
        }
        s_klm += klm; s_kls += kls; s_ent += ent; s_mle += mle;
    }
    s_klm = block_sum<MSTEP_T / 32>(s_klm, red);
    s_kls = block_sum<MSTEP_T / 32>(s_kls, red);
    s_ent = block_sum<MSTEP_T / 32>(s_ent, red);
    s_mle = block_sum<MSTEP_T / 32>(s_mle, red);
    if (tid == 0) {
        float* st = d.mstep_state;
        const float kl_mu = (float)(s_klm / B), kl_std = (float)(s_kls / B);
        const float t = st[6] + 1.0f;
        const double bc1 = 1.0 - pow(0.9, (double)t), bc2 = 1.0 - pow(0.999, (double)t);
        const AdamStep ad = {0.1f, 0.999f, 0.001f, (float)sqrt(bc2), 1e-8f, (float)(-(d.mstep_dual_lr / bc1))};
        const float g[2] = {d.mstep_kl_mu - kl_mu, d.mstep_kl_std - kl_std};
        for (int i = 0; i < 2; ++i) {
            float m = st[2 + i], v = st[4 + i];
            st[i] = adam_update(st[i], g[i], m, v, ad);
            st[2 + i] = m; st[4 + i] = v;
        }
        st[6] = t;
        const float dmu = fminf(fmaxf(st[0], 0.f), d.mstep_dual_max), dstd = fminf(fmaxf(st[1], 0.f), d.mstep_dual_max);
        const float loss_mle = (float)(-s_mle / ((double)K * B));
        const float loss_kl = dmu * (kl_mu - d.mstep_kl_mu) + dstd * (kl_std - d.mstep_kl_std);
        stat[FSRL_CVPO_ST_KL_MU] = kl_mu; stat[FSRL_CVPO_ST_KL_STD] = kl_std;
        stat[FSRL_CVPO_ST_LOSS_KL] = loss_kl; stat[FSRL_CVPO_ST_LOSS_MLE] = loss_mle;
        stat[FSRL_CVPO_ST_LOSS_TOTAL] = loss_mle + loss_kl;
        stat[FSRL_CVPO_ST_DUAL_MU] = dmu; stat[FSRL_CVPO_ST_DUAL_STD] = dstd;
        stat[FSRL_CVPO_ST_ENTROPY] = (float)(s_ent / B);
        s_dmu = dmu; s_dstd = dstd;
    }
    __syncthreads();
    const float dmu = s_dmu, dstd = s_dstd;
    const float invKB = 1.0f / ((float)K * (float)B), invB = 1.0f / (float)B;
    for (int b = tid; b < B; b += MSTEP_T) {
        const float* out = o.actor_out + (size_t)b * OD_LD;
        float* dd = o.actor_dout + (size_t)b * OD_LD;
#pragma unroll
        for (int j = 0; j < OD_LD; j += 4) *reinterpret_cast<float4*>(dd + j) = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int j = 0; j < A; ++j) {
            float mu, sig;
            cvpo_head(d, out, d.log_sigma, j, mu, sig);
            const float mo = d.mu_old[(size_t)b * A + j], so = d.std_old[(size_t)b * A + j];
            float s0 = 0.f, s1 = 0.f, s2 = 0.f;                      // sum_k w, w (a - mu), w (a - mu_old)^2
            for (int k = 0; k < K; ++k) {
                const float w = d.weights[k * B + b], a = d.particles[((size_t)k * B + b) * A + j];
                s0 += w; s1 += w * (a - mu); s2 += w * (a - mo) * (a - mo);
            }
            const float vo = fmaxf(so * so, 1e-6f), s2raw = sig * sig, v = fmaxf(s2raw, 1e-6f);
            const float g_mu = -invKB * s1 / (so * so) + dmu * invB * (mu - mo) / vo;
            const float dkl_dv = 0.5f * (1.0f / v - vo / (v * v));
            const float g_sig = -invKB * (s2 / (sig * sig * sig) - s0 / sig)
                                + dstd * invB * (s2raw >= 1e-6f ? dkl_dv * 2.0f * sig : 0.f);
            if (o.bounded) {
                const float t = tanhf(out[j]);
                dd[j] = g_mu * o.max_action * (1.0f - t * t);
            } else {
                dd[j] = g_mu;
            }
            if (d.cond_sigma) {
                const float sraw = out[A + j];
                dd[A + j] = (sraw >= o.sigma_min && sraw <= o.sigma_max) ? g_sig * sig : 0.f;
            } else {
                dd[A + j] = g_sig * sig;                            // extra column: d loss / d sigma_param_j
            }
        }
    }
}

}  // namespace fsrl

using namespace fsrl;

#define CVPO_CHECK(call) do { int rc__ = (call); if (rc__) return rc__; } while (0)

// n_steps gradient steps of CVPO.update.  idx_all: [n_steps][B] sampled flat buffer indices (device, int32);
// the Adam step of the critics continues from critic_t0, the actor's from actor_t0 (mstep_iters per step).
extern "C" int fsrl_cvpo_steps(const fsrl_cvpo_t* d, const int* idx_all, int n_steps, int B,
                               long long critic_t0, long long actor_t0, unsigned long long noise_t0, float* stats,
                               void* stream) {
    FSRL_REQUIRE(d && idx_all && stats, "cvpo: null pointer");
    const fsrl_offpolicy_t* o = &d->off;
    FSRL_REQUIRE(o->world <= 1, "cvpo: world=%d: the CVPO update runs on a single GPU", o->world);
    FSRL_REQUIRE(o->C >= 1 && o->C <= 2, "cvpo: C=%d critic streams unsupported (reward + at most one cost)", o->C);
    FSRL_REQUIRE(o->A >= 1 && o->A <= 8, "cvpo: action dim A=%d out of range [1, 8]", o->A);
    FSRL_REQUIRE(d->K >= 1, "cvpo: sample_act_num K=%d must be positive", d->K);
    FSRL_REQUIRE(B >= 2 && (long long)d->K * B <= o->eng.bmax,
                 "cvpo: K*B = %d*%d exceeds the engine's bmax %d (or B < 2)", d->K, B, o->eng.bmax);
    FSRL_REQUIRE(d->estep_iters >= 1 && d->mstep_iters >= 1, "cvpo: estep_iter_num=%d / mstep_iter_num=%d must be >= 1",
                 d->estep_iters, d->mstep_iters);
    FSRL_REQUIRE(o->use_alpha == 0, "cvpo: the n-step target has no entropy term (use_alpha must be 0)");
    FSRL_REQUIRE(d->cond_sigma || (d->log_sigma && d->log_sigma_old), "cvpo: state-independent sigma needs log_sigma pointers");
    FSRL_REQUIRE(d->estep_state && d->mstep_state && d->particles && d->part_idx && d->mu_old && d->std_old && d->comb &&
                 d->weights, "cvpo: null work array");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int T = 128, G = (B + T - 1) / T;
    const int D = o->D, A = o->A, KB = d->K * B;
    for (int it = 0; it < n_steps; ++it) {
        const int* idx = idx_all + (size_t)it * B;
        float* stat = stats + (size_t)it * FSRL_CVPO_STATS;
        const unsigned long long step = noise_t0 + it;
        // ---- process_fn: n-step targets (cvpo.py:206-222) -----------------------------------------------
        CVPO_CHECK(fsrl_nstep_prepare(o, idx, B, stream));
        {
            fsrl_eng_input_t in = mk_in(o->b_obs_next, o->w_term_idx, D, nullptr, nullptr, 0);
            CVPO_CHECK(fsrl_engine_forward(&o->eng, &o->actor, &in, B, 0, stream));
            cvpo_next_action_kernel<<<G, T, 0, s>>>(*d, B, step);
            FSRL_LAUNCH_CHECK();
            fsrl_eng_input_t inq = mk_in(o->b_obs_next, o->w_term_idx, D, o->w_act_next, nullptr, A);
            CVPO_CHECK(fsrl_engine_forward(&o->eng, &o->critics_old, &inq, B, 0, stream));
            launch_nstep_target(*o, B, s);
            FSRL_LAUNCH_CHECK();
        }
        // ---- critics_loss (:248-276) -------------------------------------------------------------------------
        {
            fsrl_eng_input_t in = mk_in(o->b_obs, idx, D, o->b_act, idx, A);
            CVPO_CHECK(fsrl_engine_forward(&o->eng, &o->critics, &in, B, 1, stream));
            launch_critic_grad(*o, B, stat, s);
            FSRL_LAUNCH_CHECK();
            CVPO_CHECK(fsrl_engine_backward(&o->eng, &o->critics, B, 0, stream));
            CVPO_CHECK(fsrl_engine_wgrad(&o->eng, &o->critics, &in, B, 0, nullptr, stream));
            CVPO_CHECK(fsrl_engine_adam(&o->eng, &o->critics, o->critic_lr, 0.9, 0.999, 1e-8, critic_t0 + it + 1, 1.0, 0.0,
                                        nullptr, 0.0, stream));
        }
        // ---- E-step (:320-363): K particles of actor_old, Q of the updated critics, duals, weights ------------
        {
            fsrl_eng_input_t in = mk_in(o->b_obs, idx, D, nullptr, nullptr, 0);
            CVPO_CHECK(fsrl_engine_forward(&o->eng, &o->actor_old, &in, B, 0, stream));
            cvpo_particle_kernel<<<(KB + T - 1) / T, T, 0, s>>>(*d, idx, B, step);
            FSRL_LAUNCH_CHECK();
            fsrl_eng_input_t inq = mk_in(o->b_obs, d->part_idx, D, d->particles, nullptr, A);
            CVPO_CHECK(fsrl_engine_forward(&o->eng, &o->critics, &inq, KB, 0, stream));
            cvpo_estep_kernel<<<1, ESTEP_T, 0, s>>>(*d, B, stat);
            FSRL_LAUNCH_CHECK();
        }
        // ---- M-step (:369-418) --------------------------------------------------------------------------------
        {
            fsrl_eng_input_t in = mk_in(o->b_obs, idx, D, nullptr, nullptr, 0);
            for (int m = 0; m < d->mstep_iters; ++m) {
                CVPO_CHECK(fsrl_engine_forward(&o->eng, &o->actor, &in, B, 1, stream));
                cvpo_mstep_kernel<<<1, MSTEP_T, 0, s>>>(*d, B, stat);
                FSRL_LAUNCH_CHECK();
                CVPO_CHECK(fsrl_engine_backward(&o->eng, &o->actor, B, 0, stream));
                CVPO_CHECK(fsrl_engine_wgrad(&o->eng, &o->actor, &in, B, 0, nullptr, stream));
                CVPO_CHECK(fsrl_engine_adam(&o->eng, &o->actor, o->actor_lr, 0.9, 0.999, 1e-8,
                                            actor_t0 + (long long)it * d->mstep_iters + m + 1, 1.0, 0.0, nullptr, 0.0, stream));
            }
        }
        // ---- sync_weight (:202-204): critics_old only; the actor has no target network ------------------------------
        CVPO_CHECK(fsrl_engine_polyak(&o->eng, &o->critics_old, &o->critics, o->tau, stream));
    }
    return FSRL_OK;
}
