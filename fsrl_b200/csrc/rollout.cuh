// The device side of rollout collection (see rollout.cu): the fused collect step, the caller-action step,
// the resolve pass, resets and the gym-protocol step, templated over the env kind, and the host launchers
// of a kind with the table that carries them to the C entry points of rollout.cu.
#pragma once
#include "envs.cuh"
#include "mlp.cuh"
#include "obsnorm.cuh"
#include "fsrl_b200.h"
#include <cstdlib>

namespace fsrl {

static_assert(sizeof(fsrl_mlp3_t) == sizeof(Mlp3), "ABI struct mismatch");
static_assert(FSRL_BOUND_CLIP == 1 && FSRL_BOUND_TANH == 2, "map_action() codes");

// buffer.add of one transition of env e (env-major sub-buffer ring; reserved keys of tianshou's buffer);
// a no-op when the collect stores nothing.  DC is the observation width when it is known at compile time
// (the device envs), else 0 and d gives it (host-stepped envs).  Every collect path stores through here.
template <int DC, int A>
__device__ __forceinline__ void ring_store(const fsrl_rollout_t& a, int e, int d, const float* obs, const float* on,
                                           const float* act, float logp, float rew, float cost, bool term, bool trunc) {
    const int D = DC ? DC : d;
    if (a.b_obs) {
        const int ptr = a.b_ptr[e];
        const size_t p = (size_t)e * a.cap + ptr;
#pragma unroll
        for (int k = 0; k < D; ++k) {
            a.b_obs[p * D + k] = obs[k];
            a.b_obs_next[p * D + k] = on[k];
        }
#pragma unroll
        for (int j = 0; j < A; ++j) a.b_act[p * A + j] = act[j];
        a.b_rew[p] = rew; a.b_cost[p] = cost; a.b_logp[p] = logp;
        a.b_term[p] = term ? 1 : 0; a.b_trunc[p] = trunc ? 1 : 0;
        a.b_ptr[e] = (ptr + 1 == a.cap) ? 0 : ptr + 1;
        const int len = a.b_len[e];
        if (len < a.cap) a.b_len[e] = len + 1;
    }
}

// Everything of one collect step that follows the policy's action, for env e: map_action, env.step,
// buffer.add of (obs, act, logp), statistics and the done bookkeeping.  The fused step and the
// caller-action step both end here, so the two collect paths apply the same episode rules.
template <int KIND>
__device__ __forceinline__ void collect_step_tail(const fsrl_rollout_t& a, int e, const float* obs,
                                                  const float* act, float logp) {
    using E_ = Env<KIND>;
    constexpr int D = E_::D, A = E_::A, S = E_::S;
    fsrl_collect_stats_t* st = a.stats;
    float aenv[A];
    // ---- map_action (base_policy.py:244-256) ---------------------------------------------------
#pragma unroll
    for (int j = 0; j < A; ++j)
        aenv[j] = map_action(act[j], a.action_bound, a.action_scaling, a.act_low[j], a.act_high[j]);
    // ---- env.step ---------------------------------------------------------------------------------
    float s[S];
#pragma unroll
    for (int i = 0; i < S; ++i) s[i] = a.env_state[(size_t)i * a.E + e];
    float rew, cost;
    bool term;
    const uint32_t ep = a.ep_idx[e] - 1u;
    E_::step(s, aenv, a.seed_env, (uint32_t)e, ep, rew, cost, term);
    const int t_new = a.env_t[e] + 1;
    const bool trunc = (t_new >= a.max_steps) && !term;
    const bool done = term || trunc;
    float on[D];
    E_::observe(s, on, a.seed_env, (uint32_t)e, ep);

    ring_store<D, A>(a, e, D, obs, on, act, logp, rew, cost, term, trunc);
    // ---- statistics (:326, :338-348) --------------------------------------------------------------
    atomicAdd(&st->step_count, 1ull);
    if (cost != 0.f) atomicAdd(&st->total_cost, (double)cost);
    const double er = a.ep_rew[e] + (double)rew;
    const int el = a.ep_len[e] + 1;
    a.ep_rew[e] = er; a.ep_len[e] = el;
    a.env_t[e] = t_new;

    if (done) {
        if (a.inline_done) {
            // n_episode <= ready envs: every finished env is surplus (:357-363) -> retire it
            atomicAdd(&st->sum_ep_rew, er);
            atomicAdd(&st->sum_ep_len, (unsigned long long)el);
            atomicAdd(term ? &st->term_count : &st->trunc_count, 1);
            a.active[e] = 0;
            a.ep_rew[e] = 0.0; a.ep_len[e] = 0;
            const int c = atomicAdd(&st->episode_count, 1) + 1;
            if (c >= st->n_episode) st->finished_next = 1;
        } else {
            a.done_now[e] = term ? 1 : 2;
        }
    }
#pragma unroll
    for (int i = 0; i < S; ++i) a.env_state[(size_t)i * a.E + e] = s[i];
#pragma unroll
    for (int k = 0; k < D; ++k) a.obs_cur[(size_t)e * D + k] = on[k];
}

// The policy's raw action act[A] for env e from the actor's head output `out` (Philox sampling keyed by
// (e, act_ctr[e]), the heads, log-prob and DDPG noise; random mode draws uniform actions instead); returns
// its log-prob.  Both fused paths sample through here: the device-env step and the host-env step.
template <int A>
__device__ __forceinline__ float policy_sample(const fsrl_rollout_t& a, int e, const float* out, float (&act)[A]) {
    float mu[A], sig[A];
    float logp = 0.f;
    const uint32_t ctr = a.act_ctr[e];
    float eps[(A + 3) / 4 * 4];
    if (a.mode == FSRL_MODE_TRAIN || a.mode == FSRL_MODE_RANDOM) {
#pragma unroll
        for (int c = 0; c < (A + 3) / 4; ++c) {
            uint32_t rr[4];
            Philox::gen((uint32_t)e, ctr, (uint32_t)c, 0u, a.seed_act, KEY_ACT, rr);
            if (a.mode == FSRL_MODE_RANDOM) {
#pragma unroll
                for (int j = 0; j < 4; ++j) eps[4 * c + j] = usym(rr[j]);   // uniform in [-1, 1)
            } else {
                gauss_pair(rr[0], rr[1], eps[4 * c], eps[4 * c + 1]);
                gauss_pair(rr[2], rr[3], eps[4 * c + 2], eps[4 * c + 3]);
            }
        }
        a.act_ctr[e] = ctr + 1u;
    }
#pragma unroll
    for (int j = 0; j < A; ++j) {
        if (a.mode == FSRL_MODE_RANDOM) {
            // action_space.sample() then map_action_inverse (fast_collector.py:258-264):
            // uniform in [low, high] maps to uniform in [-1, 1] under scaling
            float v = eps[j];
            if (a.action_bound == FSRL_BOUND_TANH) v = 0.5f * (log1pf(v) - log1pf(-v));
            act[j] = v; mu[j] = 0.f; sig[j] = 1.f;
            continue;
        }
        if (a.head == FSRL_HEAD_GAUSS_INDEP) {
            // tianshou ActorProb, state-independent sigma (collect_dataset.py:199-214)
            mu[j] = a.bounded ? a.max_action * tanhf(out[j]) : out[j];
            sig[j] = expf(__ldg(a.log_sigma + j));
        } else if (a.head == FSRL_HEAD_GAUSS_COND || a.head == FSRL_HEAD_GAUSS_COND_RAW) {
            mu[j] = a.bounded ? a.max_action * tanhf(out[j]) : out[j];
            sig[j] = expf(fminf(fmaxf(out[A + j], a.sigma_min), a.sigma_max));
        } else {   // FSRL_HEAD_DETERMINISTIC (tianshou Actor): max_action * tanh(logits)
            mu[j] = a.max_action * tanhf(out[j]);
            sig[j] = 0.f;
        }
        if (a.mode == FSRL_MODE_EVAL || a.head == FSRL_HEAD_DETERMINISTIC) act[j] = mu[j];
        else act[j] = fmaf(sig[j], eps[j], mu[j]);               // dist.sample()  (:189)
    }
    if (a.head == FSRL_HEAD_GAUSS_COND && a.mode != FSRL_MODE_RANDOM) {
        // SAC (sac_lag.py:147-183): squash, log-prob with the tanh correction
        float lp = 0.f;
#pragma unroll
        for (int j = 0; j < A; ++j) {
            const float z = (a.mode == FSRL_MODE_EVAL) ? 0.f : eps[j];
            lp += -0.5f * z * z - logf(sig[j]) - LOG_SQRT_2PI;
            const float sq = tanhf(act[j]);
            lp -= logf(1.0f - sq * sq + a.tanh_eps);
            act[j] = sq;
        }
        logp = lp;
    } else if ((a.head == FSRL_HEAD_GAUSS_INDEP || a.head == FSRL_HEAD_GAUSS_COND_RAW) && a.mode != FSRL_MODE_RANDOM) {
        // Independent(Normal(mu, sigma), 1).log_prob(act)  (ppo_lag.py:148; CVPO, cvpo.py:245, no squash)
        float lp = 0.f;
#pragma unroll
        for (int j = 0; j < A; ++j) {
            const float z = (act[j] - mu[j]) / sig[j];
            lp += -0.5f * z * z - logf(sig[j]) - LOG_SQRT_2PI;
        }
        logp = lp;
    }
    if (a.head == FSRL_HEAD_DETERMINISTIC && a.mode == FSRL_MODE_TRAIN && a.expl_sigma > 0.f) {
        // DDPG exploration_noise (ddpg_lag.py:225-231): act + N(0, sigma^2)
#pragma unroll
        for (int j = 0; j < A; ++j) act[j] = fmaf(a.expl_sigma, eps[j], act[j]);
    }
    return logp;
}

// The policy's action for env e from the actor's head output `out`, then collect_step_tail.  obs: the
// observation the actor saw.
template <int KIND>
__device__ __forceinline__ void fused_step_env(const fsrl_rollout_t& a, int e, const float* out, const float* obs) {
    float act[Env<KIND>::A];
    const float logp = policy_sample<Env<KIND>::A>(a, e, out, act);
    collect_step_tail<KIND>(a, e, obs, act, logp);
}

// n_steps collect steps of the fused path in one launch: a CTA owns a tile of R envs and steps it n_steps
// times, or until none of its envs is active.  Envs of different tiles never interact within a step, so
// this equals n_steps single-step launches when nothing between the steps changes which envs are active:
// the inline path, where a finished env retires.  The resolve path launches it with n_steps = 1, followed
// by rollout_resolve_kernel after every step.
template <int KIND, int H>
__global__ void __launch_bounds__(MLP_TPB, 1)
rollout_step_kernel(const fsrl_rollout_t a, int n_steps) {
    using E_ = Env<KIND>;
    using TT = MlpTile<H>;
    constexpr int D = E_::D;
    extern __shared__ __align__(16) float smem[];
    fsrl_collect_stats_t* st = a.stats;
    if (st->finished) return;

    const int tid = threadIdx.x;
    const int e0 = blockIdx.x * TT::R;
    const Mlp3& actor = *reinterpret_cast<const Mlp3*>(&a.actor);
    const MlpSmem<H> sm(smem, D, actor.out);
    constexpr int INP = TT::in_pad(D);
    float* xtile = sm.x;
    const int r = tid / TT::PARTS, part = tid % TT::PARTS;
    const int e = e0 + r;

    __shared__ int s_any;
    for (int step = 0; step < n_steps; ++step) {
        // tile-level early out: nothing active in this tile (the previous step's last barrier orders the
        // reads of s_any before this store)
        if (tid == 0) s_any = 0;
        __syncthreads();
        if (tid < TT::R) {
            const int et = e0 + tid;
            if (et < a.E && a.active[et]) s_any = 1;
        }
        __syncthreads();
        if (!s_any) return;

        // ---- stage the observation tile -----------------------------------------------------
        mlp_stage_rows<H>(sm, D, [&](int rr) -> const float* {
            const int et = e0 + rr;
            return et < a.E ? a.obs_cur + (size_t)et * D : nullptr;
        });
        __syncthreads();

        float out[MLP_MAX_OUT];
        if (a.mode != FSRL_MODE_RANDOM) {
            mlp_hidden_forward<H>(actor, sm);
            mlp_head_forward<H>(actor, sm, out);
        }

        // ---- one thread per env: sample, log-prob, map, step, store --------------------------
        if (part == 0 && e < a.E && a.active[e]) fused_step_env<KIND>(a, e, out, xtile + r * INP);
        // this step's stores to obs_cur / active are read by other threads of the tile in the next one
        __syncthreads();
    }
}

// One collect step with the caller's actions act[E][A] (the generic FastCollector path: any torch
// policy computes them).  The raw action is stored, as the reference stores `act`, and logp = 0, as
// in random mode; act_ctr does not move.  Followed by rollout_resolve_kernel like the fused step.
template <int KIND>
__global__ void __launch_bounds__(128) rollout_act_step_kernel(const fsrl_rollout_t a, const float* __restrict__ act_in) {
    constexpr int D = Env<KIND>::D, A = Env<KIND>::A;
    if (a.stats->finished) return;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= a.E || !a.active[e]) return;
    float act[A];
#pragma unroll
    for (int j = 0; j < A; ++j) act[j] = act_in[(size_t)e * A + j];
    collect_step_tail<KIND>(a, e, a.obs_cur + (size_t)e * D, act, 0.f);
}

// Resolve finished episodes in env order (general path, n_episode > n_env): count, retire the
// first `surplus` finished envs (fast_collector.py:357-363), reset the rest (:351).
template <int KIND>
__global__ void __launch_bounds__(1024) rollout_resolve_kernel(const fsrl_rollout_t a) {
    using E_ = Env<KIND>;
    constexpr int D = E_::D, S = E_::S;
    fsrl_collect_stats_t* st = a.stats;
    __shared__ int s_scan[1024];
    __shared__ int s_base, s_total, s_surplus;
    const int tid = threadIdx.x;
    if (st->finished) return;
    if (st->finished_next) {          // inline path signalled completion during the last step
        if (tid == 0) st->finished = 1;
        return;
    }
    if (a.inline_done) return;
    // pass 1: total number of done envs this step
    int local = 0;
    for (int e = tid; e < a.E; e += 1024) local += (a.active[e] && a.done_now[e]) ? 1 : 0;
    s_scan[tid] = local;
    __syncthreads();
    for (int o = 512; o > 0; o >>= 1) {
        if (tid < o) s_scan[tid] += s_scan[tid + o];
        __syncthreads();
    }
    if (tid == 0) {
        s_total = s_scan[0];
        const int epc = st->episode_count + s_total;
        int surplus = st->n_ready - (st->n_episode - epc);
        if (surplus < 0) surplus = 0;
        if (surplus > s_total) surplus = s_total;
        s_surplus = surplus;
        s_base = 0;
    }
    __syncthreads();
    const int total = s_total;
    if (total == 0) return;
    const int surplus = s_surplus;
    // pass 2: ordered walk in chunks of 1024 envs; rank = number of done envs with lower id
    for (int c0 = 0; c0 < a.E; c0 += 1024) {
        const int e = c0 + tid;
        const int flag = (e < a.E && a.active[e] && a.done_now[e]) ? 1 : 0;
        s_scan[tid] = flag;
        __syncthreads();
        for (int o = 1; o < 1024; o <<= 1) {      // Hillis-Steele inclusive scan
            int v = (tid >= o) ? s_scan[tid - o] : 0;
            __syncthreads();
            s_scan[tid] += v;
            __syncthreads();
        }
        const int rank = s_base + s_scan[tid] - flag;   // exclusive rank among done envs
        if (flag) {
            const bool term = a.done_now[e] == 1;
            atomicAdd(&st->sum_ep_rew, a.ep_rew[e]);
            atomicAdd(&st->sum_ep_len, (unsigned long long)a.ep_len[e]);
            atomicAdd(term ? &st->term_count : &st->trunc_count, 1);
            a.ep_rew[e] = 0.0; a.ep_len[e] = 0; a.done_now[e] = 0;
            if (rank < surplus) {
                a.active[e] = 0;
            } else {
                float s[S], o[D];
                const uint32_t ep = a.ep_idx[e];
                E_::reset(s, a.seed_env, (uint32_t)e, ep);
                a.ep_idx[e] = ep + 1u;
                a.env_t[e] = 0;
                E_::observe(s, o, a.seed_env, (uint32_t)e, ep);
                for (int i = 0; i < S; ++i) a.env_state[(size_t)i * a.E + e] = s[i];
                for (int k = 0; k < D; ++k) a.obs_cur[(size_t)e * D + k] = o[k];
            }
        }
        __syncthreads();
        if (tid == 1023) s_base += s_scan[1023];
        __syncthreads();
    }
    if (tid == 0) {
        st->episode_count += total;
        st->n_ready -= surplus;
        if (st->episode_count >= st->n_episode) st->finished = 1;
    }
}

// fresh episode in env e: its k-th reset draws Philox stream (e, k) on every path; returns obs in o
template <int KIND>
__device__ __forceinline__ void env_reset_one(const fsrl_rollout_t& a, int e, float* o) {
    using E_ = Env<KIND>;
    constexpr int D = E_::D, S = E_::S;
    float s[S];
    const uint32_t ep = a.ep_idx[e];
    E_::reset(s, a.seed_env, (uint32_t)e, ep);
    a.ep_idx[e] = ep + 1u;
    a.env_t[e] = 0;
    a.ep_rew[e] = 0.0; a.ep_len[e] = 0; a.done_now[e] = 0;
    E_::observe(s, o, a.seed_env, (uint32_t)e, ep);
    for (int i = 0; i < S; ++i) a.env_state[(size_t)i * a.E + e] = s[i];
    for (int k = 0; k < D; ++k) a.obs_cur[(size_t)e * D + k] = o[k];
}

// reset_env (fast_collector.py:131-152): fresh episode in every env; stats untouched
template <int KIND>
__global__ void env_reset_all_kernel(const fsrl_rollout_t a) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= a.E) return;
    float o[Env<KIND>::D];
    env_reset_one<KIND>(a, e, o);
}

// Env ids of rows [i0, i0 + n) of a gym-protocol call, passed by value (the ids are host data, checked
// on the host).  all != 0: row i is env i and e[] is unused.
constexpr int ENV_IDS_CHUNK = 512;
struct EnvIds {
    int n, i0, all, pad;
    int e[ENV_IDS_CHUNK];
};

__device__ __forceinline__ int env_of_row(const EnvIds& ids, int k) { return ids.all ? ids.i0 + k : ids.e[k]; }

// reset(id): fresh episode in the listed envs, obs[i] = the new observation of row i (obs may be NULL)
template <int KIND>
__global__ void __launch_bounds__(128) env_reset_ids_kernel(const fsrl_rollout_t a, const __grid_constant__ EnvIds ids,
                                                            float* __restrict__ obs) {
    constexpr int D = Env<KIND>::D;
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= ids.n) return;
    float o[D];
    env_reset_one<KIND>(a, env_of_row(ids, k), o);
    if (obs) {
        const size_t i = (size_t)(ids.i0 + k);
#pragma unroll
        for (int c = 0; c < D; ++c) obs[i * D + c] = o[c];
    }
}

// step(act, id): gymnasium's env.step with env-range actions act[n][A] (no map_action, no ring, no
// collect statistics).  Advances the same per-env state the collect reads (env_state, obs_cur, env_t,
// ep_rew, ep_len), so a later collect continues from it.
template <int KIND>
__global__ void __launch_bounds__(128) env_step_ids_kernel(const fsrl_rollout_t a, const __grid_constant__ EnvIds ids,
                                                           const float* __restrict__ act, float* __restrict__ obs_next,
                                                           float* __restrict__ rew_out, float* __restrict__ cost_out,
                                                           uint8_t* __restrict__ term_out, uint8_t* __restrict__ trunc_out) {
    using E_ = Env<KIND>;
    constexpr int D = E_::D, A = E_::A, S = E_::S;
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= ids.n) return;
    const size_t i = (size_t)(ids.i0 + k);
    const int e = env_of_row(ids, k);
    float aenv[A];
#pragma unroll
    for (int j = 0; j < A; ++j) aenv[j] = act[i * A + j];
    float s[S];
#pragma unroll
    for (int c = 0; c < S; ++c) s[c] = a.env_state[(size_t)c * a.E + e];
    float rew, cost;
    bool term;
    const uint32_t ep = a.ep_idx[e] - 1u;
    E_::step(s, aenv, a.seed_env, (uint32_t)e, ep, rew, cost, term);
    const int t_new = a.env_t[e] + 1;
    const bool trunc = (t_new >= a.max_steps) && !term;
    float on[D];
    E_::observe(s, on, a.seed_env, (uint32_t)e, ep);
    a.ep_rew[e] += (double)rew;
    a.ep_len[e] += 1;
    a.env_t[e] = t_new;
#pragma unroll
    for (int c = 0; c < S; ++c) a.env_state[(size_t)c * a.E + e] = s[c];
#pragma unroll
    for (int c = 0; c < D; ++c) {
        a.obs_cur[(size_t)e * D + c] = on[c];
        obs_next[i * D + c] = on[c];
    }
    rew_out[i] = rew; cost_out[i] = cost;
    term_out[i] = term ? 1 : 0; trunc_out[i] = trunc ? 1 : 0;
}

// one launch of rollout_step_kernel<KIND, H> over the tiles of all E envs, n_steps steps each; the kernel's
// dynamic shared memory limit is raised on its first launch
template <int KIND, int H>
int launch_step_tiles(const fsrl_rollout_t& a, int n_steps, cudaStream_t s) {
    using TT = MlpTile<H>;
    const size_t smem = TT::smem_bytes(Env<KIND>::D);
    static bool attr_done = false;
    if (!attr_done) {
        FSRL_CUDA(cudaFuncSetAttribute(rollout_step_kernel<KIND, H>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem));
        attr_done = true;
    }
    rollout_step_kernel<KIND, H><<<(a.E + TT::R - 1) / TT::R, MLP_TPB, smem, s>>>(a, n_steps);
    FSRL_LAUNCH_CHECK();
    return FSRL_OK;
}

// launch_step_tiles at the actor's hidden width
template <int KIND>
int launch_step_kernel(const fsrl_rollout_t& a, int n_steps, cudaStream_t s) {
    switch (a.actor.H) {
        case 64: return launch_step_tiles<KIND, 64>(a, n_steps, s);
        case 128: return launch_step_tiles<KIND, 128>(a, n_steps, s);
        case 256: return launch_step_tiles<KIND, 256>(a, n_steps, s);
        case 512: return launch_step_tiles<KIND, 512>(a, n_steps, s);
        default: set_error("rollout: hidden width %d unsupported (64/128/256/512)", a.actor.H); return FSRL_EINVAL;
    }
}

// n_steps steps of the fused kernel, each followed by the resolve kernel; or, with `one_launch`, all of them
// in one launch followed by one resolve (which turns finished_next into finished)
template <int KIND>
int launch_steps_h(const fsrl_rollout_t& a, int n_steps, bool one_launch, cudaStream_t s) {
    const int launches = one_launch ? 1 : n_steps, steps = one_launch ? n_steps : 1;
    for (int i = 0; i < launches; ++i) {
        const int rc = launch_step_kernel<KIND>(a, steps, s);
        if (rc) return rc;
        rollout_resolve_kernel<KIND><<<1, 1024, 0, s>>>(a);
        FSRL_LAUNCH_CHECK();
    }
    return FSRL_OK;
}

template <int KIND>
int launch_env_reset_all(const fsrl_rollout_t& a, cudaStream_t s) {
    env_reset_all_kernel<KIND><<<(a.E + 127) / 128, 128, 0, s>>>(a);
    FSRL_LAUNCH_CHECK();
    return FSRL_OK;
}

template <int KIND>
int launch_act_step(const fsrl_rollout_t& a, const float* act, cudaStream_t s) {
    rollout_act_step_kernel<KIND><<<(a.E + 127) / 128, 128, 0, s>>>(a, act);
    FSRL_LAUNCH_CHECK();
    rollout_resolve_kernel<KIND><<<1, 1024, 0, s>>>(a);
    FSRL_LAUNCH_CHECK();
    return FSRL_OK;
}

// launch(chunk) once per ENV_IDS_CHUNK rows of host ids (once over all E rows without ids)
template <typename F>
static int for_id_chunks(const int32_t* ids, int n, F&& launch) {
    EnvIds c;
    c.pad = 0;
    c.all = ids == nullptr;
    const int step = ids ? ENV_IDS_CHUNK : n;
    for (int i0 = 0; i0 < n; i0 += step) {
        c.i0 = i0;
        c.n = n - i0 < step ? n - i0 : step;
        if (ids)
            for (int k = 0; k < c.n; ++k) c.e[k] = ids[i0 + k];
        int rc = launch(c);
        if (rc) return rc;
    }
    return FSRL_OK;
}

template <int KIND>
int launch_env_step(const fsrl_rollout_t& a, const float* act, const int32_t* ids, int n, float* obs_next,
                           float* rew, float* cost, uint8_t* term, uint8_t* trunc, cudaStream_t s) {
    return for_id_chunks(ids, n, [&](const EnvIds& c) {
        env_step_ids_kernel<KIND><<<(c.n + 127) / 128, 128, 0, s>>>(a, c, act, obs_next, rew, cost, term, trunc);
        FSRL_LAUNCH_CHECK();
        return FSRL_OK;
    });
}

template <int KIND>
int launch_env_reset_ids(const fsrl_rollout_t& a, const int32_t* ids, int n, float* obs, cudaStream_t s) {
    return for_id_chunks(ids, n, [&](const EnvIds& c) {
        env_reset_ids_kernel<KIND><<<(c.n + 127) / 128, 128, 0, s>>>(a, c, obs);
        FSRL_LAUNCH_CHECK();
        return FSRL_OK;
    });
}

// n_steps vector steps of a collect over an env wrapped by VectorEnvNormObs (fsrl_rollout_norm_steps): per step
// the fused step kernel (act == NULL) or the caller-action one, the update + normalize pass over the envs that
// stepped (the snapshot of active in the workspace mask), the resolve kernel, and the pass over the envs it
// restarted, which also takes the snapshot for the next step.  The kernels are those of the unwrapped paths.
template <int KIND>
int launch_norm_steps(const fsrl_rollout_t& a, const fsrl_obs_rms_t& n, int n_steps, const float* act, cudaStream_t s) {
    const int H = a.actor.H;
    if (!act && H != 64 && H != 128 && H != 256 && H != 512) {
        set_error("rollout: hidden width %d unsupported (64/128/256/512)", H);
        return FSRL_EINVAL;
    }
    int rc = launch_obs_norm_snapshot(a, n, s);
    if (rc) return rc;
    const ObsNormPass stepped{&n, a.obs_cur, a.E, OBS_SEL_STEPPED, 1, &a};
    const ObsNormPass restarted{&n, a.obs_cur, a.E, OBS_SEL_RESTARTED, 0, &a};
    for (int i = 0; i < n_steps; ++i) {
        if (act) {
            rollout_act_step_kernel<KIND><<<(a.E + 127) / 128, 128, 0, s>>>(a, act);
            FSRL_LAUNCH_CHECK();
        } else if ((rc = launch_step_kernel<KIND>(a, 1, s))) {
            return rc;
        }
        if ((rc = launch_obs_norm(stepped, s))) return rc;
        rollout_resolve_kernel<KIND><<<1, 1024, 0, s>>>(a);
        FSRL_LAUNCH_CHECK();
        if ((rc = launch_obs_norm(restarted, s))) return rc;
    }
    return FSRL_OK;
}

// The launcher table of kind K: Env<K>'s widths and horizon and its six launchers behind the C signatures of
// fsrl_env_plugin_t.  Every env-dependent entry point reaches a kind through such a table (env_table(kind)): the
// built-in kinds' tables are defined in the translation unit of their group (ENV_KINDS_*), a plugin's in
// env_plugin.cu.
template <int K>
constexpr fsrl_env_plugin_t env_table() {
    return {FSRL_ABI_VERSION, Env<K>::D, Env<K>::A, Env<K>::S, Env<K>::T, 0,
            [](const fsrl_rollout_t* r, void* s) { return launch_env_reset_all<K>(*r, static_cast<cudaStream_t>(s)); },
            [](const fsrl_rollout_t* r, int n_steps, int one_launch, void* s) {
                return launch_steps_h<K>(*r, n_steps, one_launch != 0, static_cast<cudaStream_t>(s));
            },
            [](const fsrl_rollout_t* r, const float* act, void* s) {
                return launch_act_step<K>(*r, act, static_cast<cudaStream_t>(s));
            },
            [](const fsrl_rollout_t* r, const float* act, const int32_t* ids, int n, float* obs_next, float* rew,
               float* cost, uint8_t* term, uint8_t* trunc, void* s) {
                return launch_env_step<K>(*r, act, ids, n, obs_next, rew, cost, term, trunc,
                                          static_cast<cudaStream_t>(s));
            },
            [](const fsrl_rollout_t* r, const int32_t* ids, int n, float* obs, void* s) {
                return launch_env_reset_ids<K>(*r, ids, n, obs, static_cast<cudaStream_t>(s));
            },
            [](const fsrl_rollout_t* r, const fsrl_obs_rms_t* n, int n_steps, const float* act, void* s) {
                return launch_norm_steps<K>(*r, *n, n_steps, act, static_cast<cudaStream_t>(s));
            }};
}

// `case K:` of a switch over kinds that returns kind K's table, a constant-initialized static
#define ENV_TABLE_CASE(K)                                             \
    case K: {                                                         \
        static constexpr fsrl_env_plugin_t t = env_table<K>();        \
        return &t;                                                    \
    }

// host: the table of a Button or Push kind (rollout_bp.cu), of a velocity kind (rollout_vel.cu); NULL for any other
const fsrl_env_plugin_t* env_table_bp(int kind);
const fsrl_env_plugin_t* env_table_vel(int kind);
// host: the table of a built-in kind or of a registered plugin kind (rollout.cu); NULL for an unknown kind
const fsrl_env_plugin_t* env_table(int kind);
// host: the render launcher registered for a plugin kind (fsrl_env_register_renderer), NULL when it has none
const fsrl_env_renderer_t* env_plugin_renderer(int kind);
// host: the rows of a call over the envs ids[0..n) (host ids), or over all E envs in order when ids is NULL
int check_ids(const char* fn, const fsrl_rollout_t* a, const int32_t* ids, int n);

}  // namespace fsrl
