// Rollout collection around host-stepped envs (gymnasium / tianshou env objects the device cannot run):
// one launch per vector step of FastCollector.collect (fast_collector.py:252-368) does the two device
// parts of the step, the host steps the envs in between.
//   store phase: buffer.add of the previous vector step (:333-335) through ring_store, the function the
//                device-env paths store with
//   act phase:   the actor forward on this step's observations in MlpTile<H> row tiles (:267-269), the
//                sampling / heads / log-prob / DDPG noise of policy_sample (:279-280) and map_action (:284)
// The observation width D is a runtime value (any host env up to FSRL_ENG_DX_LD - A); the kernel is
// instantiated per hidden width H and action width A.  A row's actor output does not depend on the other
// rows of its tile, so a host env sees the action the device-env kernel would compute for the same
// observation, key and counter, bit for bit.
#include "rollout.cuh"
#include "obsnorm.cuh"

#include <vector>

namespace fsrl {

// fsrl_host_step_t with the packed upload resolved into device pointers
struct HostStepArgs {
    const int *store_ids, *act_ids;
    const float *obs, *obs_next, *rew, *cost;
    const uint8_t *term, *trunc;
    float* scratch;   // [2][E][D + A + 1]
    float* act_out;   // [n_act][A]
    int D, n_store, n_act, parity;
};

template <int H, int A>
__global__ void __launch_bounds__(MLP_TPB, 1) host_collect_step_kernel(const fsrl_rollout_t a, const HostStepArgs h) {
    using TT = MlpTile<H>;
    extern __shared__ __align__(16) float smem[];
    const int D = h.D, W = D + A + 1;
    const int tid = threadIdx.x;

    // ---- store phase: the transitions of the previous step, from the other scratch half ----------------
    const float* prev = h.scratch + (size_t)(h.parity ^ 1) * a.E * W;
    for (int i = blockIdx.x * MLP_TPB + tid; i < h.n_store; i += gridDim.x * MLP_TPB) {
        const int e = h.store_ids[i];
        const float* s = prev + (size_t)e * W;
        ring_store<0, A>(a, e, D, s, h.obs_next + (size_t)i * D, s + D, s[D + A], h.rew[i], h.cost[i],
                         h.term[i] != 0, h.trunc[i] != 0);
    }

    // ---- act phase: one row tile of this step's observations per CTA ------------------------------------
    const int row0 = blockIdx.x * TT::R;
    if (row0 >= h.n_act) return;                 // uniform over the CTA: no barrier is skipped by a part of it
    const Mlp3& actor = *reinterpret_cast<const Mlp3*>(&a.actor);
    const MlpSmem<H> sm(smem, D, actor.out);
    const int inp = TT::in_pad(D);
    mlp_stage_rows<H>(sm, D, [&](int rr) -> const float* {
        const int k = row0 + rr;
        return k < h.n_act ? h.obs + (size_t)k * D : nullptr;
    });
    __syncthreads();
    float out[MLP_MAX_OUT];
    if (a.mode != FSRL_MODE_RANDOM) {
        mlp_hidden_forward<H>(actor, sm);
        mlp_head_forward<H>(actor, sm, out);
    }
    const int r = tid / TT::PARTS, part = tid % TT::PARTS;
    const int k = row0 + r;
    if (part == 0 && k < h.n_act) {
        const int e = h.act_ids[k];
        float act[A];
        const float logp = policy_sample<A>(a, e, out, act);
        float* s = h.scratch + (size_t)h.parity * a.E * W + (size_t)e * W;
        const float* x = sm.x + (size_t)r * inp;
        for (int c = 0; c < D; ++c) s[c] = x[c];
#pragma unroll
        for (int j = 0; j < A; ++j) {
            s[D + j] = act[j];
            h.act_out[(size_t)k * A + j] = map_action(act[j], a.action_bound, a.action_scaling, a.act_low[j], a.act_high[j]);
        }
        s[D + A] = logp;
    }
}

template <int H, int A>
static int launch_host_step(const fsrl_rollout_t& a, const HostStepArgs& h, cudaStream_t s) {
    using TT = MlpTile<H>;
    static bool attr_done = false;
    if (!attr_done) {     // sized for the widest observation an entry admits
        FSRL_CUDA(cudaFuncSetAttribute(host_collect_step_kernel<H, A>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)TT::smem_bytes(FSRL_ENG_DX_LD)));
        attr_done = true;
    }
    const int tiles = (h.n_act + TT::R - 1) / TT::R;
    const int stores = (h.n_store + MLP_TPB - 1) / MLP_TPB;
    const int grid = tiles > stores ? tiles : stores;
    host_collect_step_kernel<H, A><<<grid, MLP_TPB, TT::smem_bytes(h.D), s>>>(a, h);
    FSRL_LAUNCH_CHECK();
    return FSRL_OK;
}

template <int H>
static int dispatch_a(const fsrl_rollout_t& a, const HostStepArgs& h, int A, cudaStream_t s) {
    switch (A) {
        case 1: return launch_host_step<H, 1>(a, h, s);
        case 2: return launch_host_step<H, 2>(a, h, s);
        case 3: return launch_host_step<H, 3>(a, h, s);
        case 4: return launch_host_step<H, 4>(a, h, s);
        case 5: return launch_host_step<H, 5>(a, h, s);
        case 6: return launch_host_step<H, 6>(a, h, s);
        case 7: return launch_host_step<H, 7>(a, h, s);
        case 8: return launch_host_step<H, 8>(a, h, s);
        default: set_error("fsrl_host_collect_step: action width %d outside 1..8", A); return FSRL_EINVAL;
    }
}

}  // namespace fsrl

using namespace fsrl;

extern "C" size_t fsrl_host_pack_bytes(int D, int n_store, int n_act) {
    return sizeof(int32_t) * ((size_t)n_store + n_act) + sizeof(float) * ((size_t)n_act * D + (size_t)n_store * D + 2 * (size_t)n_store) +
           2 * (size_t)n_store;
}

// the wrapped pack (obs_rms set): the unwrapped layout, then from a 16-byte boundary fresh_ids | fresh_obs
extern "C" size_t fsrl_host_pack_norm_bytes(int D, int n_store, int n_act, int n_fresh) {
    const size_t base = (fsrl_host_pack_bytes(D, n_store, n_act) + 15) & ~(size_t)15;
    return base + sizeof(int32_t) * (size_t)n_fresh + sizeof(float) * (size_t)n_fresh * D;
}

// ids[0..n) each in [0, E) and listed once
static int check_host_ids(const char* what, const int32_t* ids, int n, int E, std::vector<unsigned char>& seen) {
    seen.assign(E, 0);
    for (int i = 0; i < n; ++i) {
        FSRL_REQUIRE(ids[i] >= 0 && ids[i] < E, "fsrl_host_collect_step: %s[%d] = %d outside [0, E = %d)", what, i, ids[i], E);
        FSRL_REQUIRE(!seen[ids[i]], "fsrl_host_collect_step: env %d listed twice in %s", ids[i], what);
        seen[ids[i]] = 1;
    }
    return FSRL_OK;
}

// both entry points; nrm == NULL: no normalization
static int host_collect_step(const fsrl_rollout_t* r, const fsrl_host_step_t* h, const fsrl_host_norm_t* nrm,
                             void* stream) {
    FSRL_REQUIRE(r != nullptr && h != nullptr, "fsrl_host_collect_step: null descriptor");
    const int E = r->E, D = h->D, A = h->A;
    FSRL_REQUIRE(E > 0, "fsrl_host_collect_step: E must be positive");
    FSRL_REQUIRE(A >= 1 && A <= 8, "fsrl_host_collect_step: action width %d outside 1..8", A);
    FSRL_REQUIRE(D >= 1 && D + A <= FSRL_ENG_DX_LD, "fsrl_host_collect_step: D = %d with A = %d outside D >= 1, D + A <= %d",
                 D, A, FSRL_ENG_DX_LD);
    const int H = r->actor.H;
    FSRL_REQUIRE(H == 64 || H == 128 || H == 256 || H == 512, "fsrl_host_collect_step: hidden width %d unsupported (64/128/256/512)", H);
    FSRL_REQUIRE(h->n_store >= 0 && h->n_store <= E && h->n_act >= 0 && h->n_act <= E,
                 "fsrl_host_collect_step: n_store = %d / n_act = %d outside [0, E = %d]", h->n_store, h->n_act, E);
    FSRL_REQUIRE(h->parity == 0 || h->parity == 1, "fsrl_host_collect_step: parity %d is not 0 or 1", h->parity);
    FSRL_REQUIRE(h->pack_host && h->pack_dev && h->scratch && h->act_dev && h->act_host && r->act_ctr,
                 "fsrl_host_collect_step: null pointer");
    if (h->n_act > 0 && r->mode != FSRL_MODE_RANDOM) {
        FSRL_REQUIRE(r->actor.in == D, "fsrl_host_collect_step: actor input dim %d != obs dim %d", r->actor.in, D);
        FSRL_REQUIRE(r->actor.w1t && r->actor.b1 && r->actor.w2t && r->actor.b2 && r->actor.w3t && r->actor.b3,
                     "fsrl_host_collect_step: null actor weights");
        // the conditioned-sigma heads read mu from out[0, A) and log-sigma from out[A, 2A)
        const bool cond = r->head == FSRL_HEAD_GAUSS_COND || r->head == FSRL_HEAD_GAUSS_COND_RAW;
        const int need = cond ? 2 * A : A;
        FSRL_REQUIRE(r->actor.out >= need && r->actor.out <= MLP_MAX_OUT,
                     "fsrl_host_collect_step: actor out dim %d outside [%d, %d] for head %d with A = %d",
                     r->actor.out, need, MLP_MAX_OUT, r->head, A);
        FSRL_REQUIRE(r->head != FSRL_HEAD_GAUSS_INDEP || r->log_sigma, "fsrl_host_collect_step: null log_sigma");
    }
    const bool norm = nrm != nullptr;
    const int n_fresh = norm ? nrm->n_fresh : 0;
    if (norm) {
        int rc = check_obs_rms("fsrl_host_collect_step", nrm->obs_rms, E, D);
        if (rc) return rc;
        FSRL_REQUIRE(nrm->obs_norm != nullptr, "fsrl_host_collect_step: null obs_norm");
        FSRL_REQUIRE(n_fresh >= 0 && n_fresh <= E, "fsrl_host_collect_step: n_fresh = %d outside [0, E = %d]", n_fresh, E);
    }
    if (h->n_store > 0 && !norm)
        FSRL_REQUIRE(r->b_obs && r->b_obs_next && r->b_act && r->b_rew && r->b_cost && r->b_logp && r->b_term && r->b_trunc &&
                     r->b_ptr && r->b_len && r->cap > 0,
                     "fsrl_host_collect_step: n_store = %d without a complete ring", h->n_store);
    const int32_t* ids = static_cast<const int32_t*>(h->pack_host);
    std::vector<unsigned char> seen;
    int rc = check_host_ids("store_ids", ids, h->n_store, E, seen);
    if (rc) return rc;
    rc = check_host_ids("act_ids", ids + h->n_store, h->n_act, E, seen);
    if (rc) return rc;
    const size_t fresh_off = (fsrl_host_pack_bytes(D, h->n_store, h->n_act) + 15) & ~(size_t)15;
    if (norm) {
        rc = check_host_ids("fresh_ids", reinterpret_cast<const int32_t*>(static_cast<const char*>(h->pack_host) + fresh_off),
                            n_fresh, E, seen);
        if (rc) return rc;
    }
    if (h->n_store == 0 && h->n_act == 0 && n_fresh == 0) return FSRL_OK;

    // resolve the packed layout on the device copy
    char* p = static_cast<char*>(h->pack_dev);
    HostStepArgs g;
    g.store_ids = reinterpret_cast<const int*>(p); p += sizeof(int32_t) * h->n_store;
    g.act_ids = reinterpret_cast<const int*>(p);   p += sizeof(int32_t) * h->n_act;
    g.obs = reinterpret_cast<const float*>(p);     p += sizeof(float) * (size_t)h->n_act * D;
    g.obs_next = reinterpret_cast<const float*>(p); p += sizeof(float) * (size_t)h->n_store * D;
    g.rew = reinterpret_cast<const float*>(p);     p += sizeof(float) * h->n_store;
    g.cost = reinterpret_cast<const float*>(p);    p += sizeof(float) * h->n_store;
    g.term = reinterpret_cast<const uint8_t*>(p);  p += h->n_store;
    g.trunc = reinterpret_cast<const uint8_t*>(p);
    g.scratch = h->scratch;
    g.act_out = h->act_dev;
    g.D = D; g.n_store = h->n_store; g.n_act = h->n_act; g.parity = h->parity;

    cudaStream_t s = static_cast<cudaStream_t>(stream);
    FSRL_CUDA(cudaMemcpyAsync(h->pack_dev, h->pack_host,
                              norm ? fsrl_host_pack_norm_bytes(D, h->n_store, h->n_act, n_fresh)
                                   : fsrl_host_pack_bytes(D, h->n_store, h->n_act),
                              cudaMemcpyHostToDevice, s));
    if (norm) {
        // the order of the device-env collect: the rows of the envs that stepped, then those restarted since;
        // then every acting env's current normalized row into the pack
        const int* fresh_ids = reinterpret_cast<const int*>(static_cast<char*>(h->pack_dev) + fresh_off);
        const float* fresh_obs = reinterpret_cast<const float*>(fresh_ids + n_fresh);
        float* obs_next = const_cast<float*>(g.obs_next);
        rc = launch_obs_norm_rows(*nrm->obs_rms, nrm->obs_norm, E, g.store_ids, h->n_store, obs_next, obs_next, s);
        if (rc) return rc;
        rc = launch_obs_norm_rows(*nrm->obs_rms, nrm->obs_norm, E, fresh_ids, n_fresh, fresh_obs, nullptr, s);
        if (rc) return rc;
        rc = launch_obs_gather(nrm->obs_norm, D, g.act_ids, h->n_act, const_cast<float*>(g.obs), s);
        if (rc) return rc;
        if (h->n_store == 0 && h->n_act == 0) return FSRL_OK;
    }
    switch (H) {
        case 64: rc = dispatch_a<64>(*r, g, A, s); break;
        case 128: rc = dispatch_a<128>(*r, g, A, s); break;
        case 256: rc = dispatch_a<256>(*r, g, A, s); break;
        default: rc = dispatch_a<512>(*r, g, A, s); break;
    }
    if (rc) return rc;
    if (h->n_act > 0)
        FSRL_CUDA(cudaMemcpyAsync(h->act_host, h->act_dev, sizeof(float) * (size_t)h->n_act * A, cudaMemcpyDeviceToHost, s));
    return FSRL_OK;
}

extern "C" int fsrl_host_collect_step(const fsrl_rollout_t* r, const fsrl_host_step_t* h, void* stream) {
    return host_collect_step(r, h, nullptr, stream);
}

extern "C" int fsrl_host_collect_step_norm(const fsrl_rollout_t* r, const fsrl_host_step_t* h, const fsrl_host_norm_t* n,
                                           void* stream) {
    FSRL_REQUIRE(n != nullptr, "fsrl_host_collect_step_norm: null normalization descriptor");
    return host_collect_step(r, h, n, stream);
}
