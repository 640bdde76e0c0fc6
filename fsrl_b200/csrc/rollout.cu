// Rollout collection on the device: one loop iteration of rollout_step_kernel == one vector step of
// FastCollector.collect (reference: /root/reference/fsrl/data/fast_collector.py:252-368):
//   policy forward      (:267-269 -> base_policy.py:178-190, tianshou ActorProb/Actor)
//   exploration noise   (:279-280 -> ddpg_lag.py:225-231)
//   map_action          (:284     -> base_policy.py:226-256; remapped action NOT stored)
//   env.step            (:286)    -> envs.cuh (our analytic models)
//   cost / buffer.add   (:325-335) -> SoA transition buffers, env-major, per-env ring
//   done bookkeeping    (:340-363) -> inline when n_episode <= n_env, else rollout_resolve
// fused into a single kernel: the actor MLP forward for a tile of envs (mlp.cuh), Gaussian
// sampling from a Philox stream, log-prob, clip/scale, the env step and the SoA stores, so no
// observation or action ever leaves the GPU.  With inline bookkeeping a whole collect is one
// launch; the resolve path launches one step at a time (FSRL_ROLLOUT_PER_STEP=1 forces that
// everywhere, for A/B runs and the tests).
#include "rollout.cuh"

#include <atomic>
#include <mutex>

namespace fsrl {

// Registered plugin kinds: slot k holds kind FSRL_ENV_PLUGIN_FIRST + k.  Slots are filled in order under the
// mutex and never change afterwards; the count is published after its slot is written, so lookups take no lock.
static fsrl_env_plugin_t g_plugins[FSRL_ENV_PLUGIN_END - FSRL_ENV_PLUGIN_FIRST];
static std::atomic<int> g_n_plugins{0};
static std::mutex g_register_mu;
// The render launcher of slot k, attached after the slot is published (fsrl_env_register_renderer): set once from
// NULL, read with acquire, so lookups take no lock either.
static fsrl_env_renderer_t g_renderer_tables[FSRL_ENV_PLUGIN_END - FSRL_ENV_PLUGIN_FIRST];
static std::atomic<const fsrl_env_renderer_t*> g_renderers[FSRL_ENV_PLUGIN_END - FSRL_ENV_PLUGIN_FIRST];

// the table of a registered plugin kind, NULL for any other kind
static const fsrl_env_plugin_t* env_plugin(int kind) {
    const int k = kind - FSRL_ENV_PLUGIN_FIRST;
    return (k >= 0 && k < g_n_plugins.load(std::memory_order_acquire)) ? &g_plugins[k] : nullptr;
}

const fsrl_env_renderer_t* env_plugin_renderer(int kind) {
    return env_plugin(kind) ? g_renderers[kind - FSRL_ENV_PLUGIN_FIRST].load(std::memory_order_acquire) : nullptr;
}

const fsrl_env_plugin_t* env_table(int kind) {
    if (kind >= FSRL_ENV_PLUGIN_FIRST) return env_plugin(kind);
    switch (kind) {
        ENV_KINDS_CORE(ENV_TABLE_CASE)
        default: break;
    }
    if (const fsrl_env_plugin_t* t = env_table_bp(kind)) return t;
    return env_table_vel(kind);
}

bool env_kind_dims(int kind, EnvDims& d) {
    const fsrl_env_plugin_t* t = env_table(kind);
    if (t) d = {t->D, t->A, t->S, t->T};
    return t != nullptr;
}

int check_ids(const char* fn, const fsrl_rollout_t* a, const int32_t* ids, int n) {
    FSRL_REQUIRE(ids != nullptr || n == a->E, "%s: without ids, n must be E = %d (got %d)", fn, a->E, n);
    if (ids)
        for (int i = 0; i < n; ++i)
            FSRL_REQUIRE(ids[i] >= 0 && ids[i] < a->E, "%s: ids[%d] = %d outside [0, E = %d)", fn, i, ids[i], a->E);
    return FSRL_OK;
}

// begin a collect: ready envs = first min(E, n_episode) (:235-236), zero the per-collect stats
__global__ void collect_begin_kernel(const fsrl_rollout_t a, int n_episode) {
    fsrl_collect_stats_t* st = a.stats;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    const int ready = n_episode < a.E ? n_episode : a.E;
    if (e < a.E) { a.active[e] = e < ready ? 1 : 0; a.done_now[e] = 0; a.ep_rew[e] = 0.0; a.ep_len[e] = 0; }
    if (e == 0) {
        st->step_count = 0; st->total_cost = 0.0; st->sum_ep_rew = 0.0; st->sum_ep_len = 0;
        st->episode_count = 0; st->n_episode = n_episode; st->n_ready = ready;
        st->term_count = 0; st->trunc_count = 0; st->finished = 0; st->finished_next = 0;
    }
}

}  // namespace fsrl

using namespace fsrl;

// the env half of the descriptor (what every entry point touches)
static int check_env_state(const fsrl_rollout_t* a) {
    FSRL_REQUIRE(a != nullptr, "rollout: null descriptor");
    EnvDims d;
    FSRL_REQUIRE(env_kind_dims(a->kind, d), "rollout: unknown env kind %d", a->kind);
    FSRL_REQUIRE(a->E > 0, "rollout: E must be positive");
    FSRL_REQUIRE(a->env_state && a->obs_cur && a->env_t && a->ep_idx && a->act_ctr && a->active &&
                 a->ep_rew && a->ep_len && a->done_now && a->stats, "rollout: null state pointer");
    return FSRL_OK;
}

static int check_rollout(const fsrl_rollout_t* a) {
    int rc = check_env_state(a);
    if (rc) return rc;
    EnvDims d;
    env_kind_dims(a->kind, d);
    FSRL_REQUIRE(a->actor.in == d.D || a->mode == FSRL_MODE_RANDOM, "rollout: actor input dim %d != obs dim %d", a->actor.in, d.D);
    return FSRL_OK;
}

extern "C" int fsrl_env_dims(int kind, int* D, int* A, int* S, int* T) {
    EnvDims d;
    FSRL_REQUIRE(env_kind_dims(kind, d), "fsrl_env_dims: unknown env kind %d", kind);
    if (D) *D = d.D; if (A) *A = d.A; if (S) *S = d.S; if (T) *T = d.T;
    return FSRL_OK;
}

extern "C" int fsrl_env_reset_all(const fsrl_rollout_t* a, void* stream) {
    int rc = check_rollout(a);
    if (rc) return rc;
    return env_table(a->kind)->reset_all(a, stream);
}

extern "C" int fsrl_collect_begin(const fsrl_rollout_t* a, int n_episode, void* stream) {
    int rc = check_env_state(a);     // either collect path follows: the actor is checked by its steps
    if (rc) return rc;
    FSRL_REQUIRE(n_episode > 0, "n_episode must be positive");   // fast_collector.py:234
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    collect_begin_kernel<<<(a->E + 127) / 128, 128, 0, s>>>(*a, n_episode);
    FSRL_LAUNCH_CHECK();
    return FSRL_OK;
}

extern "C" int fsrl_rollout_steps(const fsrl_rollout_t* a, int n_steps, void* stream) {
    int rc = check_rollout(a);
    if (rc) return rc;
    FSRL_REQUIRE(n_steps >= 0, "fsrl_rollout_steps: n_steps < 0");
    FSRL_REQUIRE(a->mode == FSRL_MODE_RANDOM || (a->actor.w1t && a->actor.w2t && a->actor.w3t),
                 "rollout: null actor weights");
    FSRL_REQUIRE(a->actor.out <= MLP_MAX_OUT, "rollout: actor out dim %d > %d", a->actor.out, MLP_MAX_OUT);
    if (n_steps == 0) return FSRL_OK;
    // inline bookkeeping: no env's step depends on another env's, so all steps run in one launch
    const char* per_step = getenv("FSRL_ROLLOUT_PER_STEP");
    const bool one_launch = a->inline_done && !(per_step && atoi(per_step) != 0);
    return env_table(a->kind)->steps(a, n_steps, one_launch, stream);
}

extern "C" int fsrl_rollout_steps_act(const fsrl_rollout_t* a, const float* act, void* stream) {
    int rc = check_env_state(a);
    if (rc) return rc;
    FSRL_REQUIRE(act != nullptr, "fsrl_rollout_steps_act: null action array");
    return env_table(a->kind)->act_step(a, act, stream);
}

extern "C" int fsrl_rollout_norm_steps(const fsrl_rollout_t* a, const fsrl_obs_rms_t* n, int n_steps, const float* act,
                                       void* stream) {
    int rc = act ? check_env_state(a) : check_rollout(a);
    if (rc) return rc;
    EnvDims d;
    env_kind_dims(a->kind, d);
    rc = check_obs_rms("fsrl_rollout_norm_steps", n, a->E, d.D);
    if (rc) return rc;
    FSRL_REQUIRE(n_steps >= 0, "fsrl_rollout_norm_steps: n_steps < 0");
    FSRL_REQUIRE(!act || n_steps == 1, "fsrl_rollout_norm_steps: caller actions cover one step (n_steps = %d)", n_steps);
    if (!act) {
        FSRL_REQUIRE(a->mode == FSRL_MODE_RANDOM || (a->actor.w1t && a->actor.w2t && a->actor.w3t),
                     "rollout: null actor weights");
        FSRL_REQUIRE(a->actor.out <= MLP_MAX_OUT, "rollout: actor out dim %d > %d", a->actor.out, MLP_MAX_OUT);
    }
    if (n_steps == 0) return FSRL_OK;
    return env_table(a->kind)->norm_steps(a, n, n_steps, act, stream);
}

extern "C" int fsrl_env_step(const fsrl_rollout_t* a, const float* act, const int32_t* ids, int n, float* obs_next,
                             float* rew, float* cost, uint8_t* term, uint8_t* trunc, void* stream) {
    int rc = check_env_state(a);
    if (rc) return rc;
    FSRL_REQUIRE(n >= 1 && n <= a->E, "fsrl_env_step: n = %d outside [1, E = %d]", n, a->E);   // one row per env at most
    rc = check_ids("fsrl_env_step", a, ids, n);
    if (rc) return rc;
    FSRL_REQUIRE(act && obs_next && rew && cost && term && trunc, "fsrl_env_step: null action or output array");
    return env_table(a->kind)->env_step(a, act, ids, n, obs_next, rew, cost, term, trunc, stream);
}

extern "C" int fsrl_env_reset_ids(const fsrl_rollout_t* a, const int32_t* ids, int n, float* obs, void* stream) {
    int rc = check_env_state(a);
    if (rc) return rc;
    FSRL_REQUIRE(n >= 1 && n <= a->E, "fsrl_env_reset_ids: n = %d outside [1, E = %d]", n, a->E);   // one row per env at most
    rc = check_ids("fsrl_env_reset_ids", a, ids, n);
    if (rc) return rc;
    return env_table(a->kind)->reset_ids(a, ids, n, obs, stream);
}

extern "C" int fsrl_env_register(const fsrl_env_plugin_t* p, int* kind) {
    FSRL_REQUIRE(p != nullptr && kind != nullptr, "fsrl_env_register: null table or kind");
    FSRL_REQUIRE(p->abi_version == fsrl_abi_version(),
                 "fsrl_env_register: the plugin was built for ABI version %d, this library has version %d",
                 p->abi_version, fsrl_abi_version());
    FSRL_REQUIRE(p->D >= 1 && p->A >= 1 && p->A <= ENV_MAX_A && p->D + p->A <= FSRL_ENG_DX_LD && p->S >= 1 &&
                 p->S <= ENV_MAX_S && p->T >= 1,
                 "fsrl_env_register: D = %d, A = %d, S = %d, T = %d outside 1 <= A <= %d, D + A <= %d, "
                 "1 <= S <= %d, T >= 1", p->D, p->A, p->S, p->T, ENV_MAX_A, FSRL_ENG_DX_LD, ENV_MAX_S);
    FSRL_REQUIRE(p->reset_all && p->steps && p->act_step && p->env_step && p->reset_ids && p->norm_steps,
                 "fsrl_env_register: null launcher in the table");
    std::lock_guard<std::mutex> lock(g_register_mu);
    const int n = g_n_plugins.load(std::memory_order_relaxed);
    FSRL_REQUIRE(n < FSRL_ENV_PLUGIN_END - FSRL_ENV_PLUGIN_FIRST, "fsrl_env_register: all %d plugin kinds are taken",
                 FSRL_ENV_PLUGIN_END - FSRL_ENV_PLUGIN_FIRST);
    g_plugins[n] = *p;
    g_n_plugins.store(n + 1, std::memory_order_release);
    *kind = FSRL_ENV_PLUGIN_FIRST + n;
    return FSRL_OK;
}

extern "C" int fsrl_env_register_renderer(int kind, const fsrl_env_renderer_t* r) {
    FSRL_REQUIRE(r != nullptr && r->render != nullptr, "fsrl_env_register_renderer: null table or launcher");
    FSRL_REQUIRE(r->abi_version == fsrl_abi_version(),
                 "fsrl_env_register_renderer: the plugin was built for ABI version %d, this library has version %d",
                 r->abi_version, fsrl_abi_version());
    FSRL_REQUIRE(env_plugin(kind) != nullptr, "fsrl_env_register_renderer: env kind %d is not a registered plugin kind",
                 kind);
    std::lock_guard<std::mutex> lock(g_register_mu);
    const int k = kind - FSRL_ENV_PLUGIN_FIRST;
    FSRL_REQUIRE(g_renderers[k].load(std::memory_order_relaxed) == nullptr,
                 "fsrl_env_register_renderer: env kind %d already has a renderer", kind);
    g_renderer_tables[k] = *r;
    g_renderers[k].store(&g_renderer_tables[k], std::memory_order_release);
    return FSRL_OK;
}
