/* fsrl_b200 -- C-ABI of the H100-native (sm_90a) FSRL hot path.
 *
 * The reference (liuzuxin/FSRL) is pure Python and has NO FFI layer of its own
 * (SURVEY.md F1, 8b): its boundary is the Python class API (fsrl.policy / fsrl.data).  This
 * header is the boundary the new engine adds underneath that API: every entry point names
 * the reference function it replaces (file:line under /root/reference).  INTEGRATION.md
 * shows the ctypes binding a maintainer of the reference would add at each call site.
 *
 * Conventions (all entry points):
 *   - plain pointers + sizes, no torch types; every pointer is DEVICE memory unless the
 *     parameter is documented "host";
 *   - the caller owns every buffer (functions never allocate or free) and passes scratch
 *     space explicitly; `*_workspace_bytes` reports the size;
 *   - asynchronous on `stream` (a cudaStream_t passed as void*); no device sync inside;
 *   - returns 0 on success, <0 on error (FSRL_EINVAL -1, FSRL_ECUDA -2,
 *     FSRL_EWORKSPACE -3); fsrl_last_error() returns the thread-local message.  The
 *     reference signals errors with Python assert/exceptions; the Python host layer
 *     (fsrl_b200/_lib.py) re-raises these codes as the same exception types/messages;
 *   - fp32 storage; the GAE / n-step scans accumulate in fp64 like the reference.
 *   - one host thread per GPU/rank; entry points are not re-entrant on the same workspace.
 */
#ifndef FSRL_B200_H
#define FSRL_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- plumbing ------------------------------------------------------------------- */
const char* fsrl_last_error(void);
#define FSRL_ABI_VERSION 2 /* what fsrl_abi_version() returns; compiled into env plugins */
int fsrl_abi_version(void);
size_t fsrl_abi_sizeof(int which); /* sizeof() of the descriptor structs, for binding self-checks */
int fsrl_sm_count(void);
/* Number of kernels this library has launched so far in this process (host-side counter,
 * one per checked launch). bench.py reports the difference across its timed region. */
unsigned long long fsrl_launch_count(void);

/* ---- a6/a7: dual GAE(lambda) -------------------------------------------------------
 * Replaces fsrl/policy/base_policy.py:524-540 (gae_return, numba) together with the
 * value_mask / end_flag / ret=adv+v / f32 cast of compute_gae_returns (:409-411,:429,
 * :438-446) for the reward and cost critics in ONE pass.
 *   v, vnext : [C][ld] f32   V_i(obs), V_i(obs_next)   (critic i at offset i*ld)
 *   rew,cost : [N] f32       metrics of critic 0 / 1 (cost may be NULL when C == 1)
 *   end_flag : [N] u8        terminated | truncated | unfinished-tail  (:410-411)
 *   terminated: [N] u8 or NULL; when given, vnext is masked by ~terminated (:375,:429)
 *   adv, ret : [C][ld] f32   outputs (batch.advs / batch.rets columns)
 * Flat order is the reference's batch order: env-major, chronological inside an env. */
size_t fsrl_gae_dual_workspace_bytes(int64_t N);
int fsrl_gae_dual(const float* v, const float* vnext, const float* rew, const float* cost,
                  const uint8_t* end_flag, const uint8_t* terminated, double gamma,
                  double gae_lambda, float* adv, float* ret, int64_t N, int64_t ld, int C,
                  void* workspace, size_t workspace_bytes, void* stream);


/* ---- network descriptor ----------------------------------------------------------------
 * A 2-hidden-layer MLP in -> H -> H -> out (tianshou Net/MLP + head; the reference builds
 * these at fsrl/agent/ppo_lag_agent.py:136-145).  Canonical layout: every Linear is stored
 * TRANSPOSED, Wt[in][out] row-major (torch's .weight is the strided view Wt.t()).
 * H must be 64, 128, 256 or 512. */
typedef struct fsrl_mlp3 {
    const float* w1t; /* [in][H]  */
    const float* b1;  /* [H]      */
    const float* w2t; /* [H][H]   */
    const float* b2;  /* [H]      */
    const float* w3t; /* [H][out] */
    const float* b3;  /* [out]    */
    int in, H, out;
} fsrl_mlp3_t;

/* ---- a1-a5: rollout collection ---------------------------------------------------------
 * One fsrl_rollout_steps() step == one iteration of the while-loop of
 * FastCollector.collect (fsrl/data/fast_collector.py:252-368): policy forward
 * (base_policy.py:178-190), exploration noise (ddpg_lag.py:225-231), map_action
 * (base_policy.py:226-256), env.step, cost extraction, buffer.add and the episode
 * bookkeeping incl. the surplus-env rule (:357-363), for all ready envs, on the device. */
enum { FSRL_MODE_TRAIN = 0, FSRL_MODE_EVAL = 1, FSRL_MODE_RANDOM = 2 };
/* GAUSS_COND is SAC's tanh-squashed head; GAUSS_COND_RAW is the same conditioned-sigma Gaussian
 * without the squash (CVPO: act = mu + sigma*eps, logp = Independent(Normal(mu, sigma)).log_prob(act)) */
enum { FSRL_HEAD_GAUSS_INDEP = 0, FSRL_HEAD_GAUSS_COND = 1, FSRL_HEAD_DETERMINISTIC = 2,
       FSRL_HEAD_GAUSS_COND_RAW = 3 };
enum { FSRL_BOUND_NONE = 0, FSRL_BOUND_CLIP = 1, FSRL_BOUND_TANH = 2 };
enum { FSRL_ENV_CAR_CIRCLE = 0, FSRL_ENV_CAR_RUN = 1, FSRL_ENV_BALL_CIRCLE = 2,
       FSRL_ENV_BALL_RUN = 3, FSRL_ENV_ANT_CIRCLE = 4, FSRL_ENV_POINT_GOAL = 5,
       FSRL_ENV_ANT_RUN = 6, FSRL_ENV_DRONE_CIRCLE = 7, FSRL_ENV_DRONE_RUN = 8,
       /* Safety-Gymnasium navigation family; 9-15 and 23 are unassigned */
       FSRL_ENV_POINT_CIRCLE1 = 16, FSRL_ENV_POINT_CIRCLE2 = 17, FSRL_ENV_CAR_CIRCLE1 = 18,
       FSRL_ENV_CAR_CIRCLE2 = 19, FSRL_ENV_POINT_GOAL2 = 20, FSRL_ENV_CAR_GOAL1 = 21, FSRL_ENV_CAR_GOAL2 = 22,
       FSRL_ENV_POINT_BUTTON1 = 24, FSRL_ENV_POINT_BUTTON2 = 25, FSRL_ENV_CAR_BUTTON1 = 26,
       FSRL_ENV_CAR_BUTTON2 = 27, FSRL_ENV_POINT_PUSH1 = 28, FSRL_ENV_POINT_PUSH2 = 29, FSRL_ENV_CAR_PUSH1 = 30,
       FSRL_ENV_CAR_PUSH2 = 31,
       /* Safety-Gymnasium velocity family; 32 is unassigned */
       FSRL_ENV_HALF_CHEETAH_VEL = 33, FSRL_ENV_HOPPER_VEL = 34, FSRL_ENV_SWIMMER_VEL = 35,
       FSRL_ENV_WALKER2D_VEL = 36, FSRL_ENV_ANT_VEL = 37 };

/* per-collect statistics, device resident; the keys of collect()'s result dict
 * (fast_collector.py:399-408) are derived from it on the host */
typedef struct fsrl_collect_stats {
    unsigned long long step_count;  /* n/st */
    unsigned long long sum_ep_len;  /* sum of finished episode lengths */
    double total_cost;              /* total_cost */
    double sum_ep_rew;              /* sum of finished episode returns */
    int episode_count;              /* n/ep */
    int n_episode;                  /* target */
    int n_ready;                    /* len(ready_env_ids) */
    int term_count, trunc_count;
    int finished, finished_next;
    int pad;
} fsrl_collect_stats_t;

typedef struct fsrl_rollout {
    /* environment (SoA, device) */
    int kind, E, max_steps, inline_done;
    unsigned int seed_env, seed_act;
    float* env_state;        /* [S][E] */
    float* obs_cur;          /* [E][D] */
    int* env_t;              /* [E] step inside the running episode */
    unsigned int* ep_idx;    /* [E] episodes started (reset RNG counter) */
    unsigned int* act_ctr;   /* [E] actions sampled (noise RNG counter) */
    unsigned char* active;   /* [E] ready_env_ids as a mask */
    unsigned char* done_now; /* [E] 0 / 1 terminated / 2 truncated this step */
    double* ep_rew;          /* [E] running episode return */
    int* ep_len;             /* [E] running episode length */
    /* policy */
    fsrl_mlp3_t actor;
    const float* log_sigma;  /* [A] state-independent log-sigma (HEAD_GAUSS_INDEP) */
    int head, mode, bounded, action_bound, action_scaling, pad0;
    float max_action, expl_sigma, sigma_min, sigma_max, tanh_eps, pad1;
    float act_low[8], act_high[8];
    /* transition buffer: env-major sub-buffers of `cap` slots (tianshou VectorReplayBuffer
     * order), any pointer group may be NULL to collect without storing (evaluate()) */
    float *b_obs, *b_obs_next, *b_act, *b_rew, *b_cost, *b_logp;
    unsigned char *b_term, *b_trunc;
    int* b_ptr;              /* [E] next write slot */
    int* b_len;              /* [E] valid transitions */
    long long cap;
    fsrl_collect_stats_t* stats;
} fsrl_rollout_t;

int fsrl_env_dims(int kind, int* D, int* A, int* S, int* T);
/* reset_env (fast_collector.py:131-152): start a fresh episode in every env */
int fsrl_env_reset_all(const fsrl_rollout_t* r, void* stream);
/* start of collect(n_episode): ready set = first min(E, n_episode) envs (:233-236) */
int fsrl_collect_begin(const fsrl_rollout_t* r, int n_episode, void* stream);
/* n_steps vector steps; steps after stats->finished are no-ops */
int fsrl_rollout_steps(const fsrl_rollout_t* r, int n_steps, void* stream);
/* one vector step of collect() with the caller's actions instead of r->actor: act[E][A] are the
 * policy's raw actions (after its exploration noise), one row per env, read for the active envs.
 * map_action, env.step, buffer.add and the episode bookkeeping are those of fsrl_rollout_steps; the
 * raw action is stored with logp = 0, and act_ctr is left alone.  r->actor, head and mode are unused. */
int fsrl_rollout_steps_act(const fsrl_rollout_t* r, const float* act, void* stream);

/* ---- gym vector-env protocol (tianshou BaseVectorEnv.step / reset with env ids) ----------------
 * ids: HOST int32 [n] env ids, each in [0, E), or NULL for all envs in order (then n must be E).
 * A listed env must appear once: duplicate ids are the caller's error (their order is undefined).
 * Rows of act / outputs follow ids.
 *   fsrl_env_step       act[n][A] env-range actions (no map_action); writes obs_next[n][D], rew[n],
 *                       cost[n], term[n], trunc[n] (u8; trunc = horizon reached and not terminated)
 *                       and advances env_state, obs_cur, env_t, ep_rew and ep_len of the listed envs.
 *                       No ring store, no collect statistics.
 *   fsrl_env_reset_ids  fresh episode in the listed envs (the same reset stream as every other
 *                       reset path); obs[n][D] receives their observations (obs may be NULL)
 * Both return FSRL_EINVAL before touching the device when n, an id or a pointer is invalid. */
int fsrl_env_step(const fsrl_rollout_t* r, const float* act, const int32_t* ids, int n, float* obs_next,
                  float* rew, float* cost, uint8_t* term, uint8_t* trunc, void* stream);
int fsrl_env_reset_ids(const fsrl_rollout_t* r, const int32_t* ids, int n, float* obs, void* stream);

/* ---- frames of the device envs (DeviceVectorEnv.render with render_mode="rgb_array") ------------
 * out[n][height][width][3] (u8 RGB, device) receives one top-down or side-view frame per row of ids
 * (HOST int32 env ids in [0, E), duplicates allowed; NULL = every env in order, then n must be E).
 * Row 0 is the top of the frame; pixel (i, j) samples the world point (x0 + (j + 0.5) sx,
 * y1 - (i + 0.5) sy) of the task's view window and takes the colour of the last primitive of the
 * env's scene that covers it (a fixed drawing order, one fixed palette, no antialiasing; DESIGN §7).
 * last_cost (device, E floats, may be NULL): the robot of env e is drawn in the cost colour when
 * last_cost[e] > 0.  Reads only env_state, env_t, ep_idx and seed_env of r, writes only out.
 * A plugin kind (fsrl_env_register) is drawn by the launcher its plugin registered with
 * fsrl_env_register_renderer: the same rasterizer around the scene its struct's draw describes.
 * Returns FSRL_EINVAL before touching the device on an unknown kind, n < 1, an id outside [0, E),
 * height or width outside [16, 1024], a null r, out or state pointer, or, after all of these, a
 * plugin kind without a renderer. */
int fsrl_env_render(const fsrl_rollout_t* r, const int32_t* ids, int n, int height, int width,
                    const float* last_cost, uint8_t* out, void* stream);

/* ---- host-stepped envs: one vector step of FastCollector.collect around a host env.step ----------
 * The host steps its own envs (gymnasium / tianshou objects); the device keeps the actor, the noise
 * stream and the ring.  One call per vector step enqueues, on `stream`: one H2D copy of the packed
 * upload, one launch, one D2H copy of the actions.  The launch
 *   store phase: buffer.add of the n_store transitions of the previous call (obs, raw act and logp from
 *                that call's act phase, obs_next / rew / cost / flags from this upload); advances
 *                b_ptr / b_len.  Skipped when r->b_obs is NULL (n_store must then be 0).
 *   act phase:   the actor on the n_act uploaded observations, sampling keyed by (env id, act_ctr) as in
 *                fsrl_rollout_steps (same heads, modes and noise), map_action; act_host[k][A] receives
 *                the env-range action of row k.
 * Per-env scratch [2][E][D + A + 1] (obs, raw act, logp) alternates by `parity` (0 / 1, flipped every
 * call): the act phase writes half `parity`, the store phase reads the other half.  r->kind, the env
 * state pointers and r->stats are unused; r->E, act_ctr, the actor, head / mode and the ring are read.
 * pack_host (HOST, pinned) holds, in this order and without padding:
 *   int32 store_ids[n_store] | int32 act_ids[n_act] | f32 obs[n_act][D] | f32 obs_next[n_store][D] |
 *   f32 rew[n_store] | f32 cost[n_store] | u8 term[n_store] | u8 trunc[n_store]
 * (fsrl_host_pack_bytes gives its size); pack_dev receives it.  Ids are in [0, E), each at most once per
 * list.  Returns FSRL_EINVAL before touching the device when a count, an id or a pointer is invalid,
 * D != r->actor.in (outside random mode), A is outside 1..8, D + A > FSRL_ENG_DX_LD or the actor's H
 * is not 64 / 128 / 256 / 512.  The caller synchronises `stream` before reading act_host. */
typedef struct fsrl_host_step {
    int D, A;
    int n_store, n_act;
    int parity, pad;
    const void* pack_host;
    void* pack_dev;
    float* scratch;        /* device [2][E][D + A + 1] */
    float* act_dev;        /* device [E][A] */
    float* act_host;       /* HOST, pinned [E][A] */
} fsrl_host_step_t;
size_t fsrl_host_pack_bytes(int D, int n_store, int n_act);
int fsrl_host_collect_step(const fsrl_rollout_t* r, const fsrl_host_step_t* h, void* stream);
/* fsrl_host_collect_step over an env wrapped by VectorEnvNormObs (observation normalization, csrc/obsnorm.cu).
 * pack_host continues, from byte fsrl_host_pack_norm_bytes(D, n_store, n_act, 0), with
 *   int32 fresh_ids[n_fresh] | f32 fresh_obs[n_fresh][D]
 * (the reset observations of the envs restarted since the previous call), and before the launch the device
 * (1) updates the statistics with the n_store obs_next rows and normalizes them in the pack and in obs_norm,
 * (2) does the same with the fresh rows, (3) copies obs_norm[act_ids[k]] over the n_act observation rows of the
 * pack.  The act and store phases then read normalized rows.  n_store may be positive without a ring (the store
 * phase then stores nothing).  Everything else is fsrl_host_collect_step's. */
typedef struct fsrl_host_norm {
    const struct fsrl_obs_rms* obs_rms;
    float* obs_norm;       /* device [E][D]: every env's current normalized observation */
    int n_fresh, pad;
} fsrl_host_norm_t;
size_t fsrl_host_pack_norm_bytes(int D, int n_store, int n_act, int n_fresh);
int fsrl_host_collect_step_norm(const fsrl_rollout_t* r, const fsrl_host_step_t* h, const fsrl_host_norm_t* n,
                                void* stream);

/* ---- observation normalization (tianshou's VectorEnvNormObs) on the device ---------------------------
 * Running statistics mean[D], var[D] (float64) and count (int64) of every observation the wrapped envs
 * returned.  An update with a batch of n >= 1 rows takes its mean and population variance per feature and
 * merges them into the running values by the parallel (Chan) update; an empty batch changes nothing.  A
 * value is normalized as clip((x - mean) / sqrt(var + eps), -clip_max, clip_max) in float64 (no clip when
 * clip_max <= 0) and rounded to float32 once.
 * The batch is split into fixed tiles of FSRL_OBS_RMS_TILE env ids; one launch forms each tile's
 * (count, mean, M2) over its rows in ascending id order, a second merges the tiles in tile order
 * (every CTA repeats the merge, CTA 0 publishes) and normalizes the rows.  No floating-point atomics: the
 * result depends only on which env ids hold which rows, so repeated runs, the device-env path and the
 * host-env path give the same bits.  `update` = 0 only normalizes.  `work` is per wrapper
 * (fsrl_obs_rms_work_bytes(E, D) bytes): the statistics may be shared by several wrappers.
 *   fsrl_obs_rms_rows        the rows of the envs ids[0..count) (HOST ids, each once; NULL: all E, count = E)
 *                            in x[E][D]: if rows_in (device [count][D]) is given its row k is first copied
 *                            to x[ids[k]]; update, normalize in x, and copy row ids[k] of x to out[k]
 *                            (device [count][D], may be NULL)
 *   fsrl_rollout_norm_steps  n_steps vector steps of a collect over a wrapped device env, r->obs_cur holding
 *                            normalized observations: per step the fused step kernel (act == NULL) or the
 *                            caller-action step kernel (act, device [E][A], n_steps = 1), then the update with
 *                            the obs_next of every env that stepped, normalized in obs_cur and in the ring slot
 *                            just written, then the resolve kernel, then the update with the observations of
 *                            the envs it restarted, normalized in obs_cur.  6 launches per step, plus one.
 * Both return FSRL_EINVAL before touching the device on a bad count, id, width or pointer. */
#define FSRL_OBS_RMS_TILE 128
typedef struct fsrl_obs_rms {
    double* mean;          /* device [D] */
    double* var;           /* device [D] */
    long long* count;      /* device [1] */
    void* work;            /* device, fsrl_obs_rms_work_bytes(E, D) bytes */
    int D, update;
    double clip_max, eps;
} fsrl_obs_rms_t;
size_t fsrl_obs_rms_work_bytes(int E, int D);
int fsrl_obs_rms_rows(const fsrl_obs_rms_t* n, float* x, int E, const int32_t* ids, int count, const float* rows_in,
                      float* out, void* stream);
int fsrl_rollout_norm_steps(const fsrl_rollout_t* r, const fsrl_obs_rms_t* n, int n_steps, const float* act,
                            void* stream);

/* ---- user-defined device envs (plugins) --------------------------------------------------------------
 * A plugin (csrc/env_plugin.cu compiled against a user's env struct, linked against this library) hands
 * over the six launchers every env-dependent entry point reaches a kind through, instantiated for its
 * struct by the same templates the built-in kinds use, and the struct's widths and horizon.
 * fsrl_env_register copies the table and returns in *kind the next free id of
 * [FSRL_ENV_PLUGIN_FIRST, FSRL_ENV_PLUGIN_END); from then on fsrl_env_dims, the rollout, gym-protocol,
 * observation-normalizing and trajectory entry points accept that kind like a built-in one, and
 * fsrl_env_render does once a renderer is registered for it (below).  Returns FSRL_EINVAL, registering nothing, when abi_version differs from
 * fsrl_abi_version(), a width is outside the limits below, a launcher is NULL or the range is full.
 * Limits: 1 <= D, 1 <= A <= 8, D + A <= FSRL_ENG_DX_LD, 1 <= S <= 32, T >= 1. */
#define FSRL_ENV_PLUGIN_FIRST 64
#define FSRL_ENV_PLUGIN_END 128
typedef struct fsrl_env_plugin {
    int abi_version;
    int D, A, S, T, pad;
    int (*reset_all)(const fsrl_rollout_t* r, void* stream);
    int (*steps)(const fsrl_rollout_t* r, int n_steps, int one_launch, void* stream);
    int (*act_step)(const fsrl_rollout_t* r, const float* act, void* stream);
    int (*env_step)(const fsrl_rollout_t* r, const float* act, const int32_t* ids, int n, float* obs_next,
                    float* rew, float* cost, uint8_t* term, uint8_t* trunc, void* stream);
    int (*reset_ids)(const fsrl_rollout_t* r, const int32_t* ids, int n, float* obs, void* stream);
    int (*norm_steps)(const fsrl_rollout_t* r, const fsrl_obs_rms_t* n, int n_steps, const float* act, void* stream);
} fsrl_env_plugin_t;
int fsrl_env_register(const fsrl_env_plugin_t* p, int* kind);
/* A plugin whose struct defines draw also hands over a render launcher (its fsrl_env_plugin_render()):
 * fsrl_env_render's rasterizer instantiated for the struct, called by fsrl_env_render with the
 * arguments it has checked.  fsrl_env_register_renderer attaches it to the registered plugin kind
 * `kind`, once.  Returns FSRL_EINVAL, attaching nothing, on a null table or launcher, an abi_version
 * other than fsrl_abi_version(), a kind that is not a registered plugin kind, or a kind that already
 * has a renderer.  A plugin built without draw, or before this entry point existed, has no renderer. */
typedef struct fsrl_env_renderer {
    int abi_version, pad;
    int (*render)(const fsrl_rollout_t* r, const int32_t* ids, int n, int height, int width, const float* last_cost,
                  uint8_t* out, void* stream);
} fsrl_env_renderer_t;
int fsrl_env_register_renderer(int kind, const fsrl_env_renderer_t* r);

/* ---- offline datasets: finished episodes of the rollout ring -> trajectory arena ----------------
 * Replaces the per-transition Batch.cat / return sums of TrajectoryBuffer.store
 * (fsrl/data/traj_buf.py:60-95), fed by BasicCollector (basic_collector.py:238-248), and the
 * Batch.cat of get_all() (:183-189).  The host decides which episodes to keep; the device scans,
 * copies and packs.
 *   fsrl_traj_begin  start of a collect: the harvest state forgets any open episode
 *   fsrl_traj_scan   walk every env's ring slots written since the last scan; append one row per
 *                    episode that finished there to rows[] (atomic counter *n_rows, which keeps
 *                    counting past row_cap: the caller treats *n_rows > row_cap as an error).  Ring
 *                    slots may be overwritten only after the scan that saw them, and an env's
 *                    unscanned slots must be fewer than cap, except on the one-episode-per-env path:
 *                    there n_ready > 0, and a ready env (e < n_ready) whose pointer did not move
 *                    wrote exactly cap slots.  n_ready = 0 otherwise.
 *   fsrl_traj_copy   jobs[n][4] = (env, start slot, length, arena slot): copy episodes into the
 *                    arena; act is stored remapped, as the env received it (map_action)
 *   fsrl_traj_copy_host  fsrl_traj_copy from the ring of host-stepped envs (r->kind = -1, whose widths the
 *                    descriptor does not carry): D >= 1 and 1 <= A <= 8 are the ring's widths and must equal
 *                    the arena's.  The host knows every finished episode (the collector's own loop), so
 *                    there is no scan on this path; the caller copies an episode after the launch that
 *                    stores its last transition and before its first slot is written again.  map_action
 *                    takes r's action bounds (HostVectorEnv.fill).
 *   fsrl_traj_gather jobs[n][3] = (arena slot, length, first output row): pack into `out`, whose
 *                    arrays are contiguous rows (out->stride and out->n_slots are ignored) */
typedef struct fsrl_traj_row {
    int env, start, len;      /* ring slot of the first transition, number of transitions */
    int finish;               /* transitions env wrote since fsrl_traj_begin, the last one included */
    int terminated, truncated;
    double ret, cost;         /* fp64 sums of the stored fp32 rewards / costs in time order */
} fsrl_traj_row_t;
typedef struct fsrl_traj_scan {
    int *last, *open, *open_len, *steps; /* [E] ring pointer at the last scan, first slot and length of the
                                          * open episode, transitions since fsrl_traj_begin */
    double *rew, *cost;                  /* [E] running sums of the open episode */
    fsrl_traj_row_t* rows;
    int* n_rows;
    int row_cap, pad;
} fsrl_traj_scan_t;
typedef struct fsrl_traj_arena {
    float *obs, *obs_next, *act, *rew, *cost; /* [n_slots * stride] rows of D / D / A / 1 / 1 floats */
    unsigned char *term, *trunc;
    long long stride;                          /* transitions per slot (the env's max_episode_steps) */
    long long n_slots;
    int D, A;
} fsrl_traj_arena_t;

int fsrl_traj_begin(const fsrl_rollout_t* r, const fsrl_traj_scan_t* h, void* stream);
int fsrl_traj_scan(const fsrl_rollout_t* r, const fsrl_traj_scan_t* h, int n_ready, void* stream);
int fsrl_traj_copy(const fsrl_rollout_t* r, const fsrl_traj_arena_t* a, const int* jobs, int n_jobs,
                   void* stream);
int fsrl_traj_copy_host(const fsrl_rollout_t* r, const fsrl_traj_arena_t* a, int D, int A, const int* jobs,
                        int n_jobs, void* stream);
int fsrl_traj_gather(const fsrl_traj_arena_t* a, const fsrl_traj_arena_t* out, const long long* jobs,
                     int n_jobs, void* stream);

/* ---- a9/a10: PPO-Lagrangian update --------------------------------------------------------
 * Replaces PPOLagrangian.policy_loss / critics_loss / learn
 * (fsrl/policy/ppo_lag.py:152-257) and LagrangianPolicy.safety_loss
 * (fsrl/policy/lagrangian_base.py:145-166): per-minibatch advantage normalisation, clipped
 * surrogate, unclipped lambda-weighted cost term, rescaling, value losses, backward,
 * clip_grad_norm_ and Adam, with per-minibatch statistics accumulated on the device.
 *
 * All networks of the policy live in ONE flat fp32 buffer `theta`; network n (0 = actor,
 * 1.. = critics) starts at net_off[n] with layout
 *     w1t[D][H] | b1[H] | w2t[H][H] | b2[H] | w3t[H][out] | b3[out] | (actor) log_sigma[A]
 * grad / adam_m / adam_v mirror that layout; w2n[n][H][H] is the out-major copy of w2t kept
 * in sync by the Adam kernel (fsrl_ppo_sync_mirror initialises it). */
#define FSRL_PPO_STATS 8 /* per-minibatch: actor_rew, actor_safety, kl, vf0, vf1, entropy, grad_norm, - */
typedef struct fsrl_ppo_update {
    float *theta, *grad, *adam_m, *adam_v, *w2n, *scratch, *norm_sq, *stats;
    long long net_off[3];
    long long n_params;
    int n_nets, D, H, A, C, actor_out, bmax, pad2;
    /* the processed batch (flat env-major arrays) and the minibatch permutation */
    const float *obs, *act, *logp_old, *adv, *ret, *values; /* adv/ret/values: [C][ld] */
    long long ld;
    const int* perm;
    /* hyper-parameters (ppo_lag.py:86-99) */
    float eps_clip, dual_clip, vf_coef, max_grad_norm;
    float max_action, lagrangian, rescaling, pad0;
    int bounded, norm_adv, value_clip, use_lagrangian;
    double lr, beta1, beta2, adam_eps;
    /* data-parallel run (world > 1): NCCL communicator, per-minibatch advantage moments
     * [n_mb][2][2] (sum, sum of squares; reduced over ranks once per repeat); moments must
     * alias moments_w */
    void* comm;
    double* moments_w;
    const double* moments;
    int world, batch_size;
    /* required [N*(D+A+1+3C)] floats: the epoch driver gathers the permuted batch into it once
     * per repeat so that every minibatch is a contiguous row range */
    float* gather;
    /* [n_minibatches][2][2] floats: (mean, 1/std) of the advantages of every minibatch of the
     * repeat, filled by the epoch driver */
    float* mb_stats;
    /* required device u64: ticket counter of the in-kernel grid barrier (fused wgrad + Adam
     * launch), reset by the epoch driver */
    unsigned long long* barrier;
    /* peer-memory gradient exchange (world > 1, optional; NCCL all-reduce when p2p_on == 0):
     * rank r's exchange block (fsrl_p2p_alloc) mapped into this process -- p2p_xg[b][r] its
     * gradient buffer of step parity b, p2p_flags[r] its arrival flags [FSRL_P2P_MAX_RANKS] --
     * entries [.][p2p_rank] are this rank's own block.  The weight-gradient kernel writes into the
     * local buffer; ppo_dp_reduce_kernel signals the peers, waits for their flags and sums all
     * ranks' buffers over NVLink in rank order (bit-identical result everywhere). */
    const float* p2p_xg[2][8];
    unsigned long long* p2p_flags[8];
    int* p2p_err;                  /* local: set to 1 if a peer never arrived (wait timed out) */
    float* p2p_part;               /* local [FSRL_P2P_PARTIALS]: per-CTA sums of g^2 (summed in a fixed
                                    * order by the Adam kernel: atomics would break rank lock-step) */
    int p2p_rank, p2p_on;
    /* persistent wgmma path (csrc/ppo_persist.cu; H = 256, batch 256): workspace of
     * fsrl_ppo_persist_ws_floats() floats for the operand images / partials / flags; NULL or
     * persist_off != 0 selects the three-launch chain.  With world > 1 the launch exchanges gradients
     * itself: it treats every p2p_xg[b][r] as fsrl_ppo_persist_p2p_floats() floats of packet regions
     * (one per source rank + one for reduced tiles; ranks push, receivers poll their own buffer) and
     * needs p2p_on, p2p_rank and p2p_stride >= that size; p2p_flags / p2p_part stay with the chain */
    float* persist_ws;
    long long persist_ws_floats;
    int persist_off, pad1;
    long long p2p_stride;          /* floats available in every p2p_xg buffer (fsrl_p2p_stride of the allocation) */
} fsrl_ppo_update_t;

size_t fsrl_ppo_scratch_floats(int n_nets, int H, int bmax);
size_t fsrl_ppo_persist_ws_floats(int n_nets, int D, int H);
/* floats each peer-mapped exchange buffer must hold for the data-parallel persistent path */
size_t fsrl_ppo_persist_p2p_floats(int n_nets);
/* 1 if fsrl_ppo_lag_epoch would take the persistent path for this descriptor / batch */
int fsrl_ppo_persist_active(const fsrl_ppo_update_t* u, long long n_total, int batch_size);
int fsrl_ppo_sync_mirror(const fsrl_ppo_update_t* u, void* stream);
/* one repeat of learn()'s inner loop: all minibatches of Batch.split(batch_size,
 * merge_last=True) over u->perm[0..n_total); Adam step counter continues from adam_t0;
 * statistics go to stats[stats_slot0 + i]; *n_minibatches (host) receives the count */
int fsrl_ppo_lag_epoch(const fsrl_ppo_update_t* u, long long n_total, int batch_size,
                       int stats_slot0, long long adam_t0, int* n_minibatches, void* stream);

/* ---- a6: batched critic / actor forward ---------------------------------------------------
 * y[r][:] = net(x[idx ? idx[r] : r][:]) for r < n_rows.  Replaces the chunked no_grad
 * critic passes of compute_gae_returns (fsrl/policy/base_policy.py:416-422). */
int fsrl_mlp_forward(const fsrl_mlp3_t* net, const float* x, const int* idx, long long n_rows,
                     float* y, void* stream);

/* ---- generic minibatch MLP engine (SAC / DDPG / CPO updates are assembled from it) --------
 * Replaces the eager autograd forward/backward/optimizer.step of the reference's learners
 * (fsrl/policy/sac_lag.py:185-258, ddpg_lag.py:165-213, cpo.py:147-162) and soft_update
 * (fsrl/policy/base_policy.py:220-224).  Networks live in the flat arena (layout as for
 * fsrl_ppo_update_t); each has a scratch slot of fsrl_engine_slot_floats(H, bmax) floats:
 *   h1 | h2 | dz1 | dz2 : [bmax][H],  out | dout : [bmax][16],  dx : [bmax][FSRL_ENG_DX_LD]
 * forward writes `out` (+ h1, h2 when save != 0); the caller fills `dout` (d loss / d head
 * output, columns [out, out+n_extra) = d loss / d extra parameters); backward produces dz1,
 * dz2 (+ dx = d loss / d input); wgrad reduces them into `grad`; adam applies them. */
#define FSRL_ENG_MAX_NETS 8
#define FSRL_ENG_DX_LD 80   /* the widest input a net may have (obs + act of the widest task: 76 + 2) */
typedef struct fsrl_netref {
    long long off;      /* start of the net inside theta / grad / adam_m / adam_v */
    long long w2n_off;  /* start of its W2 mirror inside w2n */
    int D, H, out, n_extra;
    int slot, pad;
} fsrl_netref_t;
typedef struct fsrl_netlist {
    int n, pad;
    fsrl_netref_t nets[FSRL_ENG_MAX_NETS];
} fsrl_netlist_t;
typedef struct fsrl_engine {
    float *theta, *grad, *adam_m, *adam_v, *w2n, *scratch;
    int bmax, pad;
} fsrl_engine_t;
/* input row r = concat(xa[ia ? ia[r] : r][0..Da), xb[ib ? ib[r] : r][0..Db)) */
typedef struct fsrl_eng_input {
    const float* xa;
    const int* ia;
    const float* xb;
    const int* ib;
    int Da, Db;
} fsrl_eng_input_t;

size_t fsrl_engine_slot_floats(int H, int bmax);
int fsrl_engine_dx_ld(void); /* FSRL_ENG_DX_LD: the row stride of dx, and the widest input */
int fsrl_engine_forward(const fsrl_engine_t* e, const fsrl_netlist_t* nets, const fsrl_eng_input_t* in,
                        int B, int save, void* stream);
int fsrl_engine_backward(const fsrl_engine_t* e, const fsrl_netlist_t* nets, int B, int want_dx, void* stream);
/* grad (+)= the weight gradients of B rows; when norm_sq != NULL, *norm_sq += the squared norm of the
 * listed nets' final gradients (above 4096 rows the rows are split and a separate pass sums it) */
int fsrl_engine_wgrad(const fsrl_engine_t* e, const fsrl_netlist_t* nets, const fsrl_eng_input_t* in, int B,
                      int accumulate, float* norm_sq, void* stream);
/* torch.optim.Adam step `step` (1-based) on the listed nets; grad <- grad*grad_scale + 2*l2_reg*p
 * and, when norm_sq != NULL && max_grad_norm > 0, clip_grad_norm_ by sqrt(*norm_sq) */
int fsrl_engine_adam(const fsrl_engine_t* e, const fsrl_netlist_t* nets, double lr, double beta1,
                     double beta2, double eps, long long step, double grad_scale, double l2_reg,
                     const float* norm_sq, double max_grad_norm, void* stream);
int fsrl_engine_polyak(const fsrl_engine_t* e, const fsrl_netlist_t* dst, const fsrl_netlist_t* src,
                       double tau, void* stream);
int fsrl_engine_sync_mirror(const fsrl_engine_t* e, const fsrl_netlist_t* nets, void* stream);

/* ---- a12-a14, a16: SAC- / DDPG-Lagrangian gradient steps -------------------------------------
 * fsrl_offpolicy_steps runs n_steps iterations of `policy.update(batch_size, buffer)`
 * (fsrl/trainer/offpolicy.py:102-104): process_fn = n-step targets for the reward and cost
 * critics (fsrl/policy/base_policy.py:453-512,543-567; sac_lag.py:136-145; ddpg_lag.py:
 * 125-131), critics_loss, policy_loss (lambda-weighted cost-Q term + rescaling,
 * lagrangian_base.py:145-166; SAC: tanh-squashed rsample, log-prob correction, auto-alpha),
 * sync_weight.  Networks are engine netlists: SAC critics = C x DoubleCritic = 2C nets
 * (twin = 1, order r1 r2 c1 c2), DDPG critics = C nets. */
#define FSRL_MAX_NSTEP 8
#define FSRL_OFF_STATS 8
enum { FSRL_OFF_ST_Q0 = 0, FSRL_OFF_ST_Q1 = 1, FSRL_OFF_ST_ACTOR_REW = 2, FSRL_OFF_ST_ACTOR_SAFETY = 3,
       FSRL_OFF_ST_LOGP = 4, FSRL_OFF_ST_ALPHA_LOSS = 5, FSRL_OFF_ST_ALPHA = 6 };
enum { FSRL_ALGO_SAC = 0, FSRL_ALGO_DDPG = 1 };
typedef struct fsrl_offpolicy {
    fsrl_engine_t eng;
    fsrl_netlist_t actor, actor_old, critics, critics_old;
    int algo, D, A, C, twin, n_step, bounded, use_alpha, auto_alpha, use_lagrangian;
    unsigned int seed, pad0;
    double gamma, tau, critic_lr, actor_lr;
    float alpha_lr, target_entropy, max_action, sigma_min, sigma_max, tanh_eps, lagrangian, rescaling;
    /* replay buffer (env-major sub-buffer rings, see fsrl_rollout_t) */
    const float *b_obs, *b_obs_next, *b_act, *b_rew, *b_cost;
    const unsigned char *b_term, *b_trunc;
    const int *b_ptr, *b_len;
    long long cap;
    /* per-step work arrays, all sized for eng.bmax rows */
    int* w_term_idx;
    double *w_partial, *w_gpow;      /* [2][B], [B] */
    float *w_vmask, *w_target;       /* [B], [2][B] */
    float *w_act_next, *w_logp_next, *w_act, *w_logp, *w_keep; /* [B][A], [B], [B][A], [B], [B][24] */
    /* engine scratch views (host-resolved): head outputs / gradients / input gradients */
    float *actor_out, *actor_old_out, *actor_dout;
    float *q_out[4], *q_dout[4], *q_dx[4], *q_old_out[4];
    float* alpha;        /* device scalar */
    float* alpha_state;  /* device [log_alpha, adam_m, adam_v, adam_t] */
    /* data parallel (world > 1): every rank samples its own replay shard; per gradient step the
     * critics' and the actor's gradients are all-reduced (one grouped NCCL call each) and averaged,
     * and the entropy-tuning statistic is all-reduced so that alpha stays identical on all ranks */
    void* comm;
    int world, pad1;
} fsrl_offpolicy_t;

int fsrl_nstep_prepare(const fsrl_offpolicy_t* d, const int* idx, int B, void* stream);
int fsrl_offpolicy_steps(const fsrl_offpolicy_t* d, const int* idx_all, int n_steps, int B,
                         long long critic_t0, long long actor_t0, unsigned long long noise_t0,
                         float* stats, void* stream);

/* ---- f4: CVPO gradient steps ------------------------------------------------------------------------
 * fsrl_cvpo_steps runs n_steps iterations of CVPO.update (fsrl/policy/cvpo.py:206-430): n-step targets
 * with an unsquashed sample of the CURRENT actor and min-over-heads critics_old (:206-222), critic
 * regression (:248-276), E-step on K particles of actor_old scored by the just-updated critics (dual
 * Adam, clamp, softmax weights; :320-363, including the in-place `combined_q -=` of :284 that keeps
 * subtracting lambda*q_c from q_r), mstep_iters M-steps (weighted MLE + decoupled KL with the dual
 * Adam and the clip of its uses; :369-418), Polyak of critics_old (:201-204).  No host sync: every dual
 * and its Adam moments live in the device arrays below.  `off` carries the engine, the net lists
 * (actor, actor_old, critics, critics_old), the replay ring and the n-step work arrays; off.use_alpha
 * must be 0.  Single GPU (off.world <= 1), C <= 2, A <= 8, K*B <= off.eng.bmax.
 *   estep_state [8]: eta, lambda, adam m[2], adam v[2], adam step, -   (persists for the policy's life)
 *   mstep_state [8]: dual_mu, dual_std, adam m[2], adam v[2], adam step, -   (zeroed by pre_update_fn)
 *   particles [K*B][A], part_idx [K*B], mu_old / std_old [B][A], comb / weights [K*B]: work arrays
 *   log_sigma / log_sigma_old: sigma_param [A] of the actor / actor_old (the nets' extra parameter)
 *   when cond_sigma == 0, NULL otherwise
 * stats: [n_steps][FSRL_CVPO_STATS] (zeroed by the caller), columns FSRL_CVPO_ST_*; the
 * last E-step / M-step iteration of a step is reported (the reference logs every iteration). */
#define FSRL_CVPO_STATS 16
enum { FSRL_CVPO_ST_Q0 = 0, FSRL_CVPO_ST_Q1 = 1, FSRL_CVPO_ST_VAL_Q0 = 2, FSRL_CVPO_ST_VAL_Q1 = 3,
       FSRL_CVPO_ST_ESTEP_LOSS = 4, FSRL_CVPO_ST_DUAL0 = 5, FSRL_CVPO_ST_DUAL1 = 6, FSRL_CVPO_ST_KL_MU = 7,
       FSRL_CVPO_ST_KL_STD = 8, FSRL_CVPO_ST_LOSS_KL = 9, FSRL_CVPO_ST_LOSS_MLE = 10, FSRL_CVPO_ST_LOSS_TOTAL = 11,
       FSRL_CVPO_ST_DUAL_MU = 12, FSRL_CVPO_ST_DUAL_STD = 13, FSRL_CVPO_ST_ENTROPY = 14 };
typedef struct fsrl_cvpo {
    fsrl_offpolicy_t off;
    int K, estep_iters, mstep_iters, cond_sigma;
    float estep_kl, estep_dual_max, estep_dual_lr, qc_thres;
    float mstep_kl_mu, mstep_kl_std, mstep_dual_max, mstep_dual_lr;
    float* estep_state;
    float* mstep_state;
    float* particles;
    int* part_idx;
    float *mu_old, *std_old, *comb, *weights;
    const float *log_sigma, *log_sigma_old;
} fsrl_cvpo_t;

int fsrl_cvpo_steps(const fsrl_cvpo_t* d, const int* idx_all, int n_steps, int B,
                    long long critic_t0, long long actor_t0, unsigned long long noise_t0, float* stats,
                    void* stream);

/* ---- a11: CPO (and the CG / Fisher machinery TRPO-Lag shares) ------------------------------------
 * Replaces CPO._get_objective/_get_cost_surrogate/_MVP/_conjugate_gradients/policy_loss
 * (fsrl/policy/cpo.py:163-204,234-351).  The batch is resident: a saved engine forward of the
 * actor (P slot = actor.nets[0].slot) caches h1, h2 and the head output for all N rows;
 * actor_r is the SAME network with a second scratch slot for the R-op quantities.
 *   fsrl_cpo_head(mode)  per-row ratio / KL terms: sums[0..2] = sum ratio*adv_r, sum ratio*adv_c,
 *                        sum kl; mode 1/2/3 also writes the head gradient of the objective,
 *                        of -cost_surrogate, of the mean KL into the P slot's dout
 *   fsrl_cpo_hvp         hv = Hessian(mean KL) v + damping v, exact (R-op), needs the P slot's
 *                        dout / dz2 of the KL gradient pass
 *   fsrl_vec_*           the O(P) vector arithmetic of conjugate gradients / line search */
typedef struct fsrl_cpo {
    fsrl_engine_t eng;
    fsrl_netlist_t actor, actor_r;
    long long N, ld;
    int A, bounded;
    float max_action, pad0;
    const float *obs, *act, *logp_old, *mean_old, *std_old, *adv; /* adv: [2][ld] */
    const int* perm;       /* optional minibatch row indices (NULL = rows 0..N-1) */
    const float* out;      /* P slot head output  [bmax][16] */
    float* dout;           /* P slot head gradient [bmax][16] */
    const float* log_sigma;
} fsrl_cpo_t;

int fsrl_cpo_head(const fsrl_cpo_t* d, int mode, double* sums_dev4, void* stream);
/* FOCOPS actor head (fsrl/policy/focops.py:188-215): loss = mean((KL(new||old) - ratio (A_r - nu A_c) /
 * lambda) * 1[KL <= eta]); d->adv = per-minibatch-normalised advantages; writes d->dout, and
 * sums_dev4 = [sum loss_i, sum KL_i, #rows inside the trust region, 0] */
int fsrl_focops_head(const fsrl_cpo_t* d, double inv_lambda, double nu, double eta, double* sums_dev4,
                     void* stream);
int fsrl_cpo_hvp(const fsrl_cpo_t* d, const float* v, float* v_w2n_scratch, float* hv, double damping,
                 void* stream);
/* x_out = CG(H, rhs), H v = fsrl_cpo_hvp(v): CPO._conjugate_gradients (fsrl/policy/cpo.py:184-204) / TRPOLagrangian
 * (trpo_lag.py:261-283) with every scalar on the device -- `nsteps` iterations enqueued without host synchronisation,
 * the reference's residual break is a device flag.  work: 4 P floats, state_dev: 8 doubles. */
int fsrl_cg_solve(const fsrl_cpo_t* d, const float* rhs, float* x_out, float* work, float* v_w2n_scratch,
                  double* state_dev, long long P, int nsteps, double tol, double damping, void* stream);
int fsrl_vec_dot(const float* a, const float* b, long long n, double* out_dev, void* stream);
int fsrl_vec_axpby(double a, const float* x, double b, float* y, long long n, void* stream);
int fsrl_vec_add_scaled(const float* a, double s, const float* b, float* out, long long n, void* stream);
/* critic regression head (cpo.py:147-157, trpo_lag.py:135-146): dout[i][0] = 2 (V_i - ret_i) / N,
 * sums_dev[0] += sum td^2;  fsrl_standardize: x <- (x - mean) / std (unbiased), cpo.py:127-131 */
int fsrl_mse_head(const float* out, const float* ret, const int* perm, long long N, float* dout,
                  double* sums_dev, void* stream);
int fsrl_standardize(float* x, long long n, void* stream);
int fsrl_engine_wgrad_to(const fsrl_engine_t* e, const fsrl_netlist_t* net1, const fsrl_eng_input_t* in,
                         long long B, float* dst, void* stream);

/* ---- 8(e): multi-GPU plumbing (one process per GPU, NCCL over NVLink) -------------------------
 * The reference has no distributed code; ranks own env shards and replay shards, and per
 * optimiser step ONE all-reduce of the flat gradient buffer is issued from the C update loop.
 * The 128-byte unique id is created on rank 0 and broadcast by the host (torch.distributed). */
int fsrl_comm_unique_id(char* out128);
int fsrl_comm_init(const char* id128, int rank, int world, void** comm_out);
int fsrl_comm_destroy(void* comm);
int fsrl_allreduce_fused(void* comm, float* buf, long long n, void* stream);
int fsrl_allreduce_f64(void* comm, double* buf, long long n, void* stream);
/* Peer-memory exchange block of one rank: [xg0 | xg1 | flags | err | partials], each gradient buffer padded
 * to fsrl_p2p_stride(n) floats.  alloc: cudaMalloc + zero + IPC handle (64 bytes) for the other
 * processes; open / close: map / unmap a peer's block; free: release the own block. */
#define FSRL_P2P_MAX_RANKS 8
#define FSRL_P2P_PARTIALS 4096   /* one per 1024 parameters: peer exchange handles up to 4M parameters */
long long fsrl_p2p_stride(long long n_floats);
long long fsrl_p2p_block_bytes(long long n_floats);
int fsrl_p2p_alloc(long long n_floats, void** base_out, char* ipc64_out);
int fsrl_p2p_open(const char* ipc64, void** peer_base_out);
int fsrl_p2p_close(void* peer_base);
int fsrl_p2p_free(void* base);
int fsrl_p2p_poll_error(const int* err_dev, int* out_host); /* 1 = a peer never arrived */
/* in-place sum of `n_ranges` sub-ranges [base + offs[i], base + offs[i] + counts[i]) in ONE grouped
 * NCCL call (the gradient slices of a net list inside the flat gradient buffer) */
int fsrl_allreduce_ranges(void* comm, float* base, const long long* offs, const long long* counts,
                          int n_ranges, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FSRL_B200_H */
