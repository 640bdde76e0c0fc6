// Observation normalization on the device: tianshou's VectorEnvNormObs / RunningMeanStd with the running
// statistics in float64 on the GPU (fsrl_obs_rms_t in fsrl_b200.h).
//   obs_rms_partials_kernel  one CTA per tile of FSRL_OBS_RMS_TILE env ids: (count, mean, M2) of the tile's
//                            selected rows, summed in ascending id order; CTA 0 also snapshots the running
//                            statistics, which the next launch reads while its CTA 0 overwrites them
//   obs_rms_apply_kernel     every CTA merges the tile partials in tile order into the batch moments and
//                            those into the snapshot (the Chan update of utils/optim_util.RunningMeanStd),
//                            CTA 0 publishes; then each CTA normalizes the selected rows of its env range
// The two launches have no floating-point atomics and fixed reduction orders, so the bits depend only on
// which rows the envs hold.
#include "obsnorm.cuh"

#include <vector>

namespace fsrl {

constexpr int OBS_TILE = FSRL_OBS_RMS_TILE;
constexpr int OBS_APPLY_ROWS = 32;     // env rows per CTA of obs_rms_apply_kernel
constexpr int OBS_APPLY_TPB = 256;
constexpr int OBS_MAX_D = FSRL_ENG_DX_LD;

// the workspace, in bytes from `work`
struct ObsWork {
    size_t snap_count, snap_mean, snap_var, part_n, part_mean, part_m2, ids, mask, total;
    __host__ __device__ ObsWork(int E, int D) {
        const size_t T = ((size_t)E + OBS_TILE - 1) / OBS_TILE;
        auto up = [](size_t v) { return (v + 15) & ~(size_t)15; };
        snap_count = 0;
        snap_mean = 16;
        snap_var = up(snap_mean + 8 * (size_t)D);
        part_n = up(snap_var + 8 * (size_t)D);
        part_mean = up(part_n + 8 * T);
        part_m2 = up(part_mean + 8 * T * D);
        ids = up(part_m2 + 8 * T * D);
        mask = up(ids + 4 * (size_t)E);
        total = up(mask + (size_t)E);
    }
};

template <class T>
__host__ __device__ __forceinline__ T* work_at(void* w, size_t off) {
    return reinterpret_cast<T*>(static_cast<char*>(w) + off);
}

struct ObsKArgs {
    fsrl_obs_rms_t n;
    float* x;
    int E, sel, ring;
    // rollout state of the collect passes
    const uint8_t* active;
    const int* env_t;
    const fsrl_collect_stats_t* stats;
    float* b_obs_next;
    const int* b_ptr;
    long long cap;
};

__device__ __forceinline__ bool obs_selected(const ObsKArgs& p, const uint8_t* mask, int e) {
    if (!mask[e]) return false;
    if (p.sel == OBS_SEL_STEPPED) return !p.stats->finished;
    if (p.sel == OBS_SEL_RESTARTED) return p.active[e] && p.env_t[e] == 0;
    return true;
}

__global__ void __launch_bounds__(OBS_TILE) obs_rms_partials_kernel(const ObsKArgs p) {
    const int D = p.n.D, t = blockIdx.x, tid = threadIdx.x;
    const ObsWork w(p.E, D);
    const uint8_t* mask = work_at<uint8_t>(p.n.work, w.mask);
    __shared__ unsigned char s_sel[OBS_TILE];
    const int e0 = t * OBS_TILE;
    const int e = e0 + tid;
    const bool sel = e < p.E && obs_selected(p, mask, e);
    s_sel[tid] = sel ? 1 : 0;
    const int cnt = __syncthreads_count(sel);
    double* pm = work_at<double>(p.n.work, w.part_mean) + (size_t)t * D;
    double* pm2 = work_at<double>(p.n.work, w.part_m2) + (size_t)t * D;
    for (int d = tid; d < D; d += OBS_TILE) {
        double sum = 0.0;
        for (int r = 0; r < OBS_TILE; ++r)
            if (s_sel[r]) sum = __dadd_rn(sum, (double)p.x[(size_t)(e0 + r) * D + d]);
        const double mean = cnt ? __ddiv_rn(sum, (double)cnt) : 0.0;
        double m2 = 0.0;
        for (int r = 0; r < OBS_TILE; ++r)
            if (s_sel[r]) {
                const double dv = __dsub_rn((double)p.x[(size_t)(e0 + r) * D + d], mean);
                m2 = __dadd_rn(m2, __dmul_rn(dv, dv));
            }
        pm[d] = mean;
        pm2[d] = m2;
    }
    if (tid == 0) work_at<long long>(p.n.work, w.part_n)[t] = cnt;
    if (t == 0) {
        for (int d = tid; d < D; d += OBS_TILE) {
            work_at<double>(p.n.work, w.snap_mean)[d] = p.n.mean[d];
            work_at<double>(p.n.work, w.snap_var)[d] = p.n.var[d];
        }
        if (tid == 0) *work_at<long long>(p.n.work, w.snap_count) = *p.n.count;
    }
}

__global__ void __launch_bounds__(OBS_APPLY_TPB) obs_rms_apply_kernel(const ObsKArgs p) {
    const int D = p.n.D, tid = threadIdx.x;
    const ObsWork w(p.E, D);
    uint8_t* mask = work_at<uint8_t>(p.n.work, w.mask);
    __shared__ double s_mean[OBS_MAX_D], s_sd[OBS_MAX_D];
    __shared__ unsigned char s_sel[OBS_APPLY_ROWS];
    const int e0 = blockIdx.x * OBS_APPLY_ROWS;
    if (tid < OBS_APPLY_ROWS) {
        const int e = e0 + tid;
        s_sel[tid] = (e < p.E && obs_selected(p, mask, e)) ? 1 : 0;
    }
    for (int d = tid; d < D; d += OBS_APPLY_TPB) {
        double mean, var;
        if (p.n.update) {
            // the batch: tile partials merged in tile order
            const long long* pn = work_at<long long>(p.n.work, w.part_n);
            const double* pm = work_at<double>(p.n.work, w.part_mean);
            const double* pm2 = work_at<double>(p.n.work, w.part_m2);
            const int T = (p.E + OBS_TILE - 1) / OBS_TILE;
            long long nb = 0;
            double mb = 0.0, m2b = 0.0;
            for (int t = 0; t < T; ++t) {
                const long long nt = pn[t];
                if (nt == 0) continue;
                const double mt = pm[(size_t)t * D + d], m2t = pm2[(size_t)t * D + d];
                if (nb == 0) { nb = nt; mb = mt; m2b = m2t; continue; }
                const long long tot = nb + nt;
                const double delta = __dsub_rn(mt, mb);
                mb = __dadd_rn(mb, __ddiv_rn(__dmul_rn(delta, (double)nt), (double)tot));
                m2b = __dadd_rn(__dadd_rn(m2b, m2t),
                                __ddiv_rn(__dmul_rn(__dmul_rn(__dmul_rn(delta, delta), (double)nb), (double)nt), (double)tot));
                nb = tot;
            }
            const long long na = *work_at<long long>(p.n.work, w.snap_count);
            mean = work_at<double>(p.n.work, w.snap_mean)[d];
            var = work_at<double>(p.n.work, w.snap_var)[d];
            if (nb > 0) {
                // RunningMeanStd.update_moments(batch mean, batch population variance, nb)
                const double var_b = __ddiv_rn(m2b, (double)nb);
                const double delta = __dsub_rn(mb, mean);
                const long long tot = na + nb;
                const double m2 = __dadd_rn(__dadd_rn(__dmul_rn(var, (double)na), __dmul_rn(var_b, (double)nb)),
                                            __ddiv_rn(__dmul_rn(__dmul_rn(__dmul_rn(delta, delta), (double)na), (double)nb),
                                                      (double)tot));
                mean = __dadd_rn(mean, __ddiv_rn(__dmul_rn(delta, (double)nb), (double)tot));
                var = __ddiv_rn(m2, (double)tot);
                if (blockIdx.x == 0) {
                    p.n.mean[d] = mean;
                    p.n.var[d] = var;
                    if (d == 0) *p.n.count = tot;
                }
            }
        } else {
            mean = p.n.mean[d];
            var = p.n.var[d];
        }
        s_mean[d] = mean;
        s_sd[d] = __dsqrt_rn(__dadd_rn(var, p.n.eps));
    }
    __syncthreads();
    if (p.sel == OBS_SEL_RESTARTED && tid < OBS_APPLY_ROWS) {
        const int e = e0 + tid;
        if (e < p.E) mask[e] = (p.active[e] && !p.stats->finished) ? 1 : 0;
    }
    const double clip = p.n.clip_max;
    for (int i = tid; i < OBS_APPLY_ROWS * D; i += OBS_APPLY_TPB) {
        const int r = i / D, d = i - r * D;
        if (!s_sel[r]) continue;
        const int e = e0 + r;
        float* xp = p.x + (size_t)e * D + d;
        double y = __ddiv_rn(__dsub_rn((double)*xp, s_mean[d]), s_sd[d]);
        // comparisons rather than fmin/fmax, which return the non-NaN operand: a NaN stays NaN, as in np.clip
        if (clip > 0.0) y = y < -clip ? -clip : (y > clip ? clip : y);
        const float f = (float)y;
        *xp = f;
        if (p.ring) {
            const int ptr = p.b_ptr[e];
            const long long slot = (long long)e * p.cap + (ptr == 0 ? p.cap - 1 : ptr - 1);
            p.b_obs_next[slot * D + d] = f;
        }
    }
}

// mask[e] = active[e] && !finished
__global__ void obs_norm_snapshot_kernel(const uint8_t* active, const fsrl_collect_stats_t* st, uint8_t* mask, int E) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < E) mask[e] = (active[e] && !st->finished) ? 1 : 0;
}

// mask[ids[k]] = 1 and, with rows_in, x[ids[k]] = rows_in[k]
__global__ void obs_rows_mark_kernel(const int* ids, int count, uint8_t* mask, float* x, const float* rows_in, int D) {
    const int k = blockIdx.x * blockDim.y + threadIdx.y;
    if (k >= count) return;
    const int e = ids ? ids[k] : k;
    if (threadIdx.x == 0) mask[e] = 1;
    if (rows_in)
        for (int d = threadIdx.x; d < D; d += blockDim.x) x[(size_t)e * D + d] = rows_in[(size_t)k * D + d];
}

__global__ void obs_rows_gather_kernel(const float* x, int D, const int* ids, int count, float* out) {
    const int k = blockIdx.x * blockDim.y + threadIdx.y;
    if (k >= count) return;
    const int e = ids ? ids[k] : k;
    for (int d = threadIdx.x; d < D; d += blockDim.x) out[(size_t)k * D + d] = x[(size_t)e * D + d];
}

int check_obs_rms(const char* fn, const fsrl_obs_rms_t* n, int E, int D) {
    FSRL_REQUIRE(n != nullptr, "%s: null obs_rms descriptor", fn);
    FSRL_REQUIRE(E > 0, "%s: E must be positive", fn);
    FSRL_REQUIRE(n->D >= 1 && n->D <= OBS_MAX_D, "%s: obs_rms D = %d outside [1, %d]", fn, n->D, OBS_MAX_D);
    FSRL_REQUIRE(D < 0 || n->D == D, "%s: obs_rms D = %d != observation width %d", fn, n->D, D);
    FSRL_REQUIRE(n->mean && n->var && n->count && n->work, "%s: null obs_rms pointer", fn);
    FSRL_REQUIRE(n->eps >= 0.0, "%s: eps %g < 0", fn, n->eps);
    return FSRL_OK;
}

static ObsKArgs kargs(const fsrl_obs_rms_t& n, float* x, int E, int sel, int ring, const fsrl_rollout_t* a) {
    ObsKArgs k;
    k.n = n; k.x = x; k.E = E; k.sel = sel; k.ring = 0;
    k.active = nullptr; k.env_t = nullptr; k.stats = nullptr; k.b_obs_next = nullptr; k.b_ptr = nullptr; k.cap = 0;
    if (a) {
        k.active = a->active; k.env_t = a->env_t; k.stats = a->stats;
        if (ring && a->b_obs_next) {
            k.ring = 1; k.b_obs_next = a->b_obs_next; k.b_ptr = a->b_ptr; k.cap = a->cap;
        }
    }
    return k;
}

int launch_obs_norm(const ObsNormPass& p, cudaStream_t s) {
    const ObsKArgs k = kargs(*p.n, p.x, p.E, p.sel, p.ring, p.a);
    if (p.n->update) {
        obs_rms_partials_kernel<<<(p.E + OBS_TILE - 1) / OBS_TILE, OBS_TILE, 0, s>>>(k);
        FSRL_LAUNCH_CHECK();
    }
    obs_rms_apply_kernel<<<(p.E + OBS_APPLY_ROWS - 1) / OBS_APPLY_ROWS, OBS_APPLY_TPB, 0, s>>>(k);
    FSRL_LAUNCH_CHECK();
    return FSRL_OK;
}

int launch_obs_norm_snapshot(const fsrl_rollout_t& a, const fsrl_obs_rms_t& n, cudaStream_t s) {
    const ObsWork w(a.E, n.D);
    obs_norm_snapshot_kernel<<<(a.E + 255) / 256, 256, 0, s>>>(a.active, a.stats, work_at<uint8_t>(n.work, w.mask), a.E);
    FSRL_LAUNCH_CHECK();
    return FSRL_OK;
}

int launch_obs_gather(const float* x, int D, const int* ids, int count, float* out, cudaStream_t s) {
    if (count <= 0) return FSRL_OK;
    const dim3 blk(32, 8);
    obs_rows_gather_kernel<<<(count + 7) / 8, blk, 0, s>>>(x, D, ids, count, out);
    FSRL_LAUNCH_CHECK();
    return FSRL_OK;
}

int launch_obs_norm_rows(const fsrl_obs_rms_t& n, float* x, int E, const int* ids, int count, const float* rows_in,
                         float* out, cudaStream_t s) {
    if (count <= 0) return FSRL_OK;             // an empty batch: no update, nothing to normalize
    const ObsWork w(E, n.D);
    uint8_t* mask = work_at<uint8_t>(n.work, w.mask);
    FSRL_CUDA(cudaMemsetAsync(mask, 0, (size_t)E, s));
    const dim3 blk(32, 8);
    obs_rows_mark_kernel<<<(count + 7) / 8, blk, 0, s>>>(ids, count, mask, x, rows_in, n.D);
    FSRL_LAUNCH_CHECK();
    ObsNormPass p{&n, x, E, OBS_SEL_MASK, 0, nullptr};
    int rc = launch_obs_norm(p, s);
    if (rc) return rc;
    if (out) return launch_obs_gather(x, n.D, ids, count, out, s);
    return FSRL_OK;
}

}  // namespace fsrl

using namespace fsrl;

extern "C" size_t fsrl_obs_rms_work_bytes(int E, int D) {
    if (E <= 0 || D <= 0) return 0;
    return ObsWork(E, D).total;
}

extern "C" int fsrl_obs_rms_rows(const fsrl_obs_rms_t* n, float* x, int E, const int32_t* ids, int count,
                                 const float* rows_in, float* out, void* stream) {
    int rc = check_obs_rms("fsrl_obs_rms_rows", n, E, -1);
    if (rc) return rc;
    FSRL_REQUIRE(x != nullptr, "fsrl_obs_rms_rows: null observation array");
    FSRL_REQUIRE(count >= 0 && count <= E, "fsrl_obs_rms_rows: count = %d outside [0, E = %d]", count, E);
    FSRL_REQUIRE(ids != nullptr || count == E, "fsrl_obs_rms_rows: without ids, count must be E = %d (got %d)", E, count);
    if (ids) {
        std::vector<unsigned char> seen(E, 0);
        for (int k = 0; k < count; ++k) {
            FSRL_REQUIRE(ids[k] >= 0 && ids[k] < E, "fsrl_obs_rms_rows: ids[%d] = %d outside [0, E = %d)", k, ids[k], E);
            FSRL_REQUIRE(!seen[ids[k]], "fsrl_obs_rms_rows: env %d listed twice", ids[k]);
            seen[ids[k]] = 1;
        }
    }
    if (count == 0) return FSRL_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int* ids_dev = nullptr;
    if (ids) {
        int* w = work_at<int>(n->work, ObsWork(E, n->D).ids);
        FSRL_CUDA(cudaMemcpyAsync(w, ids, sizeof(int32_t) * (size_t)count, cudaMemcpyHostToDevice, s));
        ids_dev = w;
    }
    return launch_obs_norm_rows(*n, x, E, ids_dev, count, rows_in, out, s);
}
