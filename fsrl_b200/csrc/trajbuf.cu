// Offline-dataset harvest: finished episodes go from the rollout ring (rollout.cu) into the
// trajectory arena of TrajectoryBuffer (fsrl_b200/data/traj_buf.py) without a host round trip.
// The reference grows every trajectory with a per-transition Batch.cat on the host
// (/root/reference/fsrl/data/traj_buf.py:60-95, fed one step at a time by basic_collector.py:238-248).
//   scan   one thread per env walks the ring slots written since the last scan and emits one
//          row per finished episode (return / cost summed in fp64 in time order, as ep_rew)
//   copy   one CTA per kept episode: ring -> arena slot, actions remapped like the env saw them; the
//          ring of host-stepped envs takes the same kernel with its widths from the caller (no scan:
//          the host collect loop knows every finished episode)
//   gather one CTA per kept trajectory: arena slots -> contiguous tensors (get_all / save)
// copy and gather are bandwidth-bound: 16-byte streaming loads and stores wherever source and
// destination share their alignment.
#include "envs.cuh"
#include "fsrl_b200.h"

namespace fsrl {

constexpr int TRAJ_TPB = 256;

__global__ void __launch_bounds__(128) traj_begin_kernel(const fsrl_rollout_t r, const fsrl_traj_scan_t h) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= r.E) return;
    const int ptr = r.b_ptr[e];
    h.last[e] = ptr; h.open[e] = ptr; h.open_len[e] = 0; h.steps[e] = 0;
    h.rew[e] = 0.0; h.cost[e] = 0.0;
}

__global__ void __launch_bounds__(128) traj_scan_kernel(const fsrl_rollout_t r, const fsrl_traj_scan_t h, int n_ready) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= r.E) return;
    const int cap = (int)r.cap;
    int p = h.last[e];
    int n = r.b_ptr[e] - p;
    if (n < 0) n += cap;
    if (n == 0 && e < n_ready) n = cap;        // one-episode path: a full ring wrap
    int open = h.open[e], olen = h.open_len[e], steps = h.steps[e];
    double rw = h.rew[e], cs = h.cost[e];
    const size_t base = (size_t)e * r.cap;
    for (int i = 0; i < n; ++i) {
        const size_t q = base + p;
        rw = rw + (double)r.b_rew[q];           // same order and rounding as ep_rew in rollout.cu
        cs = cs + (double)r.b_cost[q];
        ++olen; ++steps;
        const int te = r.b_term[q], tr = r.b_trunc[q];
        if (++p == cap) p = 0;
        if (te | tr) {
            const int k = atomicAdd(h.n_rows, 1);
            if (k < h.row_cap) {
                fsrl_traj_row_t row;
                row.env = e; row.start = open; row.len = olen; row.finish = steps;
                row.terminated = te; row.truncated = tr; row.ret = rw; row.cost = cs;
                h.rows[k] = row;
            }
            open = p; olen = 0; rw = 0.0; cs = 0.0;
        }
    }
    h.last[e] = p; h.open[e] = open; h.open_len[e] = olen; h.steps[e] = steps;
    h.rew[e] = rw; h.cost[e] = cs;
}

// dst[0..n) = src[0..n) by the whole CTA; float4 body when both pointers share their 16-byte phase
__device__ __forceinline__ void copy_span(float* __restrict__ dst, const float* __restrict__ src, long long n) {
    long long head = 0;
    const bool vec = ((reinterpret_cast<uintptr_t>(dst) ^ reinterpret_cast<uintptr_t>(src)) & 15u) == 0;
    if (vec) {
        head = (long long)((16u - (reinterpret_cast<uintptr_t>(dst) & 15u)) & 15u) / 4;
        if (head > n) head = n;
        const long long n4 = (n - head) / 4;
        const float* s4 = src + head;
        float* d4 = dst + head;
        for (long long i = threadIdx.x; i < n4; i += blockDim.x) stg_stream4(d4 + 4 * i, ldg_stream4(s4 + 4 * i));
        for (long long i = head + 4 * n4 + threadIdx.x; i < n; i += blockDim.x) dst[i] = __ldcs(src + i);
        for (long long i = threadIdx.x; i < head; i += blockDim.x) dst[i] = __ldcs(src + i);
    } else {
        for (long long i = threadIdx.x; i < n; i += blockDim.x) dst[i] = __ldcs(src + i);
    }
}

__device__ __forceinline__ void copy_bytes(unsigned char* __restrict__ dst, const unsigned char* __restrict__ src,
                                           long long n) {
    for (long long i = threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
}

__global__ void __launch_bounds__(TRAJ_TPB) traj_copy_kernel(const fsrl_rollout_t r, const fsrl_traj_arena_t a,
                                                             const int4* __restrict__ jobs) {
    const int4 j = jobs[blockIdx.x];
    const int e = j.x, start = j.y, len = j.z;
    const long long cap = r.cap, D = a.D, A = a.A;
    const long long first = (len < cap - start) ? len : cap - start;   // slots before the ring wraps
    const long long src0 = (long long)e * cap + start, src1 = (long long)e * cap;
    const long long dst = (long long)j.w * a.stride;
    copy_span(a.obs + dst * D, r.b_obs + src0 * D, first * D);
    copy_span(a.obs + (dst + first) * D, r.b_obs + src1 * D, (len - first) * D);
    copy_span(a.obs_next + dst * D, r.b_obs_next + src0 * D, first * D);
    copy_span(a.obs_next + (dst + first) * D, r.b_obs_next + src1 * D, (len - first) * D);
    copy_span(a.rew + dst, r.b_rew + src0, first);
    copy_span(a.rew + dst + first, r.b_rew + src1, len - first);
    copy_span(a.cost + dst, r.b_cost + src0, first);
    copy_span(a.cost + dst + first, r.b_cost + src1, len - first);
    copy_bytes(a.term + dst, r.b_term + src0, first);
    copy_bytes(a.term + dst + first, r.b_term + src1, len - first);
    copy_bytes(a.trunc + dst, r.b_trunc + src0, first);
    copy_bytes(a.trunc + dst + first, r.b_trunc + src1, len - first);
    // the env's action: map_action of the raw action the ring holds (basic_collector.py:191,242)
    for (long long i = threadIdx.x; i < (long long)len * A; i += blockDim.x) {
        const long long t = i / A;
        const int c = (int)(i - t * A);
        const long long src = (t < first ? src0 + t : src1 + (t - first)) * A + c;
        a.act[dst * A + i] = map_action(__ldcs(r.b_act + src), r.action_bound, r.action_scaling,
                                        r.act_low[c], r.act_high[c]);
    }
}

__global__ void __launch_bounds__(TRAJ_TPB) traj_gather_kernel(const fsrl_traj_arena_t a, const fsrl_traj_arena_t o,
                                                               const longlong3* __restrict__ jobs) {
    const longlong3 j = jobs[blockIdx.x];
    const long long src = j.x * a.stride, len = j.y, dst = j.z, D = a.D, A = a.A;
    copy_span(o.obs + dst * D, a.obs + src * D, len * D);
    copy_span(o.obs_next + dst * D, a.obs_next + src * D, len * D);
    copy_span(o.act + dst * A, a.act + src * A, len * A);
    copy_span(o.rew + dst, a.rew + src, len);
    copy_span(o.cost + dst, a.cost + src, len);
    copy_bytes(o.term + dst, a.term + src, len);
    copy_bytes(o.trunc + dst, a.trunc + src, len);
}

}  // namespace fsrl

using namespace fsrl;

// host: the descriptor of a host-stepped env (kind -1), whose widths the caller gives
static int check_ring(const fsrl_rollout_t* r, bool host = false) {
    FSRL_REQUIRE(r != nullptr, "trajectory harvest: null rollout descriptor");
    if (host)
        FSRL_REQUIRE(r->kind == -1, "trajectory copy: a host ring has env kind -1, got %d", r->kind);
    else {
        EnvDims d;
        FSRL_REQUIRE(env_kind_dims(r->kind, d), "trajectory harvest: unknown env kind %d", r->kind);
    }
    FSRL_REQUIRE(r->E > 0 && r->cap > 0, "trajectory harvest: E and cap must be positive");
    FSRL_REQUIRE(r->b_obs && r->b_obs_next && r->b_act && r->b_rew && r->b_cost && r->b_term && r->b_trunc &&
                 r->b_ptr, "trajectory harvest: the rollout has no transition ring");
    return FSRL_OK;
}

static int check_scan(const fsrl_traj_scan_t* h) {
    FSRL_REQUIRE(h != nullptr && h->last && h->open && h->open_len && h->steps && h->rew && h->cost && h->rows &&
                 h->n_rows && h->row_cap >= 0, "trajectory scan: null harvest state");
    return FSRL_OK;
}

static int check_arena(const fsrl_traj_arena_t* a) {
    FSRL_REQUIRE(a != nullptr && a->obs && a->obs_next && a->act && a->rew && a->cost && a->term && a->trunc,
                 "trajectory arena: null pointer");
    FSRL_REQUIRE(a->D > 0 && a->A > 0 && a->A <= ENV_MAX_A, "trajectory arena: bad dims D=%d A=%d", a->D, a->A);
    return FSRL_OK;
}

extern "C" int fsrl_traj_begin(const fsrl_rollout_t* r, const fsrl_traj_scan_t* h, void* stream) {
    int rc = check_ring(r);
    if (rc || (rc = check_scan(h))) return rc;
    traj_begin_kernel<<<(r->E + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(*r, *h);
    FSRL_LAUNCH_CHECK();
    return FSRL_OK;
}

extern "C" int fsrl_traj_scan(const fsrl_rollout_t* r, const fsrl_traj_scan_t* h, int n_ready, void* stream) {
    int rc = check_ring(r);
    if (rc || (rc = check_scan(h))) return rc;
    FSRL_REQUIRE(n_ready >= 0 && n_ready <= r->E, "trajectory scan: n_ready %d outside [0, E]", n_ready);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    FSRL_CUDA(cudaMemsetAsync(h->n_rows, 0, sizeof(int), s));
    traj_scan_kernel<<<(r->E + 127) / 128, 128, 0, s>>>(*r, *h, n_ready);
    FSRL_LAUNCH_CHECK();
    return FSRL_OK;
}

static int launch_copy(const fsrl_rollout_t* r, const fsrl_traj_arena_t* a, int D, int A, const int* jobs,
                       int n_jobs, void* stream) {
    FSRL_REQUIRE(a->D == D && a->A == A, "trajectory copy: arena dims (%d, %d) != env dims (%d, %d)",
                 a->D, a->A, D, A);
    FSRL_REQUIRE(n_jobs >= 0 && (n_jobs == 0 || jobs), "trajectory copy: bad job list");
    FSRL_REQUIRE((reinterpret_cast<uintptr_t>(jobs) & 15u) == 0, "trajectory copy: jobs must be 16-byte aligned");
    if (n_jobs == 0) return FSRL_OK;
    traj_copy_kernel<<<n_jobs, TRAJ_TPB, 0, static_cast<cudaStream_t>(stream)>>>(
        *r, *a, reinterpret_cast<const int4*>(jobs));
    FSRL_LAUNCH_CHECK();
    return FSRL_OK;
}

extern "C" int fsrl_traj_copy(const fsrl_rollout_t* r, const fsrl_traj_arena_t* a, const int* jobs, int n_jobs,
                              void* stream) {
    int rc = check_ring(r);
    if (rc || (rc = check_arena(a))) return rc;
    EnvDims d;
    env_kind_dims(r->kind, d);
    return launch_copy(r, a, d.D, d.A, jobs, n_jobs, stream);
}

extern "C" int fsrl_traj_copy_host(const fsrl_rollout_t* r, const fsrl_traj_arena_t* a, int D, int A,
                                   const int* jobs, int n_jobs, void* stream) {
    int rc = check_ring(r, true);
    if (rc || (rc = check_arena(a))) return rc;
    FSRL_REQUIRE(D >= 1 && A >= 1 && A <= ENV_MAX_A, "trajectory copy: bad host ring dims D=%d A=%d", D, A);
    return launch_copy(r, a, D, A, jobs, n_jobs, stream);
}

extern "C" int fsrl_traj_gather(const fsrl_traj_arena_t* a, const fsrl_traj_arena_t* out, const long long* jobs,
                                int n_jobs, void* stream) {
    int rc = check_arena(a);
    if (rc || (rc = check_arena(out))) return rc;
    FSRL_REQUIRE(a->D == out->D && a->A == out->A, "trajectory gather: dims differ");
    FSRL_REQUIRE(n_jobs >= 0 && (n_jobs == 0 || jobs), "trajectory gather: bad job list");
    FSRL_REQUIRE((reinterpret_cast<uintptr_t>(jobs) & 7u) == 0, "trajectory gather: jobs must be 8-byte aligned");
    if (n_jobs == 0) return FSRL_OK;
    traj_gather_kernel<<<n_jobs, TRAJ_TPB, 0, static_cast<cudaStream_t>(stream)>>>(
        *a, *out, reinterpret_cast<const longlong3*>(jobs));
    FSRL_LAUNCH_CHECK();
    return FSRL_OK;
}
