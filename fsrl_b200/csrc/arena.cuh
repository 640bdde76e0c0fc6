// One network inside the flat fp32 parameter arena, and the two updates every optimiser kernel
// shares: torch's Adam step and the upkeep of the out-major W2 mirror.
//
// Layout of one network (gradients and Adam moments use the same one); the host side is
// nets.py::Arena, and include/fsrl_b200.h documents it with fsrl_ppo_update_t:
//   w1t[D][H] | b1[H] | w2t[H][H] | b2[H] | w3t[H][out] | b3[out] | extra[n_extra]
// Every Linear is stored transposed, Wt[in][out] row-major; `extra` holds the actor's log-sigma.
#pragma once
#include "common.cuh"

namespace fsrl {

struct Mlp3 {            // device pointers, canonical layout
    const float* w1t;    // [in][H]
    const float* b1;     // [H]
    const float* w2t;    // [H][H]
    const float* b2;     // [H]
    const float* w3t;    // [H][out]
    const float* b3;     // [out]
    int in, H, out;
};

struct ArenaLayout {     // offsets (floats) of the blocks of one network, and its size
    long long w1, b1, w2, b2, w3, b3, extra, size;
};

__host__ __device__ constexpr ArenaLayout arena_layout(int D, int H, int out, int n_extra) {
    const long long b1 = (long long)D * H, w2 = b1 + H, b2 = w2 + (long long)H * H, w3 = b2 + H,
                    b3 = w3 + (long long)H * out, extra = b3 + out;
    return ArenaLayout{0, b1, w2, b2, w3, b3, extra, extra + n_extra};
}

// Parameter and gradient half of a network view: theta / grad point at the network's start in
// the arena (or in any vector of the same layout), w2n at its W2 mirror.
struct ArenaNet {
    Mlp3 m;
    const float* w2n;      // out-major mirror [H][H] of w2t (the backward GEMM's B operand)
    const float* extra;
    float *g_w1t, *g_b1, *g_w2t, *g_b2, *g_w3t, *g_b3, *g_extra;
};

// Fills v in place, walking the blocks in arena_layout's order with a running offset: the views
// live in registers of the update kernels, and this form keeps their code as compact as before.
__host__ __device__ __forceinline__ void arena_net(ArenaNet& v, const float* theta, float* grad, const float* w2n,
                                                   int D, int H, int out) {
    size_t o = 0;
    v.m.w1t = theta + o; v.g_w1t = grad + o; o += (size_t)D * H;
    v.m.b1 = theta + o;  v.g_b1 = grad + o;  o += H;
    v.m.w2t = theta + o; v.g_w2t = grad + o; o += (size_t)H * H;
    v.m.b2 = theta + o;  v.g_b2 = grad + o;  o += H;
    v.m.w3t = theta + o; v.g_w3t = grad + o; o += (size_t)H * out;
    v.m.b3 = theta + o;  v.g_b3 = grad + o;  o += out;
    v.extra = theta + o; v.g_extra = grad + o;
    v.m.in = D; v.m.H = H; v.m.out = out;
    v.w2n = w2n;
}

// ---- Adam (torch.optim.Adam, single-tensor arithmetic order) ---------------------------------
struct AdamStep {
    float w1, b2, w2, bc2s, eps, neg_step;   // 1 - beta1, beta2, 1 - beta2, sqrt(1 - beta2^t), eps, -lr / (1 - beta1^t)
};

// the scalars of step t as torch computes them: python doubles, rounded to f32 at the op
__host__ __device__ inline AdamStep adam_step_scalars(double lr, double beta1, double beta2, double eps, long long t) {
    const double bc1 = 1.0 - pow(beta1, (double)t), bc2 = 1.0 - pow(beta2, (double)t);
    return AdamStep{(float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2), (float)sqrt(bc2), (float)eps,
                    (float)(-(lr / bc1))};
}

__device__ __forceinline__ float adam_update(float p, float g, float& m, float& v, const AdamStep& a) {
    m = m + a.w1 * (g - m);                 // exp_avg.lerp_(grad, 1 - beta1)
    v = v * a.b2 + (a.w2 * g) * g;          // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2)
    const float denom = sqrtf(v) / a.bc2s + a.eps;
    return p + (a.neg_step * m) / denom;    // param.addcdiv_(exp_avg, denom, value=-step_size)
}

// ---- W2 mirror -------------------------------------------------------------------------------
// One 32 x 32 tile (rows k0.., columns o0..) of an [H][H] W2 block, 256 threads: thread (ly, lx)
// visits w2t[k0 + ly + 8q][o0 + lx] for q < 4, `upd(k, o)` returns the element's new value (and
// stores it wherever the caller keeps w2t), and the tile goes through shared memory so that the
// out-major mirror w2n[o][k] is written coalesced as well.
template <class Upd>
__device__ __forceinline__ void w2_tile(float* w2n, int H, int k0, int o0, Upd&& upd) {
    __shared__ float tile[32][33];
    const int lx = threadIdx.x % 32, ly = threadIdx.x / 32;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int kk = ly + 8 * q;
        tile[kk][lx] = upd(k0 + kk, o0 + lx);
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int oo = ly + 8 * q;
        w2n[(size_t)(o0 + oo) * H + k0 + lx] = tile[lx][oo];
    }
}

// w2n[n] = w2t[n]^T for the networks n = blockIdx.y of one launch (grid (H/32)^2 x n_nets, 256 threads)
constexpr int W2_MIRROR_MAX_NETS = 8;
struct W2Mirror {
    const float* w2t[W2_MIRROR_MAX_NETS];
    float* w2n[W2_MIRROR_MAX_NETS];
};
int launch_w2_mirror(const W2Mirror& mr, int n_nets, int H, cudaStream_t s);

}  // namespace fsrl
