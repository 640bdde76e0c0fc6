// Batched MLP forward over N rows (optionally gathered by index): the critic passes of
// compute_gae_returns (/root/reference/fsrl/policy/base_policy.py:416-422) and any other
// "no_grad forward over the whole buffer" of the reference (ppo_lag.py:144-149, cpo.py:135-141).
//
// H = 128 / 256 run mlp_forward_rows_kernel: a persistent grid (as many CTAs as fit on the device)
// walks tiles of FWD_ROWS = 64 rows.  Every CTA streams W1t/W2t from L2 once per tile, so 64 rows
// instead of MlpTile<H>::R = 32 / 16 share one pass over the weights (4x less L2 -> SM weight traffic
// at H = 256), and every warp issues FWD_ROWS/16 m-tiles of
// MMAs per pipeline stage instead of one.  Each output element is computed by the same operation
// sequence as in mlp_forward_kernel (bias-initialised 3xTF32 accumulators, ascending k; the head in
// MlpTile<H>::PARTS lanes per row), so both kernels give the same bits.  H = 64 already has 64-row
// tiles, and H = 512 does not fit 64 rows in shared memory: both keep mlp_forward_kernel, as does an
// input too wide for a 64-row tile.
// FSRL_MLPFWD_TILED=1 forces mlp_forward_kernel at every width (A/B runs and the bit-identity tests).
#include "mlp.cuh"
#include "fsrl_b200.h"
#include <cstdlib>

namespace fsrl {

template <int H>
__global__ void __launch_bounds__(MLP_TPB)
mlp_forward_kernel(const Mlp3 m, const float* __restrict__ x, const int* __restrict__ idx,
                   long long n_rows, float* __restrict__ y) {
    using TT = MlpTile<H>;
    extern __shared__ __align__(16) float smem[];
    const int tid = threadIdx.x;
    const MlpSmem<H> sm(smem, m.in, m.out);
    const long long r0 = (long long)blockIdx.x * TT::R;
    mlp_stage_rows<H>(sm, m.in, [&](int r) -> const float* {
        const long long row = r0 + r;
        if (row >= n_rows) return nullptr;
        const long long src = idx ? (long long)idx[row] : row;
        return x + src * m.in;
    });
    __syncthreads();
    mlp_hidden_forward<H>(m, sm);
    float out[MLP_MAX_OUT];
    mlp_head_forward<H>(m, sm, out);
    const int r = tid / TT::PARTS, part = tid % TT::PARTS;
    const long long row = r0 + r;
    if (part == 0 && row < n_rows) {
#pragma unroll
        for (int j = 0; j < MLP_MAX_OUT; ++j)
            if (j < m.out) y[row * m.out + j] = out[j];
    }
}

constexpr int FWD_ROWS = 64;

// x[FWD_ROWS][in_pad] | h[FWD_ROWS][LDA] (h1, then h2 in place) | wstage | w3s[H][out]
template <int H>
__host__ __device__ constexpr size_t fwd_rows_smem_bytes(int in, int out) {
    using TT = MlpTile<H>;
    return sizeof(float) * ((size_t)FWD_ROWS * TT::in_pad(in) + (size_t)FWD_ROWS * TT::LDA + TT::stage_floats() +
                            (size_t)H * out);
}

template <int H>
__global__ void __launch_bounds__(MLP_TPB)
mlp_forward_rows_kernel(const Mlp3 m, const float* __restrict__ x, const int* __restrict__ idx,
                        long long n_rows, float* __restrict__ y) {
    using TT = MlpTile<H>;
    constexpr int MT = FWD_ROWS / 16;
    static_assert(FWD_ROWS % TT::R == 0, "the head runs in passes of MlpTile<H>::R rows");
    extern __shared__ __align__(16) float smem[];
    const int tid = threadIdx.x;
    const int inp = TT::in_pad(m.in);
    float* xs = smem;
    float* hs = xs + (size_t)FWD_ROWS * inp;
    float* wst = hs + (size_t)FWD_ROWS * TT::LDA;
    float* w3s = wst + TT::stage_floats();
    for (int i = tid; i < H * m.out; i += MLP_TPB) w3s[i] = __ldg(m.w3t + i);
    const long long n_tiles = (n_rows + FWD_ROWS - 1) / FWD_ROWS;
    for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const long long r0 = tile * FWD_ROWS;
        // the previous tile last read xs in its layer-1 GEMM and hs before the barrier of this tile's
        // first GEMM stage, so both may be rewritten here
        for (int i = tid; i < FWD_ROWS * inp; i += MLP_TPB) {
            const int r = i / inp, k = i % inp;
            const long long row = r0 + r;
            float v = 0.f;
            if (row < n_rows && k < m.in) v = x[(idx ? (long long)idx[row] : row) * m.in + k];
            xs[i] = v;
        }
        float c[MT][TT::NT][4];
        tc_init_bias<H, MT>(c, m.b1);
        tc_gemm<H, MT>(c, xs, inp, m.in, m.w1t, wst, false);
        stage_load<H>(m.w2t, H, wst, 0, 0);            // prefetch W2t stage 0 under the epilogue
        tc_foreach<H, MT>(c, [&](int row, int col, float v0, float v1) {
            *reinterpret_cast<float2*>(hs + (size_t)row * TT::LDA + col) = make_float2(fmaxf(v0, 0.f), fmaxf(v1, 0.f));
        });
        tc_init_bias<H, MT>(c, m.b2);
        tc_gemm<H, MT>(c, hs, TT::LDA, H, m.w2t, wst, true);
        // tc_gemm ends on a barrier after its last read of h1: h2 overwrites it in place
        tc_foreach<H, MT>(c, [&](int row, int col, float v0, float v1) {
            *reinterpret_cast<float2*>(hs + (size_t)row * TT::LDA + col) = make_float2(fmaxf(v0, 0.f), fmaxf(v1, 0.f));
        });
        __syncthreads();
        const int r = tid / TT::PARTS, part = tid % TT::PARTS;
#pragma unroll 1
        for (int p = 0; p < FWD_ROWS / TT::R; ++p) {
            float out[MLP_MAX_OUT];
            mlp_head_forward<H>(m, hs + (size_t)p * TT::R * TT::LDA, w3s, out);
            const long long row = r0 + p * TT::R + r;
            if (part == 0 && row < n_rows) {
#pragma unroll
                for (int j = 0; j < MLP_MAX_OUT; ++j)
                    if (j < m.out) y[row * m.out + j] = out[j];
            }
        }
    }
}

// grid of the persistent launch for the tile's shared-memory size (cached per device: it depends on H, in and
// out only);
// 0 when 64 rows do not fit in one CTA's shared memory (input widths far above those of any network here):
// the caller then takes mlp_forward_kernel
template <int H>
static int rows_grid(size_t smem, long long n_tiles, long long* grid) {
    static size_t cached_smem[64] = {0};      // per device: the attribute is set on the current one
    static int cached_per_sm[64] = {0};
    int dev = 0;
    FSRL_CUDA(cudaGetDevice(&dev));
    FSRL_REQUIRE(dev >= 0 && dev < 64, "fsrl_mlp_forward: device %d", dev);
    if (smem != cached_smem[dev]) {
        int optin = 0, per_sm = 0;
        FSRL_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
        if (smem <= (size_t)optin) {
            FSRL_CUDA(cudaFuncSetAttribute(mlp_forward_rows_kernel<H>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            FSRL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, mlp_forward_rows_kernel<H>, MLP_TPB, smem));
        }
        cached_per_sm[dev] = per_sm;
        cached_smem[dev] = smem;
    }
    const long long cap = (long long)sm_count() * cached_per_sm[dev];
    *grid = n_tiles < cap ? n_tiles : cap;
    return FSRL_OK;
}

template <int H>
static int launch_forward_rows(const Mlp3& m, const float* x, const int* idx, long long n_rows, float* y,
                               cudaStream_t s, bool* launched) {
    const size_t smem = fwd_rows_smem_bytes<H>(m.in, m.out);
    long long grid = 0;
    const int rc = rows_grid<H>(smem, (n_rows + FWD_ROWS - 1) / FWD_ROWS, &grid);
    if (rc) return rc;
    *launched = grid > 0;
    if (*launched) mlp_forward_rows_kernel<H><<<(unsigned)grid, MLP_TPB, smem, s>>>(m, x, idx, n_rows, y);
    return FSRL_OK;
}

}  // namespace fsrl

using namespace fsrl;

extern "C" int fsrl_mlp_forward(const fsrl_mlp3_t* net, const float* x, const int* idx,
                                long long n_rows, float* y, void* stream) {
    FSRL_REQUIRE(n_rows >= 0, "fsrl_mlp_forward: n_rows < 0");
    if (n_rows == 0) return FSRL_OK;
    FSRL_REQUIRE(net && x && y, "fsrl_mlp_forward: null pointer");
    FSRL_REQUIRE(net->out >= 1 && net->out <= MLP_MAX_OUT, "fsrl_mlp_forward: out dim %d unsupported", net->out);
    if (n_rows == 0) return FSRL_OK;
    const Mlp3 m = *reinterpret_cast<const Mlp3*>(net);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const char* tiled = getenv("FSRL_MLPFWD_TILED");
    const bool rows = !(tiled && atoi(tiled) != 0);
#define GO(HH)                                                                                     \
    {                                                                                              \
        using TT = MlpTile<HH>;                                                                    \
        const size_t smem = TT::smem_bytes(m.in);                                                  \
        FSRL_CUDA(cudaFuncSetAttribute(mlp_forward_kernel<HH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        const long long grid = (n_rows + TT::R - 1) / TT::R;                                       \
        mlp_forward_kernel<HH><<<(unsigned)grid, MLP_TPB, smem, s>>>(m, x, idx, n_rows, y);        \
    }
    switch (m.H) {
        case 64: GO(64) break;
        case 128: {
            bool done = false;
            if (rows) { int rc = launch_forward_rows<128>(m, x, idx, n_rows, y, s, &done); if (rc) return rc; }
            if (!done) GO(128)
        } break;
        case 256: {
            bool done = false;
            if (rows) { int rc = launch_forward_rows<256>(m, x, idx, n_rows, y, s, &done); if (rc) return rc; }
            if (!done) GO(256)
        } break;
        case 512: GO(512) break;
        default: set_error("fsrl_mlp_forward: hidden width %d unsupported (64/128/256/512)", m.H); return FSRL_EINVAL;
    }
#undef GO
    FSRL_LAUNCH_CHECK();
    return FSRL_OK;
}
