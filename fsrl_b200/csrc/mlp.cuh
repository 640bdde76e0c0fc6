// Fused 2-hidden-layer MLP forward/backward building blocks for a tile of rows, shared by the
// rollout step, the critic evaluation before GAE, the PPO/CPO/SAC update kernels.
//
// Replaces the tianshou Net/MLP/ActorProb/Critic forward the reference calls at
// fsrl/policy/base_policy.py:178 (actor) and :421-422 (critics): h = ReLU(W2 ReLU(W1 x)).
//
// Canonical parameter layout (all kernels): every Linear is stored TRANSPOSED, Wt[in][out]
// row-major, so a k-row of the weight is contiguous (coalesced cp.async, conflict-free LDS).
// torch sees `.weight` as the strided view Wt.t().
//
// GEMMs run on the tensor cores with fp32-faithful "3xTF32" arithmetic: every fp32 operand is
// split into hi = tf32(x), lo = tf32(x - hi) and the product is accumulated as
// a_lo*b_hi + a_hi*b_lo + a_hi*b_hi in fp32 (mma.sync.m16n8k8.tf32), i.e. ~2^-21 relative
// error per product -- indistinguishable from an fp32 FMA chain at the parity tolerances.
// The row tiles here are 16..64 rows (a 256-row minibatch split over 16 CTAs), at or below the
// 64-row atom of a wgmma warpgroup, and the kernels are latency- not throughput-bound, so the
// warp-level mma path is the right tensor-core granularity for this workload.
//
// Thread mapping (256 threads = 8 warps): a CTA owns R rows (R = 4096/H, at least 16); warp w
// owns output columns [w*H/8, (w+1)*H/8) for all R rows: MT = R/16 m-tiles x NT = H/64
// n-tiles of m16n8 accumulators.  Weights stream through a cp.async double-buffered
// shared-memory stage of KC k-rows (row stride H+8 floats: conflict-free B fragments);
// activations stay in shared memory between layers (row stride H+4: conflict-free A
// fragments).
#pragma once
#include "arena.cuh"
#include <cuda_pipeline.h>

namespace fsrl {

constexpr int MLP_TPB = 256;
constexpr int MLP_KC = 16;          // k-rows of a weight matrix per pipeline stage
constexpr int MLP_NST = 4;          // pipeline stages in flight (L2 latency x bandwidth ~ 64 KB per SM)
constexpr int MLP_MAX_OUT = 16;

template <int H>
struct MlpTile {
    static_assert(H == 64 || H == 128 || H == 256 || H == 512, "hidden width must be 64/128/256/512");
    static constexpr int R = (4096 / H) < 16 ? 16 : (4096 / H);   // rows per CTA
    static constexpr int MT = R / 16;           // m-tiles per warp
    static constexpr int WN = H / 8;            // columns per warp
    static constexpr int NT = WN / 8;           // n-tiles per warp
    static constexpr int LDA = H + 4;           // activation row stride (floats)
    static constexpr int LDW = H + 8;           // staged weight row stride (floats)
    static constexpr int PARTS = MLP_TPB / R;   // lanes cooperating on one row in the head
    static constexpr int NST = (H >= 512) ? 2 : MLP_NST;   // weight pipeline depth (smem budget)
    __host__ __device__ static constexpr int in_pad(int in) { return ((in + 7) & ~7) + 4; }
    __host__ __device__ static constexpr int stage_floats() { return NST * MLP_KC * LDW; }
    // x[R][in_pad] | h1[R][LDA] | h2[R][LDA] | wstage[2][KC][LDW] | w3s[H][out]
    __host__ __device__ static constexpr size_t smem_floats(int in, int out) {
        return (size_t)R * in_pad(in) + 2 * (size_t)R * LDA + stage_floats() + (size_t)H * out;
    }
    __host__ __device__ static constexpr size_t smem_bytes(int in, int out = MLP_MAX_OUT) {
        return sizeof(float) * smem_floats(in, out);
    }
};

// x = hi + lo with hi, lo representable in TF32 (10 explicit mantissa bits).  Round-to-nearest,
// ties away from zero -- the result of cvt.rna.tf32.f32 -- done with integer ops: the cvt runs on
// the quarter-rate conversion pipe, which would otherwise bound every split-operand GEMM here.
__device__ __forceinline__ uint32_t round_tf32(float x) { return (__float_as_uint(x) + 0x1000u) & 0xffffe000u; }
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
    hi = round_tf32(x);
    lo = round_tf32(x - __uint_as_float(hi));
}

__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm(
        "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// cp.async rows [chunk*KC, chunk*KC+KC) of a row-major [K][H] matrix into stage buffer `buf`;
// rows >= K are zero-filled (layer 1 pads K up to a multiple of 8)
template <int H>
__device__ __forceinline__ void stage_load(const float* mat, int K, float* wst, int chunk, int buf) {
    using TT = MlpTile<H>;
    float* dst = wst + (size_t)buf * MLP_KC * TT::LDW;
    constexpr int SEG = H / 4;                      // 16-byte segments per row
    for (int i = threadIdx.x; i < MLP_KC * SEG; i += MLP_TPB) {
        const int rr = i / SEG, sg = i % SEG;
        const int k = chunk * MLP_KC + rr;
        float* d = dst + (size_t)rr * TT::LDW + 4 * sg;
        if (k < K) __pipeline_memcpy_async(d, mat + (size_t)k * H + 4 * sg, 16);
        else *reinterpret_cast<float4*>(d) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __pipeline_commit();
}

// c[mt][nt] += A[16mt.., k] * W[k][warp cols] for k in [0, Kp): A is a shared-memory tile
// (row stride lda, Kp a multiple of 8), W a row-major [K][H] global matrix streamed through
// `wst`.  All threads must call; contains __syncthreads (the first one also orders the
// caller's earlier shared-memory stores to A).
template <int H, int MT = MlpTile<H>::MT>
__device__ __forceinline__ void tc_gemm(float (&c)[MT][MlpTile<H>::NT][4], const float* A,
                                        int lda, int K, const float* W, float* wst,
                                        bool stage0_in_flight) {
    using TT = MlpTile<H>;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int n0 = warp * TT::WN;
    const int Kp = (K + 7) & ~7;
    const int nch = (Kp + MLP_KC - 1) / MLP_KC;
    // prologue: stages 0 .. NST-2 in flight (one commit group per stage, empty groups keep the
    // wait_prior arithmetic uniform)
    for (int p = stage0_in_flight ? 1 : 0; p < TT::NST - 1; ++p) {
        if (p < nch) stage_load<H>(W, K, wst, p, p);
        else __pipeline_commit();
    }
    for (int ch = 0; ch < nch; ++ch) {
        if (ch + TT::NST - 1 < nch) stage_load<H>(W, K, wst, ch + TT::NST - 1, (ch + TT::NST - 1) % TT::NST);
        else __pipeline_commit();
        __pipeline_wait_prior(TT::NST - 1);
        __syncthreads();
        const float* w = wst + (size_t)(ch % TT::NST) * MLP_KC * TT::LDW;
        const int kleft = Kp - ch * MLP_KC;
#pragma unroll
        for (int ks = 0; ks < MLP_KC; ks += 8) {
            if (ks < kleft) {
                const int k0 = ch * MLP_KC + ks;
                uint32_t bh[TT::NT][2], bl[TT::NT][2];
#pragma unroll
                for (int nt = 0; nt < TT::NT; ++nt) {
                    split_tf32(w[(size_t)(ks + t) * TT::LDW + n0 + 8 * nt + g], bh[nt][0], bl[nt][0]);
                    split_tf32(w[(size_t)(ks + t + 4) * TT::LDW + n0 + 8 * nt + g], bh[nt][1], bl[nt][1]);
                }
#pragma unroll
                for (int mt = 0; mt < MT; ++mt) {
                    uint32_t ah[4], al[4];
                    const float* a = A + (size_t)(16 * mt + g) * lda + k0 + t;
                    split_tf32(a[0], ah[0], al[0]);
                    split_tf32(a[(size_t)8 * lda], ah[1], al[1]);
                    split_tf32(a[4], ah[2], al[2]);
                    split_tf32(a[(size_t)8 * lda + 4], ah[3], al[3]);
#pragma unroll
                    for (int nt = 0; nt < TT::NT; ++nt) mma_tf32(c[mt][nt], al, bh[nt]);   // small terms first; the three
#pragma unroll
                    for (int nt = 0; nt < TT::NT; ++nt) mma_tf32(c[mt][nt], ah, bl[nt]);   // passes keep dependent MMAs
#pragma unroll
                    for (int nt = 0; nt < TT::NT; ++nt) mma_tf32(c[mt][nt], ah, bh[nt]);   // TT::NT instructions apart
                }
            }
        }
        __syncthreads();   // everyone done with stage ch before it is overwritten
    }
}

// visit every accumulator pair of this thread: f(row, col, v0, v1) with (row, col), (row, col+1)
template <int H, int MT = MlpTile<H>::MT, class F>
__device__ __forceinline__ void tc_foreach(float (&c)[MT][MlpTile<H>::NT][4], F f) {
    using TT = MlpTile<H>;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int nt = 0; nt < TT::NT; ++nt) {
            const int col = warp * TT::WN + 8 * nt + 2 * t;
            f(16 * mt + g, col, c[mt][nt][0], c[mt][nt][1]);
            f(16 * mt + g + 8, col, c[mt][nt][2], c[mt][nt][3]);
        }
}

template <int H, int MT = MlpTile<H>::MT>
__device__ __forceinline__ void tc_init_bias(float (&c)[MT][MlpTile<H>::NT][4], const float* bias) {
    using TT = MlpTile<H>;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int t = lane & 3;
#pragma unroll
    for (int nt = 0; nt < TT::NT; ++nt) {
        const int col = warp * TT::WN + 8 * nt + 2 * t;
        const float b0 = bias ? __ldg(bias + col) : 0.f, b1 = bias ? __ldg(bias + col + 1) : 0.f;
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) { c[mt][nt][0] = b0; c[mt][nt][1] = b1; c[mt][nt][2] = b0; c[mt][nt][3] = b1; }
    }
}


// -------------------------------------------------------------------------------------------------
// Column-slab GEMM: a CTA computes only NS of the H output columns (the minibatch kernels split
// every layer's N dimension over H/NS CTAs to put 4x more SMs on the same tiny problem).  The
// K range is split across the 8 warps (each warp owns all NS columns of its K/8 slice, so no
// operand is loaded twice), partial tiles are summed through shared memory.
// -------------------------------------------------------------------------------------------------
constexpr int SLAB_NS = 64;
constexpr int SLAB_LDB = SLAB_NS + 8;      // conflict-free B fragments
constexpr int SLAB_LDR = SLAB_NS + 4;

template <int H>
__host__ __device__ constexpr size_t slab_b_floats() { return (size_t)H * SLAB_LDB; }
template <int H>
__host__ __device__ constexpr size_t slab_red_floats() { return (size_t)8 * MlpTile<H>::R * SLAB_LDR; }
// one buffer serves as B slab and (afterwards) as the cross-warp reduce buffer
template <int H>
__host__ __device__ constexpr size_t slab_buf_floats() {
    return slab_b_floats<H>() > slab_red_floats<H>() ? slab_b_floats<H>() : slab_red_floats<H>();
}

// whole [H][NS] slab of a row-major matrix (row stride gld, first column c0) -> bs via cp.async
template <int H>
__device__ __forceinline__ void slab_load(const float* W, int gld, int c0, float* bs) {
    constexpr int SEG = SLAB_NS / 4;
    for (int i = threadIdx.x; i < H * SEG; i += MLP_TPB) {
        const int k = i / SEG, sg = i % SEG;
        __pipeline_memcpy_async(bs + (size_t)k * SLAB_LDB + 4 * sg, W + (size_t)k * gld + c0 + 4 * sg, 16);
    }
    __pipeline_commit();
}

// out[row][col] = sum_k A[row][k] * bs[k][col]; epi(row, col4, float4) is called once per 4 outputs.
// `red` may alias `bs` (a barrier separates the last read of bs from the first write of red).
template <int H, class F>
__device__ __forceinline__ void slab_gemm(const float* A, int lda, const float* bs, float* red, F epi) {
    using TT = MlpTile<H>;
    constexpr int NTS = SLAB_NS / 8;
    constexpr int KW = H / 8;                      // k range per warp
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = lane >> 2, t = lane & 3;
    float c[TT::MT][NTS][4];
#pragma unroll
    for (int mt = 0; mt < TT::MT; ++mt)
#pragma unroll
        for (int nt = 0; nt < NTS; ++nt) { c[mt][nt][0] = c[mt][nt][1] = c[mt][nt][2] = c[mt][nt][3] = 0.f; }
#pragma unroll
    for (int ks = 0; ks < KW; ks += 8) {
        const int k0 = warp * KW + ks;
        uint32_t bh[NTS][2], bl[NTS][2];
#pragma unroll
        for (int nt = 0; nt < NTS; ++nt) {
            split_tf32(bs[(size_t)(k0 + t) * SLAB_LDB + 8 * nt + g], bh[nt][0], bl[nt][0]);
            split_tf32(bs[(size_t)(k0 + t + 4) * SLAB_LDB + 8 * nt + g], bh[nt][1], bl[nt][1]);
        }
#pragma unroll
        for (int mt = 0; mt < TT::MT; ++mt) {
            uint32_t ah[4], al[4];
            const float* a = A + (size_t)(16 * mt + g) * lda + k0 + t;
            split_tf32(a[0], ah[0], al[0]);
            split_tf32(a[(size_t)8 * lda], ah[1], al[1]);
            split_tf32(a[4], ah[2], al[2]);
            split_tf32(a[(size_t)8 * lda + 4], ah[3], al[3]);
#pragma unroll
            for (int nt = 0; nt < NTS; ++nt) mma_tf32(c[mt][nt], al, bh[nt]);   // small terms first; the three
#pragma unroll
            for (int nt = 0; nt < NTS; ++nt) mma_tf32(c[mt][nt], ah, bl[nt]);   // passes keep dependent MMAs
#pragma unroll
            for (int nt = 0; nt < NTS; ++nt) mma_tf32(c[mt][nt], ah, bh[nt]);   // NTS instructions apart
        }
    }
    __pipeline_wait_prior(0);                      // callers may have async copies for the epilogue in flight
    __syncthreads();                               // all warps done reading bs (red may alias it)
    float* mine = red + (size_t)warp * TT::R * SLAB_LDR;
#pragma unroll
    for (int mt = 0; mt < TT::MT; ++mt)
#pragma unroll
        for (int nt = 0; nt < NTS; ++nt) {
            *reinterpret_cast<float2*>(mine + (size_t)(16 * mt + g) * SLAB_LDR + 8 * nt + 2 * t) = make_float2(c[mt][nt][0], c[mt][nt][1]);
            *reinterpret_cast<float2*>(mine + (size_t)(16 * mt + g + 8) * SLAB_LDR + 8 * nt + 2 * t) = make_float2(c[mt][nt][2], c[mt][nt][3]);
        }
    __syncthreads();
    for (int e = threadIdx.x; e < TT::R * (SLAB_NS / 4); e += MLP_TPB) {
        const int row = e / (SLAB_NS / 4), c4 = (e % (SLAB_NS / 4)) * 4;
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int w = 0; w < 8; ++w) {
            const float4 v = *reinterpret_cast<const float4*>(red + ((size_t)w * TT::R + row) * SLAB_LDR + c4);
            s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
        }
        epi(row, c4, s);
    }
}

// c += A[.., k] * W[k][warp cols] with B fragments read straight from global (small K: layer 1)
template <int H>
__device__ __forceinline__ void tc_gemm_direct(float (&c)[MlpTile<H>::MT][MlpTile<H>::NT][4], const float* A,
                                               int lda, int K, const float* W) {
    using TT = MlpTile<H>;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int n0 = warp * TT::WN;
    const int Kp = (K + 7) & ~7;
    for (int k0 = 0; k0 < Kp; k0 += 8) {
        uint32_t bh[TT::NT][2], bl[TT::NT][2];
#pragma unroll
        for (int nt = 0; nt < TT::NT; ++nt) {
            const float w0 = (k0 + t < K) ? __ldg(W + (size_t)(k0 + t) * H + n0 + 8 * nt + g) : 0.f;
            const float w1 = (k0 + t + 4 < K) ? __ldg(W + (size_t)(k0 + t + 4) * H + n0 + 8 * nt + g) : 0.f;
            split_tf32(w0, bh[nt][0], bl[nt][0]);
            split_tf32(w1, bh[nt][1], bl[nt][1]);
        }
#pragma unroll
        for (int mt = 0; mt < TT::MT; ++mt) {
            uint32_t ah[4], al[4];
            const float* a = A + (size_t)(16 * mt + g) * lda + k0 + t;
            split_tf32(a[0], ah[0], al[0]);
            split_tf32(a[(size_t)8 * lda], ah[1], al[1]);
            split_tf32(a[4], ah[2], al[2]);
            split_tf32(a[(size_t)8 * lda + 4], ah[3], al[3]);
#pragma unroll
            for (int nt = 0; nt < TT::NT; ++nt) mma_tf32(c[mt][nt], al, bh[nt]);   // small terms first; the three
#pragma unroll
            for (int nt = 0; nt < TT::NT; ++nt) mma_tf32(c[mt][nt], ah, bl[nt]);   // passes keep dependent MMAs
#pragma unroll
            for (int nt = 0; nt < TT::NT; ++nt) mma_tf32(c[mt][nt], ah, bh[nt]);   // TT::NT instructions apart
        }
    }
}

// Shared-memory carve-up used by every kernel built on these blocks
template <int H>
struct MlpSmem {
    float *x, *h1, *h2, *wst, *w3s;
    __device__ MlpSmem(float* base, int in, int out) {
        using TT = MlpTile<H>;
        x = base;
        h1 = x + (size_t)TT::R * TT::in_pad(in);
        h2 = h1 + (size_t)TT::R * TT::LDA;
        wst = h2 + (size_t)TT::R * TT::LDA;
        w3s = wst + TT::stage_floats();
        (void)out;
    }
    __device__ float* end(int out) const { return w3s + (size_t)H * out; }
};

// Computes h1 = ReLU(W1 x + b1), h2 = ReLU(W2 h1 + b2) for the R rows staged in s.x (row
// stride in_pad, columns >= in zero).  Also stages W3t into s.w3s.  On return h1/h2 (row
// stride LDA) are valid in shared memory for all threads.
template <int H>
__device__ __forceinline__ void mlp_hidden_forward(const Mlp3& m, const MlpSmem<H>& s) {
    using TT = MlpTile<H>;
    const int inp = TT::in_pad(m.in);
    // head weights -> smem (tiny), then stage 0 of W1t; both overlap with nothing yet, but keep
    // the head copy out of the GEMM pipelines' group accounting by finishing it first
    for (int i = threadIdx.x; i < H * m.out; i += MLP_TPB) s.w3s[i] = __ldg(m.w3t + i);
    float c[TT::MT][TT::NT][4];
    tc_init_bias<H>(c, m.b1);
    tc_gemm<H>(c, s.x, inp, m.in, m.w1t, s.wst, false);
    stage_load<H>(m.w2t, H, s.wst, 0, 0);            // prefetch W2t stage 0 under the epilogue
    tc_foreach<H>(c, [&](int row, int col, float v0, float v1) {
        *reinterpret_cast<float2*>(s.h1 + (size_t)row * TT::LDA + col) = make_float2(fmaxf(v0, 0.f), fmaxf(v1, 0.f));
    });
    tc_init_bias<H>(c, m.b2);
    tc_gemm<H>(c, s.h1, TT::LDA, H, m.w2t, s.wst, true);
    tc_foreach<H>(c, [&](int row, int col, float v0, float v1) {
        *reinterpret_cast<float2*>(s.h2 + (size_t)row * TT::LDA + col) = make_float2(fmaxf(v0, 0.f), fmaxf(v1, 0.f));
    });
    __syncthreads();
}

// Layer 3 (H -> out <= 16): PARTS lanes cooperate on each row, shuffle-reduce; on return the
// lane with part == 0 of row r (thread r*PARTS) holds out[0..out) for that row.
// h2: the R rows of this pass (row stride LDA); w3s: W3t staged in shared memory.
template <int H>
__device__ __forceinline__ void mlp_head_forward(const Mlp3& m, const float* h2, const float* w3s, float* out) {
    using TT = MlpTile<H>;
    const int tid = threadIdx.x;
    const int r = tid / TT::PARTS, part = tid % TT::PARTS;
    const int no = m.out;
#pragma unroll
    for (int j = 0; j < MLP_MAX_OUT; ++j) out[j] = 0.f;
    for (int k = part; k < H; k += TT::PARTS) {
        const float x = h2[(size_t)r * TT::LDA + k];
        const float* w = w3s + (size_t)k * no;
#pragma unroll
        for (int j = 0; j < MLP_MAX_OUT; ++j)
            if (j < no) out[j] = fmaf(x, w[j], out[j]);
    }
#pragma unroll
    for (int j = 0; j < MLP_MAX_OUT; ++j) {
        if (j < no) {
            float v = out[j];
#pragma unroll
            for (int o = TT::PARTS / 2; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o, TT::PARTS);
            out[j] = v + __ldg(m.b3 + j);
        }
    }
}

template <int H>
__device__ __forceinline__ void mlp_head_forward(const Mlp3& m, const MlpSmem<H>& s, float* out) {
    mlp_head_forward<H>(m, s.h2, s.w3s, out);
}

// stage R rows of x (optionally gathered) into s.x, zero-padding columns >= in
template <int H, class RowPtr>
__device__ __forceinline__ void mlp_stage_rows(const MlpSmem<H>& s, int in, RowPtr row_ptr) {
    using TT = MlpTile<H>;
    const int inp = TT::in_pad(in);
    for (int i = threadIdx.x; i < TT::R * inp; i += MLP_TPB) {
        const int r = i / inp, k = i % inp;
        const float* p = row_ptr(r);
        s.x[i] = (p != nullptr && k < in) ? p[k] : 0.f;
    }
}

}  // namespace fsrl
