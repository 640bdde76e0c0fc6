// Persistent PPO-Lagrangian update: ONE launch per repeat runs every minibatch step of the reference's
// fsrl/policy/ppo_lag.py:223-247 (forward, clipped-surrogate + lambda * cost-advantage loss and value losses
// :152-212, lagrangian_base.py:145-166, backward, clip_grad_norm_, Adam) on a co-resident grid of 32 CTAs per
// network.  Hopper data path: the three 256^3 GEMMs of a network and step run on the warpgroup tensor cores
// (wgmma kind tf32, fp32-faithful 3-term split, accumulators in registers), operands arrive as bulk asynchronous
// copies (TMA unit) of pre-split "plane layout" images that the producing CTAs write straight from their epilogues,
// and the CTAs of a step are chained by device-scope release/acquire counters instead of kernel launches.
//
// Work decomposition of one network (H = 256, minibatch = 256 rows = 4 row blocks of 64):
//   CTA c = 8 a + b           a = row block (4), b = 32-wide column block (8)
//   S   h1 tile   [64 r x 32 k]   FFMA (K = D) over observation rows staged one step ahead
//                                                         -> images H1A (MN = r, K = k), H1T (MN = k, K = r)
//   G1  h2 tile   [64 r x 32 o] = h1[r, :] W2t[:, o]      A = H1A block a, B = W2A block b      (wgmma)
//       head partial over the tile's 32 columns -> 8 partials per row block -> loss gradient dOut
//       dz2 tile = (dOut W3^T) * relu'(h2)                -> images DZA (MN = r, K = o), DZT (MN = o, K = r)
//   G2  (CTAs 0-15: ka = c / 4, rb = c % 4)  dh1^T tile [64 k x 64 r] = W2t[k, :] dz2[r, :]^T
//       A = W2B block ka, B = DZA block rb;  * relu'(h1) -> partial dW1 / db1 over the 64 rows
//   G3  (CTAs 16-31: ka, ob = c % 4)         dW2^T tile [64 o x 64 k] = dz2[:, o]^T h1[:, k]
//       A = DZT block ob, B = H1T block ka;  the CTA owns this tile of W2: its Adam state (p, m, v) lives in the
//       epilogue threads' registers for the whole launch, the updated tile is re-published as images W2A / W2B
//   small parameters (W1, b1, b2, W3, b3, log sigma): every CTA keeps the slices it consumes (+ their
//       Adam moments) in shared memory and applies the identical update to them (deterministic
//       replicas).  Column block b's gradient slice is reduced once, by its REDUCER CTA (a = b >> 2, b): fixed-order
//       sums of the b2 / W3 / b3 row-block partials (L2, by warpgroup 1 during G2) and of the 8 dW1 / db1 partials that
//       the G2 CTAs of k block b >> 1 -- same cluster -- keep in their operand rings (read over DSMEM).
//   global-norm clip: sums of squares of the reducers' slices and the G3 tiles -> one device-wide counter hop (D2)
//       -> every CTA adds the 96 slots in the same order and reads its column block's final slice.
// All operand images are K-major no-swizzle plane images (wgmma.cuh); transposed copies are written by the producer
// (wgmma reads tf32 operands K-major only).
//
// CTA = 288 threads: warps 0-7 (two warpgroups) issue the MMAs and run the epilogue, warp 8 is the bulk-copy producer.
// Warp w holds rows 16 (w % 4) .. + 15 of a 64-row tile.  Warpgroup 0 issues every GEMM alone with full-width
// m64n32k8 / m64n64k8 MMAs (each reads the A tile once for all columns), and warps w and w + 4 exchange the finished
// rows through shared memory behind one 64-thread barrier per warp pair (stage_acc).
// The 8 CTAs of a row block form a thread-block cluster: operand chunks that several of them need are multicast
// from L2 once into all of them (copy_operand), their head partials travel over distributed shared memory
// (st.async + mbarrier complete_tx), and so do the dW1 / db1 partials (remote mbarrier arrival, ld.shared::cluster);
// all other hops are flag lines in L2.  The grid is launched as clusters only: the
// gate (ppo_persist_supported) admits a shape only when all 4 x n_nets clusters can be co-resident, and everything it
// rejects runs on the three-launch chain of ppo.cu.  The cross terms of the 3-term split
// accumulate in their own registers.  With world > 1 the <DP = true> instantiation exchanges gradients itself over peer
// memory (dp_* functions below: tagged + hashed 16-byte packets pushed into the peers' buffers).
#include "ppo_persist.cuh"
#include "arena.cuh"
#include "ppo_loss.cuh"
#include "wgmma.cuh"
#include <cuda_pipeline.h>
#include <cstdlib>
#include <cmath>
#include <vector>

namespace fsrl {
namespace pp {

using namespace wg;

constexpr int WQ = 2;                    // epilogue warpgroups = warps that share the rows of a 16-row slab
constexpr int NEPI = 128 * WQ;           // epilogue (and MMA) threads: warps 0 .. 4 WQ - 1
constexpr int TPB = NEPI + 32;           // + the bulk-copy producer warp
constexpr int C1 = 16 / WQ;              // columns a thread owns of a 32-column tile (G1: h2 / dz2)
constexpr int C2 = 32 / WQ;              // columns a thread owns of a 64-column tile (G2 / G3 and the W2 tile)
constexpr int RB = 64;                   // rows per row block
constexpr int MB = 256;                  // rows per minibatch
constexpr int KC = 32, NCH = 256 / KC;   // k per operand chunk, chunks per GEMM
constexpr int SLOT_BYTES = 32768, NSLOT = 4;   // chunk: A hi | A lo | B hi | B lo, 64 (G1: B 32) rows x KC each
constexpr int A_CHUNK = 64 * KC * 4;     // bytes of one 64-row operand chunk
constexpr int ACC_LD = 68;               // row stride (floats) of the staged accumulator tile [64][ACC_LD]
constexpr int OUTP = 8;                  // padded head width
constexpr int H_ = 256;
constexpr int IMG = 65536;               // floats per image (256 x 256)
enum { I_H1A_HI, I_H1A_LO, I_H1T_HI, I_H1T_LO, I_DZA_HI, I_DZA_LO, I_DZT_HI, I_DZT_LO, I_W2A_HI, I_W2A_LO, I_W2B_HI, I_W2B_LO, N_IMG };
// per-network partial buffers (floats)
constexpr int DB2P_OFF = N_IMG * IMG;                           // [4 a][H]
constexpr int DW3P_OFF = DB2P_OFF + 4 * H_;                     // [4 a][H][OUTP]
constexpr int DB3P_OFF = DW3P_OFF + 4 * H_ * OUTP;              // [4 a][16]
constexpr int MAXD = 40;
// byte offset in the operand ring of the h1 tiles' observation rows, staged one step ahead (stage_rows)
constexpr int XS_OFF = 2 * SLOT_BYTES;
static_assert(XS_OFF >= 2 * 32 * 65 * 2 * 4 && XS_OFF >= 2 * (MAXD + 1) * 64 * 4 &&
              XS_OFF + 128 * (MAXD + 1) * 4 <= NSLOT * SLOT_BYTES, "staged rows overlap the ring's scratch or dW1 partials");
constexpr int NSMAX = (MAXD + 1) * 32 + 32 + 32 * OUTP + 16;    // floats of the largest small-parameter slice (SliceMap)
constexpr int SLICE_OFF = DB3P_OFF + 4 * 16;                    // [8 b][NSMAX]: final gradient slices, written by the reducers
constexpr int NET_WS = SLICE_OFF + 8 * NSMAX;
constexpr int SUMSQ_FLOATS = 128;                               // global tail: per-CTA sums of squares
// flag lines (32 unsigned each): per net A, C; global D2
constexpr int FLAG_LINE = 32;
constexpr int F_A = 0, F_C = 1, F_PER_NET = 2;
// The two cross terms a_lo b_hi + a_hi b_lo accumulate in their OWN registers and meet the a_hi b_hi sum only in the
// epilogue: the cross terms are 2^-11 of the main ones, and a tensor-core accumulator add may drop low bits of a small
// addend.  Same MMA count, 8 more accumulator registers per instruction column.
// peer-mapped exchange buffer of one step parity (floats): one region per SOURCE rank [8] plus one for the W2 means
// (written by the packets' owners), each holding per net 16 gradient tiles and the locally reduced small-parameter
// slices of the 8 column blocks.  Ranks PUSH their pieces into
// every peer's buffer as 16-byte packets {3 floats, tag}: the tag (launch sequence number | step) travels with the data,
// so the receiver polls its own memory until every packet carries the tag -- one NVLink one-way latency per exchange,
// no system-scope fence (slow with posted peer writes outstanding), no flag round trip, no remote loads.
// The tag word is XORed with a hash of the three payload words: a 16-byte vector store does NOT become visible atomically
// to a concurrent 16-byte load on the receiving GPU (a torn packet would show the new tag next to a stale payload
// word, i.e. one diverging parameter update; tools/dp_identity_check.py), so the receiver accepts a packet only if tag AND payload agree and simply polls again otherwise.
constexpr int TILE_PK = (64 * 64 / NEPI + 2) / 3;                // packets per thread of a 64 x 64 tile (16 floats -> 6)
constexpr int TILE_FLOATS = TILE_PK * NEPI * 4;                  // [packet][thread][4]
constexpr int SLICE_PK = (NSMAX + 2) / 3;
constexpr int XG_PER_NET = 16 * TILE_FLOATS + 8 * SLICE_PK * 4;
constexpr int MAX_MB = 16384;                                    // minibatches per launch (Adam scalar table)
constexpr long long WAIT_CYCLES = 6000000000LL;                  // ~3 s: a lost partner must not hang the GPU

struct Args {
    fsrl_ppo_update_t u;     // batch pointers already gathered (contiguous rows, u.perm == nullptr)
    int n_mb, slot0;
    long long adam_t0;
    float* ws;
    unsigned* flags;
    int* err;
    const float* adam_tab;   // [n_mb][2]: 1 / sqrt(1 - beta2^t), -(lr / (1 - beta1^t)) of every step (host doubles -> f32)
    long long* dbg;          // optional [n_cta][DBG_N] clock stamps of step dbg_step
    int dbg_step;
    unsigned dp_seq;         // data-parallel runs: launch sequence number (same on every rank), upper half of the packet tags
    int dp_direct;           // W2 gradient tiles exchanged in one hop (2 ranks) instead of the two-hop owner scheme
};
// clock stamps per CTA: 0 .. 47 phase boundaries (tools/persist_check.py names them), then per chunk of each GEMM phase
// (g = 0: G1, 1: G2 / G3) DBG_CH + 3 NCH g + NCH e + j: e = 0 the producer's bar_empty wait returned, 1 its copies
// were issued, 2 warpgroup 0's bar_full wait returned.  The per-chunk stamps exist only in a build with
// -DFSRL_PPO_CHUNK_STAMPS: even untaken, their checks inside the chunk loops lengthen every step (~0.7 us on c2).
constexpr int DBG_CH = 48;
constexpr int DBG_N = DBG_CH + 2 * 3 * NCH;
#define STAMP(i) do { if (P.dbg && t == P.dbg_step) P.dbg[(size_t)blockIdx.x * DBG_N + (i)] = clock64(); } while (0)

struct AdamS { float w1, b2, w2, rbc2s, eps, neg_step; };
// torch.optim.Adam's single-tensor update.  The moments are the exact fp32 expressions; the parameter step
// p += step * m / (sqrt(v) / sqrt(bc2) + eps) uses the SFU reciprocal square root / reciprocal (about 2 ulp each,
// i.e. ~1e-10 absolute on a step of <= lr) instead of IEEE sqrt and division, whose slow-path calls serialise the
// 32 elements a lane owns.
__device__ __forceinline__ float adam_one(float p, float g, float& m, float& v, const AdamS& a) {
    m = m + a.w1 * (g - m);                 // exp_avg.lerp_(grad, 1 - beta1)
    v = v * a.b2 + (a.w2 * g) * g;          // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2)
    const float sq = v > 0.f ? v * rsqrtf(v) : 0.f;
    const float denom = fmaf(sq, a.rbc2s, a.eps);
    return p + __fdividef(a.neg_step * m, denom);
}

__device__ __forceinline__ void fail(int* err, int code) {
    *reinterpret_cast<volatile int*>(err) = code;
    __threadfence_system();
    asm volatile("trap;");
}
// one 16-byte packet {x, y, z, tag ^ hash(x, y, z)}: a single vector store into peer memory / a single vector load from
// local memory.  The fourth word vouches for the other three: a packet is accepted only if it carries the expected tag
// AND its payload hashes to what the sender hashed, so a reader can never combine a fresh tag with stale payload words
// (whatever the granularity at which the fabric / L2 make a 16-byte write visible).
__device__ __forceinline__ uint32_t pk_hash(float x, float y, float z) {
    const uint32_t a = __float_as_uint(x), b = __float_as_uint(y), c = __float_as_uint(z);
    return a ^ __funnelshift_l(b, b, 11) ^ __funnelshift_l(c, c, 22);
}
__device__ __forceinline__ bool pk_ok(const float4& v, uint32_t tag) { return (__float_as_uint(v.w) ^ pk_hash(v.x, v.y, v.z)) == tag; }
__device__ __forceinline__ void st_packet(float* p, float x, float y, float z, uint32_t tag) {
    asm volatile("st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(x), "f"(y), "f"(z), "f"(__uint_as_float(tag ^ pk_hash(x, y, z))) : "memory");
}
__device__ __forceinline__ float4 ld_packet(const float* p) {
    float4 v;
    asm volatile("ld.relaxed.sys.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
    return v;
}

// Wait for the packets of all ranks but `me` at src + r * stride (local memory, pushed by the peers) and add them to the
// own piece (ox, oy, oz) in rank order.  Deliberately not inlined: the exchange code runs once per step and the kernel's
// instruction footprint matters (unrolled into the epilogue, the exchange slows the whole step down).
__device__ __noinline__ float3 dp_gather(const float* src, long long stride, int me, int world, uint32_t tag,
                                        float ox, float oy, float oz, int* err, int code) {
    const long long t0w = clock64();
    float ax = 0.f, ay = 0.f, az = 0.f;
    for (int r0 = 0; r0 < world; r0 += 4) {                // four ranks' packets in flight, rank order kept
        float4 v[4];
        bool ok;
        do {
            ok = true;
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if (r0 + k < world && r0 + k != me) v[k] = ld_packet(src + (size_t)(r0 + k) * stride);
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if (r0 + k < world && r0 + k != me) ok = ok && pk_ok(v[k], tag);
            if (!ok && clock64() - t0w > 4 * WAIT_CYCLES) fail(err, code);
        } while (!ok);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (r0 + k >= world) continue;
            if (r0 + k == me) { ax += ox; ay += oy; az += oz; }
            else { ax += v[k].x; ay += v[k].y; az += v[k].z; }
        }
    }
    return make_float3(ax, ay, az);
}
// one packet to every rank but `me`: dst_r = xg[r] + off
__device__ __noinline__ void dp_push_all(const float* const* xg, size_t off, int me, int world, float x, float y, float z, uint32_t tag) {
    for (int r = 0; r < world; ++r)
        if (r != me) st_packet(const_cast<float*>(xg[r]) + off, x, y, z, tag);
}

// ---- thread-block cluster: distributed shared memory pushes + remote mbarrier arrivals (hop B) ------------------------
__device__ __forceinline__ uint32_t mapa_u32(uint32_t local_saddr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_saddr), "r"(rank));
    return r;
}
__device__ __forceinline__ void st_cluster4(uint32_t raddr, float4 v) {
    asm volatile("st.shared::cluster.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(raddr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
// asynchronous remote store that completes 16 transaction bytes on the destination CTA's mbarrier: the data signals
// its own arrival, so no release fence / arrival round trip follows the push
__device__ __forceinline__ void st_async4(uint32_t raddr, float4 v, uint32_t rbar) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.f32 [%0], {%1,%2,%3,%4}, [%5];"
                 ::"r"(raddr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "r"(rbar) : "memory");
}
__device__ __forceinline__ float ld_cluster(uint32_t raddr) {
    float v;
    asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(raddr) : "memory");
    return v;
}
// remote mbarrier arrivals with cluster-scope release on two peers: the CTA's shared-memory stores before them (ordered by
// a CTA barrier) are visible to a peer that acquires the phase (mbar_wait_cluster).  One fence, then relaxed arrivals:
// the same release pattern as two release arrivals, which would each carry a GPU-scope memory barrier.
__device__ __forceinline__ void mbar_arrive_release_cluster2(uint32_t raddr0, uint32_t raddr1) {
    asm volatile("fence.acq_rel.cluster;\n\t"
                 "mbarrier.arrive.relaxed.cluster.shared::cluster.b64 _, [%0];\n\t"
                 "mbarrier.arrive.relaxed.cluster.shared::cluster.b64 _, [%1];" ::"r"(raddr0), "r"(raddr1) : "memory");
}
__device__ __forceinline__ bool mbar_wait_cluster(uint64_t* bar, uint32_t parity, long long timeout_cycles) {
    const long long t0 = clock64();
    while (true) {
        uint32_t ok;
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
        if (ok) return true;
        if (clock64() - t0 > timeout_cycles) return false;
    }
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// one thread of a converged warp (CUTLASS elect_one_sync): lets the compiler issue the uniform-datapath
// instructions (UTCHMMA, UBLKCP) of the region directly instead of wrapping each in a vote loop
__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n\t.reg .b32 rx;\n\t.reg .pred px;\n\t"
        "elect.sync rx|px, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, px;\n\t}"
        : "=r"(pred));
    return pred != 0;
}
__device__ __forceinline__ void epi_bar() { asm volatile("bar.sync 1, %0;" ::"n"(NEPI) : "memory"); }
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// Staged accumulator tile accs[64][ACC_LD] in shared memory: the epilogue layout keeps row `row` of the tile in
// lanes l and l + 16 of a warp, NC consecutive columns from `col` (lane l < 16: the low columns, l + 16: the high ones).
template <int NC>
__device__ __forceinline__ void acc_ld(const float* accs, int row, int col, float (&v)[NC]) {
#pragma unroll
    for (int q = 0; q < NC / 4; ++q) {
        const float4 x = *reinterpret_cast<const float4*>(accs + row * ACC_LD + col + 4 * q);
        v[4 * q] = x.x; v[4 * q + 1] = x.y; v[4 * q + 2] = x.z; v[4 * q + 3] = x.w;
    }
}
template <int NC>
__device__ __forceinline__ void acc_st(float* accs, int row, int col, const float (&v)[NC]) {
#pragma unroll
    for (int q = 0; q < NC / 4; ++q)
        *reinterpret_cast<float4*>(accs + row * ACC_LD + col + 4 * q) = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
}

// One GEMM of the step, issued by warpgroup 0 alone straight from the operand ring: NCH chunks of KC k, A = 64 rows,
// B = N rows, full-width m64nNk8 MMAs.  Every output element accumulates over all of K in one register chain, in the
// same order as with narrower MMAs: the result does not depend on how the columns are cut into instructions.  Each warp
// releases a slot once its MMAs have read it: lane r < 8 arrives on the bar_empty of cluster rank r (a CTA's multicast
// copies write into the slot of all 8, so its bar_empty counts the 4 MMA warps of each of them).  One group stays in
// flight.
template <int N>
__device__ __forceinline__ void gemm_phase(const unsigned char* ring, unsigned& qq, uint64_t* bar_full, uint32_t empty_r,
                                           float (&dm)[N / 2], float (&dc)[N / 2], int* err, int code, int lane,
                                           const Args& P, int t, int g) {
#pragma unroll
    for (int e = 0; e < N / 2; ++e) dm[e] = dc[e] = 0.f;
    const uint32_t ring_a = smem_u32(ring);
    constexpr uint32_t b_lbo = 16 * N, b_chunk = N * KC * 4;
    for (int j = 0; j < NCH; ++j, ++qq) {
        const int s = qq % NSLOT;
        if (!mbar_wait(&bar_full[s], (qq / NSLOT) & 1, WAIT_CYCLES)) fail(err, code);
#ifdef FSRL_PPO_CHUNK_STAMPS
        if (P.dbg && t == P.dbg_step && threadIdx.x < 32) P.dbg[(size_t)blockIdx.x * DBG_N + DBG_CH + 3 * NCH * g + 2 * NCH + j] = clock64();
#endif
        __syncwarp();
        wgmma_fence();
        // descriptors of the slot's k-step 0; k-step ks starts 2048 (A) / 2 b_lbo (B) bytes further (the address field
        // holds bytes / 16 and the ring ends far below its 256 KB range, so adding the offset never carries out of it)
        const uint32_t base = ring_a + (uint32_t)s * SLOT_BYTES;
        const uint64_t ah0 = smem_desc(base, 1024, 128), al0 = smem_desc(base + A_CHUNK, 1024, 128);
        const uint64_t bh0 = smem_desc(base + 2 * A_CHUNK, b_lbo, 128), bl0 = smem_desc(base + 2 * A_CHUNK + b_chunk, b_lbo, 128);
#pragma unroll
        for (int ks = 0; ks < KC / 8; ++ks) {
            const uint64_t ah = ah0 + ks * (2048 / 16), al = al0 + ks * (2048 / 16);
            const uint64_t bh = bh0 + ks * (2 * b_lbo / 16), bl = bl0 + ks * (2 * b_lbo / 16);
            if constexpr (N == 32) {
                mma_m64n32k8_tf32(dc, al, bh);
                mma_m64n32k8_tf32(dc, ah, bl);
                mma_m64n32k8_tf32(dm, ah, bh);
            } else {
                mma_m64n64k8_tf32(dc, al, bh);
                mma_m64n64k8_tf32(dc, ah, bl);
                mma_m64n64k8_tf32(dm, ah, bh);
            }
        }
        wgmma_commit();
        if (j > 0) {
            wgmma_wait<1>();
            __syncwarp();
            if (lane < 8) mbar_arrive_cluster(empty_r + 8 * ((qq - 1) % NSLOT));
        }
    }
    wgmma_wait<0>();
    reg_fence(dm); reg_fence(dc);
    __syncwarp();
    if (lane < 8) mbar_arrive_cluster(empty_r + 8 * ((qq - 1) % NSLOT));
}
// Warp w of warpgroup 0 stages its fragment (main + cross terms, rows 16 w .. + 15, all N columns) into accs; warps w
// and w + 4 read those rows back in the epilogue, so one 64-thread barrier per warp pair (ids 2 .. 5) orders them.
template <int N>
__device__ __forceinline__ void stage_acc(float* accs, const float (&dm)[N / 2], const float (&dc)[N / 2], int wq, int sp,
                                          int lane) {
    if (wq == 0) {
        const int r = 16 * sp + (lane >> 2);
#pragma unroll
        for (int i = 0; i < N / 8; ++i) {
            const int c = 8 * i + 2 * (lane & 3);
            *reinterpret_cast<float2*>(accs + r * ACC_LD + c) = make_float2(dm[4 * i] + dc[4 * i], dm[4 * i + 1] + dc[4 * i + 1]);
            *reinterpret_cast<float2*>(accs + (r + 8) * ACC_LD + c) =
                make_float2(dm[4 * i + 2] + dc[4 * i + 2], dm[4 * i + 3] + dc[4 * i + 3]);
        }
    }
    asm volatile("bar.sync %0, 64;" ::"r"(2 + sp) : "memory");
}

// One operand of a ring chunk: its hi part (`bytes` from src) and lo part (`bytes` from src + IMG) go to dst and
// dst + bytes.  g == 1: this CTA copies both for itself.  Otherwise the g CTAs of cta_mask (cluster ranks) need the same
// operand: member i of the group copies the i-th of g equal pieces of [hi | lo] into all of them, so the cluster reads it
// from L2 once.  Every destination expects the bytes of the whole slot on its own bar_full, and a slot is written again
// only after the consumers of every destination CTA have released it (gemm_phase arrives on all 8 CTAs' bar_empty).
// A peer writes into this CTA's ring only after flag A or flag C, and both count this CTA's own arrival, which follows
// its fence.proxy.async.shared::cta: the epilogue's scratch use of the ring is over by then.
__device__ __forceinline__ void copy_operand(unsigned char* dst, const float* src, uint32_t bytes, uint64_t* bar, int g, int i,
                                             uint16_t cta_mask) {
    if (g == 1) {
        bulk_g2s(dst, src, bytes, bar);
        bulk_g2s(dst + bytes, src + IMG, bytes, bar);
        return;
    }
    const uint32_t piece = 2 * bytes / g, off = i * piece, part = off / bytes, in = off % bytes;
    bulk_g2s_multicast(dst + off, src + (size_t)part * IMG + in / 4, piece, bar, cta_mask);
}

// Transposed K-major image of a 64-row tile through shared memory.  Every epilogue thread holds NC consecutive
// columns [c0, c0 + NC) of tile row `row` (hi / lo parts); the tile is W columns wide.  The transposed image
// stores 4 consecutive ROWS of one column as 16 contiguous bytes: element (col, row) at
//     img[(row_base + row) / 4 * 256 + (col_base + col) * 4 + (row_base + row) % 4],     lo image at + IMG.
// (W = tile width in columns.)  Writing it straight from the registers costs NC scattered 4-byte stores per thread and image (16 sectors per warp
// instruction); staged through `scr` (an idle operand-ring slot, row stride 65: conflict-free) it becomes
// float4 stores, 512 contiguous bytes per warp instruction.
template <int NC, int W>
__device__ __forceinline__ void transposed_stage(float* scr, const float (&hi)[NC], const float (&lo)[NC], int row, int c0) {
    constexpr int LO = W * 65;
#pragma unroll
    for (int j = 0; j < NC; ++j) {
        scr[(c0 + j) * 65 + row] = hi[j];
        scr[LO + (c0 + j) * 65 + row] = lo[j];
    }
}
template <int W>
__device__ __forceinline__ void transposed_flush(const float* scr, int et, float* img_hi, int row_base, int col_base) {
    constexpr int LO = W * 65;
    const int col = et % W;
    constexpr int GPT = 16 / (NEPI / W);                       // row groups (of 4 rows) per thread
    const int g0 = (et / W) * GPT;
    float* dst = img_hi + (size_t)(row_base >> 2) * 256 + (size_t)(col_base + col) * 4;
#pragma unroll
    for (int q = 0; q < GPT; ++q) {
        const int g = g0 + q;
        const float* sh = scr + col * 65 + 4 * g;
        *reinterpret_cast<float4*>(dst + (size_t)g * 256) = make_float4(sh[0], sh[1], sh[2], sh[3]);
        *reinterpret_cast<float4*>(dst + IMG + (size_t)g * 256) = make_float4(sh[LO], sh[LO + 1], sh[LO + 2], sh[LO + 3]);
    }
}
template <int NC, int W>
__device__ __forceinline__ void store_transposed(float* scr, const float (&hi)[NC], const float (&lo)[NC], int row, int c0,
                                                 int et, float* img_hi, int row_base, int col_base) {
    transposed_stage<NC, W>(scr, hi, lo, row, c0);
    epi_bar();
    transposed_flush<W>(scr, et, img_hi, row_base, col_base);
    epi_bar();                                                 // scratch may be reused
}

// Observation rows of a G2 CTA's two h1 tiles (row blocks a and a + 2 of the minibatch whose first row is row0: 128 rows
// of D floats) into xs, row i at i * (D | 1): the S phase reads one row per lane, and the odd stride puts the 32 rows
// of a warp into 32 banks.  4-byte asynchronous copies (LDGSTS) hold no registers; the caller waits for them
// (__pipeline_wait_prior) before the barrier that precedes their readers.
//
// Liveness of the landing area, ring bytes [XS_OFF, XS_OFF + 128 (D | 1) 4) (slot 2 on): the copies for step t + 1 are
// issued after this CTA's G2 of step t has consumed every chunk (all bytes bound for this ring have landed), and peers
// copy into the ring again only after flag A of step t + 1, which counts this CTA's arrival after its S phase has read
// the rows.  Below XS_OFF the ring holds the dW1 / db1 partials until D2 ([wq][D + 1][64 k], at most 21 KB) and the
// S-phase transposed staging (two [64 x 32] hi / lo tiles, 33 KB).
__device__ __forceinline__ void stage_rows(float* xs, const float* obs, long long row0, int a, int D, int et) {
    const int i = et >> 1;                                   // row i of the 128: two threads per row, alternate d
    const float* src = obs + (row0 + 64 * a + i + (i & 64)) * D;
    float* dst = xs + i * (D | 1);
    for (int d = et & 1; d < D; d += 2) __pipeline_memcpy_async(dst + d, src + d, 4);
    __pipeline_commit();
}

// sum over the 16 lanes of a half-warp (lanes l and l ^ 16 hold different data)
__device__ __forceinline__ float half_sum(float v) {
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// layout of the small-parameter slices a CTA keeps in shared memory (floats)
struct SliceMap {
    int w1, b2, w3, b3, n;     // w1: [(D+1)][32] (row D = b1), b2: [32], w3: [32][OUTP], b3: [16] (b3 | log sigma at 8)
    __device__ __host__ SliceMap(int D) { w1 = 0; b2 = (D + 1) * 32; w3 = b2 + 32; b3 = w3 + 32 * OUTP; n = b3 + 16; }
};

// ---- data-parallel exchange, out of line ---------------------------------------------------------------------------------
// All of it lives in functions the kernel CALLS: inlined into the epilogue, the mere presence of this code slows every
// phase of the step down even with world = 1 -- register allocation and the instruction footprint of the long epilogue
// are that tight.
struct DpCtx {
    const float* const* xg;   // [rank] exchange buffers of this step's parity (shared-memory table)
    long long region;         // floats per source-rank region
    int me, world;
    uint32_t tag;
    int* err;
    int direct;               // W2 tiles in ONE hop (every rank sums all ranks' tiles itself): less latency, W - 1 tile
                              // volumes per rank -- the choice for 2 ranks; the two-hop owner scheme beyond
};
__device__ __forceinline__ int dp_owner(int et, int q, int world) { return (int)((unsigned)((et >> 5) * TILE_PK + q) % (unsigned)world); }

// hop 1 of a W2 gradient tile: every packet of the local tile (staged accumulators) to its owner
__device__ __noinline__ void dp_tile_send(DpCtx d, size_t off, const float* accs, int trow, int cb2, int et) {
    float g[C2];
    acc_ld<C2>(accs, trow, cb2, g);
#pragma unroll
    for (int q = 0; q < TILE_PK; ++q) {
        const size_t o_q = (size_t)d.me * d.region + off + (size_t)q * NEPI * 4;
        const float x = g[3 * q], y = 3 * q + 1 < C2 ? g[3 * q + 1] : 0.f, z = 3 * q + 2 < C2 ? g[3 * q + 2] : 0.f;
        if (d.direct) {
            dp_push_all(d.xg, o_q, d.me, d.world, x, y, z, d.tag);
        } else {
            const int o = dp_owner(et, q, d.world);
            if (o != d.me) st_packet(const_cast<float*>(d.xg[o]) + o_q, x, y, z, d.tag);
        }
    }
}
// hop 2: owned packets -- rank-ordered mean of the ranks' contributions, pushed into everybody's result region; the tile
// (owned entries final, the others still local) replaces the staged accumulators
__device__ __noinline__ void dp_tile_reduce(DpCtx d, size_t off, float* accs, int trow, int cb2, int et) {
    float g[C2];
    acc_ld<C2>(accs, trow, cb2, g);
    const float inv_world = 1.0f / (float)d.world;
    const float* loc = d.xg[d.me];
#pragma unroll
    for (int q = 0; q < TILE_PK; ++q) {
        if (dp_owner(et, q, d.world) != d.me) continue;
        const float3 s3 = dp_gather(loc + off + (size_t)q * NEPI * 4, d.region, d.me, d.world, d.tag, g[3 * q],
                                    3 * q + 1 < C2 ? g[3 * q + 1] : 0.f, 3 * q + 2 < C2 ? g[3 * q + 2] : 0.f, d.err, 41);
        const float ax = s3.x * inv_world, ay = s3.y * inv_world, az = s3.z * inv_world;
        dp_push_all(d.xg, (size_t)FSRL_P2P_MAX_RANKS * d.region + off + (size_t)q * NEPI * 4, d.me, d.world, ax, ay, az, d.tag);
        g[3 * q] = ax;
        if (3 * q + 1 < C2) g[3 * q + 1] = ay;
        if (3 * q + 2 < C2) g[3 * q + 2] = az;
    }
    acc_st<C2>(accs, trow, cb2, g);
}
// the other owners' means: wait for them in the local result region, complete the staged tile, return its sum of squares
__device__ __noinline__ float dp_tile_finish(DpCtx d, size_t off, float* accs, int trow, int cb2, int et) {
    float g[C2];
    const long long t0w = clock64();
    if (d.direct) {
        // one hop: all ranks' tiles are (or will be) in the local contribution regions -- rank-ordered mean, rank by rank
        float own[C2];
        acc_ld<C2>(accs, trow, cb2, own);
#pragma unroll
        for (int jq = 0; jq < C2; ++jq) g[jq] = 0.f;
        for (int r = 0; r < d.world; ++r) {
            if (r == d.me) {
#pragma unroll
                for (int jq = 0; jq < C2; ++jq) g[jq] += own[jq];
                continue;
            }
            const float* src = d.xg[d.me] + (size_t)r * d.region + off;
            float4 v[TILE_PK];
            bool ok;
            do {
                ok = true;
#pragma unroll
                for (int q = 0; q < TILE_PK; ++q) v[q] = ld_packet(src + (size_t)q * NEPI * 4);
#pragma unroll
                for (int q = 0; q < TILE_PK; ++q) ok = ok && pk_ok(v[q], d.tag);
                if (!ok && clock64() - t0w > 4 * WAIT_CYCLES) fail(d.err, 42);
            } while (!ok);
#pragma unroll
            for (int q = 0; q < TILE_PK; ++q) {
                g[3 * q] += v[q].x;
                if (3 * q + 1 < C2) g[3 * q + 1] += v[q].y;
                if (3 * q + 2 < C2) g[3 * q + 2] += v[q].z;
            }
        }
        const float inv_world = 1.0f / (float)d.world;
        float sq = 0.f;
#pragma unroll
        for (int jq = 0; jq < C2; ++jq) { g[jq] *= inv_world; sq = fmaf(g[jq], g[jq], sq); }
        acc_st<C2>(accs, trow, cb2, g);
        return sq;
    }
    const float* res = d.xg[d.me] + (size_t)FSRL_P2P_MAX_RANKS * d.region + off;
    acc_ld<C2>(accs, trow, cb2, g);
    float4 v[TILE_PK];
    bool ok;
    do {
        ok = true;
#pragma unroll
        for (int q = 0; q < TILE_PK; ++q)
            if (dp_owner(et, q, d.world) != d.me) v[q] = ld_packet(res + (size_t)q * NEPI * 4);
#pragma unroll
        for (int q = 0; q < TILE_PK; ++q)
            if (dp_owner(et, q, d.world) != d.me) ok = ok && pk_ok(v[q], d.tag);
        if (!ok && clock64() - t0w > 4 * WAIT_CYCLES) fail(d.err, 42);
    } while (!ok);
    float sq = 0.f;
#pragma unroll
    for (int q = 0; q < TILE_PK; ++q) {
        if (dp_owner(et, q, d.world) == d.me) continue;
        g[3 * q] = v[q].x;
        if (3 * q + 1 < C2) g[3 * q + 1] = v[q].y;
        if (3 * q + 2 < C2) g[3 * q + 2] = v[q].z;
    }
#pragma unroll
    for (int jq = 0; jq < C2; ++jq) sq = fmaf(g[jq], g[jq], sq);
    acc_st<C2>(accs, trow, cb2, g);
    return sq;
}
// small-parameter slice of one column block (n floats in shared memory), called by its reducer only: pushes the slice to
// every rank and replaces it by the rank-ordered mean (one hop: this exchange is on the step's critical path); the other
// CTAs of the column block read the mean from the reducer's published slice after hop D2
__device__ __noinline__ void dp_slices(DpCtx d, size_t off_s, float* sp_g, int n, int et) {
    const int n3 = (n + 2) / 3;
    const float inv_world = 1.0f / (float)d.world;
    for (int i = et; i < n3; i += NEPI)
        dp_push_all(d.xg, (size_t)d.me * d.region + off_s + 4 * (size_t)i, d.me, d.world,
                    sp_g[3 * i], 3 * i + 1 < n ? sp_g[3 * i + 1] : 0.f, 3 * i + 2 < n ? sp_g[3 * i + 2] : 0.f, d.tag);
    const float* loc = d.xg[d.me];
    for (int i = et; i < n3; i += NEPI) {
        const float3 s3 = dp_gather(loc + off_s + 4 * (size_t)i, d.region, d.me, d.world, d.tag, sp_g[3 * i],
                                    3 * i + 1 < n ? sp_g[3 * i + 1] : 0.f, 3 * i + 2 < n ? sp_g[3 * i + 2] : 0.f, d.err, 40);
        sp_g[3 * i] = s3.x * inv_world;
        if (3 * i + 1 < n) sp_g[3 * i + 1] = s3.y * inv_world;
        if (3 * i + 2 < n) sp_g[3 * i + 2] = s3.z * inv_world;
    }
}

// Reducer of column block b's small-parameter gradient (CTA c = 8 a + b with a = b >> 2): the CTA of that column block
// in the cluster whose G2 CTAs (k block b >> 1, CTAs 4 (b >> 1) .. + 3) produce its dW1 / db1 partials -- CTAs 0-3 and
// 12-15 of each network.  Re-derived from blockIdx at each use rather than kept in a register: in <DP = true> a value
// live across the exchange calls costs spill traffic.
__device__ __forceinline__ bool red_cta() { return ((blockIdx.x >> 3) & 3) == ((blockIdx.x & 7) >> 2); }

// the exchange part of the step tail behind one call site: G3 CTAs complete their W2 gradient tile with the ranks'
// mean (returns its sum of squares), reducers replace their slice by the ranks' mean
__device__ __noinline__ float dp_tail(DpCtx d, size_t off_t, size_t off_s, float* accs, float* sp_g, int n, int trow, int cb2,
                                      int et, bool tile, bool slice) {
    if (tile && !d.direct) dp_tile_reduce(d, off_t, accs, trow, cb2, et);
    if (slice) dp_slices(d, off_s, sp_g, n, et);
    __syncwarp();
    return tile ? dp_tile_finish(d, off_t, accs, trow, cb2, et) : 0.f;
}

// DP = false: single-GPU instantiation without any of the exchange code (smaller instruction footprint)
template <bool DP>
__global__ void __launch_bounds__(TPB, 1) ppo_persist_kernel(const Args P) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    __shared__ __align__(8) uint64_t bar_full[NSLOT], bar_empty[NSLOT], bar_b, bar_w1;
    __shared__ float s_red[4][320];          // cross-subpartition partial sums
    __shared__ float s_misc[32];
    __shared__ AdamS s_adam;
    __shared__ const float* s_xg[2][FSRL_P2P_MAX_RANKS];   // peers' exchange buffers (a table the exchange helpers can index)
    const fsrl_ppo_update_t& u = P.u;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int net = blockIdx.x >> 5, c = blockIdx.x & 31, a = c >> 3, b = c & 7;
    const bool is_g2 = c < 16;
    const int ka = (c & 15) >> 2, q4 = c & 3;      // G2: (k block, row block) ; G3: (k block, o block)

    const int D = u.D, A = u.A, C = u.C, H = H_;
    const int out = (net == 0) ? A : 1;
    const int n_cta = 32 * u.n_nets;
    float* wsn = P.ws + (size_t)net * NET_WS;
    float* sumsq_g = P.ws + (size_t)u.n_nets * NET_WS;
    unsigned* fl_net = P.flags + (size_t)net * F_PER_NET * FLAG_LINE;
    unsigned* fl_d2 = P.flags + (size_t)u.n_nets * F_PER_NET * FLAG_LINE;
    unsigned char* ring = smem_raw;
    float* accs = reinterpret_cast<float*>(smem_raw + NSLOT * SLOT_BYTES);     // staged accumulator tile [64][ACC_LD]
    float* small = accs + 64 * ACC_LD;
    const SliceMap sm(D);
    float* sp_p = small;                 // parameters
    float* sp_m = small + sm.n;          // Adam first moment
    float* sp_v = small + 2 * sm.n;      // Adam second moment
    float* sp_g = small + 3 * sm.n;      // reduced gradient of the current step
    float* land = small + 4 * sm.n;      // head partials pushed by the 8 CTAs of this row block [b][64][OUTP] (hop B),
                                         // G2's observation block

    if (tid == 0) {
        for (int i = 0; i < NSLOT; ++i) { mbar_init(&bar_full[i], 1); mbar_init(&bar_empty[i], 4 * 8); }
        mbar_init(&bar_b, 1);                // per step: one local expect_tx arrival + 16 KB of remote st.async bytes
        mbar_init(&bar_w1, 4);               // reducers, per step: one arrival of each of the 4 G2 CTAs of k block b >> 1
        fence_mbar_init();
    }
    __syncthreads();
    if (DP && threadIdx.x < 2 * FSRL_P2P_MAX_RANKS) s_xg[threadIdx.x / FSRL_P2P_MAX_RANKS][threadIdx.x % FSRL_P2P_MAX_RANKS] = P.u.p2p_xg[threadIdx.x / FSRL_P2P_MAX_RANKS][threadIdx.x % FSRL_P2P_MAX_RANKS];
    if (DP) __syncthreads();
    cluster_sync_all();                      // every CTA's barriers exist before a peer may arrive on them

    // parameter offsets of this network inside the flat arena
    const long long pbase = u.net_off[net];
    const ArenaLayout L = arena_layout(D, H, out, 0);
    const long long o_w1 = pbase + L.w1, o_b1 = pbase + L.b1, o_w2 = pbase + L.w2, o_b2 = pbase + L.b2,
                    o_w3 = pbase + L.w3, o_b3 = pbase + L.b3, o_ls = pbase + L.extra;

    if (warp == NEPI / 32) {
        // ============================ bulk-copy producer ==========================================
        if (elect_one()) {
            unsigned qq = 0;
            for (int t = 0; t < P.n_mb; ++t) {
                if (!flag_wait_ge<true>(fl_net + F_A * FLAG_LINE, 32u * (t + 1), WAIT_CYCLES)) fail(P.err, 10);
                STAMP(12);
                fence_proxy_async_global();
                // the producer loops stay rolled: one thread runs them, and the kernel's instruction footprint is tight
#pragma unroll 1
                for (int j = 0; j < NCH; ++j, ++qq) {             // G1: K = k in chunks of KC
                    const int s = qq % NSLOT;
                    if (!mbar_wait(&bar_empty[s], ((qq / NSLOT) & 1) ^ 1, WAIT_CYCLES)) fail(P.err, 11);
#ifdef FSRL_PPO_CHUNK_STAMPS
                    STAMP(DBG_CH + j);
#endif
                    unsigned char* dst = ring + (size_t)s * SLOT_BYTES;
                    mbar_expect_tx(&bar_full[s], 3 * A_CHUNK);
                    const size_t ao = (size_t)a * 16384 + (size_t)j * 64 * KC, bo = (size_t)b * 8192 + (size_t)j * 32 * KC;
                    // A = H1A block a: the same for the 8 CTAs of the row block (cluster)
                    copy_operand(dst, wsn + (size_t)I_H1A_HI * IMG + ao, A_CHUNK, &bar_full[s], 8, b, 0xff);
                    copy_operand(dst + 2 * A_CHUNK, wsn + (size_t)I_W2A_HI * IMG + bo, A_CHUNK / 2, &bar_full[s], 1, 0, 0);
#ifdef FSRL_PPO_CHUNK_STAMPS
                    STAMP(DBG_CH + NCH + j);
#endif
                }
                STAMP(13);
                if (!flag_wait_ge<true>(fl_net + F_C * FLAG_LINE, 32u * (t + 1), WAIT_CYCLES)) fail(P.err, 12);
                STAMP(14);
                fence_proxy_async_global();
                const int ia = is_g2 ? I_W2B_HI : I_DZT_HI, ib = is_g2 ? I_DZA_HI : I_H1T_HI;
                const int blk_a = is_g2 ? ka : q4, blk_b = is_g2 ? q4 : ka;
                // the k block ka (G2: A = W2B, G3: B = H1T) is shared by the 4 CTAs with the same b >> 2, the block q4
                // (G2: B = DZA, G3: A = DZT) by the CTAs b and b ^ 4
                const uint16_t m4 = (uint16_t)(0xfu << (b & 4)), m2 = (uint16_t)(0x11u << (b & 3));
#pragma unroll 1
                for (int j = 0; j < NCH; ++j, ++qq) {             // G2: K = o ; G3: K = r ; chunks of KC
                    const int s = qq % NSLOT;
                    if (!mbar_wait(&bar_empty[s], ((qq / NSLOT) & 1) ^ 1, WAIT_CYCLES)) fail(P.err, 13);
#ifdef FSRL_PPO_CHUNK_STAMPS
                    STAMP(DBG_CH + 3 * NCH + j);
#endif
                    unsigned char* dst = ring + (size_t)s * SLOT_BYTES;
                    mbar_expect_tx(&bar_full[s], 4 * A_CHUNK);
                    const size_t ao = (size_t)blk_a * 16384 + (size_t)j * 64 * KC, bo = (size_t)blk_b * 16384 + (size_t)j * 64 * KC;
                    copy_operand(dst, wsn + (size_t)ia * IMG + ao, A_CHUNK, &bar_full[s], is_g2 ? 4 : 2, is_g2 ? b & 3 : b >> 2, is_g2 ? m4 : m2);
                    copy_operand(dst + 2 * A_CHUNK, wsn + (size_t)ib * IMG + bo, A_CHUNK, &bar_full[s], is_g2 ? 2 : 4, is_g2 ? b >> 2 : b & 3, is_g2 ? m2 : m4);
#ifdef FSRL_PPO_CHUNK_STAMPS
                    STAMP(DBG_CH + 4 * NCH + j);
#endif
                }
            }
        }
    } else {
        // ============================ MMA + epilogue warps ========================================
        const int et = tid;                         // 0 .. NEPI - 1
        const int sp = warp & 3;                    // 16-row slab of this warp (its rank in the warpgroup)
        const int wq = warp >> 2;                   // warpgroup: which of the WQ warps of that slab
        const int r16 = lane & 15, half = lane >> 4;
        const int trow = 16 * sp + r16;             // row of the 64-row tile held by this lane
        const int cb1 = 16 * half + C1 * wq;        // first of this thread's C1 columns of a 32-column tile
        const int cb2 = 32 * half + C2 * wq;        // first of this thread's C2 columns of a 64-column tile
        unsigned qq = 0;                            // operand ring position
        // ring releases go to every CTA whose bulk copies write into this one's slots: all 8 of the cluster (multicast)
        const uint32_t empty_r = mapa_u32(smem_u32(bar_empty), lane < 8 ? lane : 0);
        float w2p[C2], w2m[C2], w2v[C2];            // owned W2 tile (G3 CTAs): parameters and Adam moments
        // ---- data-parallel exchange over peer memory (NVLink): every CTA pushes its local gradient piece into its
        // rank's region of EVERY rank's exchange buffer, one thread fences and release-stores the step id into the same
        // slot of every rank's flag array; the receiver waits for the ranks' flags and sums their pieces from its own
        // memory in rank order -- point-to-point between equal CTAs, one NVLink one-way latency, no remote loads,
        // bit-identical sums on every rank.
        const int world = DP ? u.world : 1;
        // W2 tiles travel in two hops (reduce-scatter + all-gather, 2 (W - 1) / W tile volumes per rank instead of W - 1):
        // packet q of epilogue warp w is OWNED by rank (6 w + q) mod W -- every rank sends it there, the owner sums the
        // ranks' packets in rank order and pushes the mean into everybody's result region (region 8).  Both hops are
        // hidden behind the dW1 / slice reduction of the same step; the result is bit-identical on every rank.
        auto dp_ctx = [&](int t_) {
            DpCtx d;
            const unsigned long long id = (unsigned long long)(P.adam_t0 + t_ + 1);
            d.xg = s_xg[(int)(id & 1ULL)];
            d.region = (long long)u.n_nets * XG_PER_NET;
            d.me = u.p2p_rank; d.world = world;
            d.tag = (P.dp_seq << 16) | (uint32_t)((t_ + 1) & 0xffff);
            d.err = P.err;
            d.direct = P.dp_direct;
            return d;
        };

        // ---- initial state: small slices from the arena, the W2 tile (p, m, v) into registers; step 0's h1 rows ----
        float* xs = reinterpret_cast<float*>(ring + XS_OFF);
        if (is_g2) stage_rows(xs, u.obs, 0, a, D, et);
        for (int i = et; i < sm.n; i += NEPI) {
            long long src = -1;
            if (i < sm.b2) { const int d = i / 32, kk = i % 32; src = (d < D) ? o_w1 + (long long)d * H + 32 * b + kk : o_b1 + 32 * b + kk; }
            else if (i < sm.w3) src = o_b2 + 32 * b + (i - sm.b2);
            else if (i < sm.b3) { const int oo = (i - sm.w3) / OUTP, jj = (i - sm.w3) % OUTP; if (jj < out) src = o_w3 + (long long)(32 * b + oo) * out + jj; }
            else { const int jj = i - sm.b3; if (jj < out) src = o_b3 + jj; else if (net == 0 && jj >= 8 && jj < 8 + A) src = o_ls + (jj - 8); }
            sp_p[i] = src >= 0 ? u.theta[src] : 0.f;
            sp_m[i] = src >= 0 ? u.adam_m[src] : 0.f;
            sp_v[i] = src >= 0 ? u.adam_v[src] : 0.f;
            sp_g[i] = 0.f;
        }
        if (!is_g2) {
            const int o = 64 * q4 + trow;
#pragma unroll
            for (int j = 0; j < C2; ++j) {
                const long long idx = o_w2 + (long long)(64 * ka + cb2 + j) * H + o;
                w2p[j] = u.theta[idx]; w2m[j] = u.adam_m[idx]; w2v[j] = u.adam_v[idx];
            }
        } else {
#pragma unroll
            for (int j = 0; j < C2; ++j) w2p[j] = w2m[j] = w2v[j] = 0.f;
        }
        __pipeline_wait_prior(0);
        epi_bar();

        for (int t = 0; t < P.n_mb; ++t) {
            const long long row0 = (long long)t * MB;                 // first row of the minibatch in the gathered arrays
            const int slot = P.slot0 + t;
            if (et == 0) {   // Adam scalars of this step (torch.optim.Adam: python doubles -> f32 at the op; host table)
                s_adam.w1 = (float)(1.0 - u.beta1); s_adam.b2 = (float)u.beta2; s_adam.w2 = (float)(1.0 - u.beta2);
                s_adam.rbc2s = __ldg(P.adam_tab + 2 * t); s_adam.eps = (float)u.adam_eps; s_adam.neg_step = __ldg(P.adam_tab + 2 * t + 1);
                STAMP(0);
                if (P.dbg && t == P.dbg_step) { long long gt; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt)); P.dbg[(size_t)blockIdx.x * DBG_N + 30] = gt; }
                if (P.dbg && t == P.dbg_step + 64) {     // 64 steps later: average cycles and ns per step
                    long long gt; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));
                    P.dbg[(size_t)blockIdx.x * DBG_N + 31] = gt;
                    P.dbg[(size_t)blockIdx.x * DBG_N + 29] = clock64();
                }
            }
            // rows of the NEXT minibatch towards L2 while this one is processed
            if (t + 1 < P.n_mb && et < 64) {
                const long long r = row0 + MB + 64 * a + et;
                prefetch_l2(u.obs + r * D);
                if (D > 32) prefetch_l2(u.obs + r * D + 32);
                if (is_g2) { prefetch_l2(u.obs + (r + 128) * D); if (D > 32) prefetch_l2(u.obs + (r + 128) * D + 32); }
                if (net == 0) { prefetch_l2(u.act + r * A); prefetch_l2(u.logp_old + r); prefetch_l2(u.adv + r); if (C > 1) prefetch_l2(u.adv + u.ld + r); }
                else { prefetch_l2(u.ret + (long long)(net - 1) * u.ld + r); if (u.value_clip) prefetch_l2(u.values + (long long)(net - 1) * u.ld + r); }
            }
            // ---- S(a): publish the images of the owned W2 tile (from registers) ------------------------
            float* scratch = reinterpret_cast<float*>(ring);       // the operand ring is idle outside the GEMM phases
            if (!is_g2) {
                const float (&pv)[C2] = w2p;
                float phi[C2], plo[C2];
                const int o = 64 * q4 + trow;                   // output unit of this lane
                float* w2a_hi = wsn + (size_t)I_W2A_HI * IMG + (size_t)(o >> 5) * 8192 + (size_t)(o & 31) * 4;
                float* w2a_lo = w2a_hi + IMG;
#pragma unroll
                for (int q = 0; q < C2 / 4; ++q) {              // k = 64 ka + cb2 + 4 q + (0..3)
                    float4 hi, lo;
                    tf32_split(pv[4 * q], hi.x, lo.x); tf32_split(pv[4 * q + 1], hi.y, lo.y);
                    tf32_split(pv[4 * q + 2], hi.z, lo.z); tf32_split(pv[4 * q + 3], hi.w, lo.w);
                    const size_t plane = (size_t)(16 * ka + (cb2 >> 2) + q) * 128;
                    *reinterpret_cast<float4*>(w2a_hi + plane) = hi;
                    *reinterpret_cast<float4*>(w2a_lo + plane) = lo;
                    phi[4 * q] = hi.x; phi[4 * q + 1] = hi.y; phi[4 * q + 2] = hi.z; phi[4 * q + 3] = hi.w;
                    plo[4 * q] = lo.x; plo[4 * q + 1] = lo.y; plo[4 * q + 2] = lo.z; plo[4 * q + 3] = lo.w;
                }
                // W2B (MN = k, K = o): "rows" are the output units o, "columns" the 64 k of block ka
                store_transposed<C2, 64>(scratch, phi, plo, trow, cb2, et, wsn + (size_t)I_W2B_HI * IMG + (size_t)ka * 16384, 64 * q4, 0);
            }
            // ---- S(b): h1 tiles [64 rows][32 columns of block b].  The CTAs that own a W2 tile are busy with its Adam
            // step and images, so the other half of the grid (CTAs 0-15: a in {0, 1}) computes the tiles of row
            // blocks a and a + 2 -- same column block, hence the same W1 slice.  Their observation rows are already in
            // shared memory (stage_rows, issued while the previous step waited for D2).
            if (is_g2) {
                const int r = et & 63, kc = C1 * (et >> 6);  // row, first of C1 columns
                const float* x0 = xs + r * (D | 1);
                const float* x1 = xs + (64 + r) * (D | 1);
                float acc2[2][C1];
#pragma unroll
                for (int j = 0; j < C1; ++j) acc2[0][j] = acc2[1][j] = sp_p[sm.w1 + D * 32 + kc + j];      // b1
                for (int d = 0; d < D; ++d) {
                    const float xv0 = x0[d], xv1 = x1[d];
                    const float* w = sp_p + sm.w1 + d * 32 + kc;
#pragma unroll
                    for (int j = 0; j < C1; ++j) { acc2[0][j] = fmaf(xv0, w[j], acc2[0][j]); acc2[1][j] = fmaf(xv1, w[j], acc2[1][j]); }
                }
                constexpr int TSCR = 2 * 32 * 65;                  // staging floats of one [64 x 32] tile (hi + lo)
#pragma unroll
                for (int rep = 0; rep < 2; ++rep) {
                    const int aa = a + 2 * rep;
                    float hi[C1], lo[C1];
                    float* a_hi = wsn + (size_t)I_H1A_HI * IMG + (size_t)aa * 16384 + (size_t)r * 4;
#pragma unroll
                    for (int q = 0; q < C1 / 4; ++q) {
#pragma unroll
                        for (int e = 0; e < 4; ++e) tf32_split(fmaxf(acc2[rep][4 * q + e], 0.f), hi[4 * q + e], lo[4 * q + e]);
                        const size_t plane = (size_t)(8 * b + (kc >> 2) + q) * 256;
                        *reinterpret_cast<float4*>(a_hi + plane) = make_float4(hi[4 * q], hi[4 * q + 1], hi[4 * q + 2], hi[4 * q + 3]);
                        *reinterpret_cast<float4*>(a_hi + IMG + plane) = make_float4(lo[4 * q], lo[4 * q + 1], lo[4 * q + 2], lo[4 * q + 3]);
                    }
                    transposed_stage<C1, 32>(scratch + rep * TSCR, hi, lo, r, kc);
                }
                epi_bar();
                // H1T (MN = k, K = r): block b / 2, columns 32 (b & 1) .. -- both tiles behind ONE pair of barriers
#pragma unroll
                for (int rep = 0; rep < 2; ++rep)
                    transposed_flush<32>(scratch + rep * TSCR, et, wsn + (size_t)I_H1T_HI * IMG + (size_t)(b >> 1) * 16384, 64 * (a + 2 * rep), 32 * (b & 1));
            }
            fence_proxy_async_smem();                                // scratch stores before the next bulk copies into the ring
            epi_bar();
            if (et == 0) { STAMP(1); flag_add_release(fl_net + F_A * FLAG_LINE); }

            // per-row loss inputs (independent of the GEMM): issued now, consumed after the head
            const long long grow = row0 + 64 * a + trow;
            float p_act[8], p_lpo = 0.f, p_adv0 = 0.f, p_adv1 = 0.f, p_ret = 0.f, p_val = 0.f, mean[2] = {0.f, 0.f}, rstd[2] = {1.f, 1.f};
#pragma unroll
            for (int j = 0; j < 8; ++j) p_act[j] = 0.f;
            if (net == 0) {
#pragma unroll
                for (int j = 0; j < 8; ++j) if (j < A) p_act[j] = __ldg(u.act + grow * A + j);
                p_lpo = __ldg(u.logp_old + grow);
                p_adv0 = __ldg(u.adv + grow);
                if (C > 1) p_adv1 = __ldg(u.adv + u.ld + grow);
                const float* ms = u.mb_stats + (size_t)t * 4;
                mean[0] = __ldg(ms); rstd[0] = __ldg(ms + 1); mean[1] = __ldg(ms + 2); rstd[1] = __ldg(ms + 3);
            } else {
                p_ret = __ldg(u.ret + (long long)(net - 1) * u.ld + grow);
                if (u.value_clip) p_val = __ldg(u.values + (long long)(net - 1) * u.ld + grow);
            }
            // the Gaussian's scale does not depend on the head: sigma and 1 / sigma before the GEMM wait (the actor's loss
            // phase is the longest of the three networks and every network waits for it at the global-norm hop)
            float p_ls[8], p_rsg[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                p_ls[j] = (net == 0 && j < A) ? sp_p[sm.b3 + 8 + j] : 0.f;
                p_rsg[j] = 1.0f / expf(p_ls[j]);
            }

            // ---- G1 (wgmma), then its epilogue: h2 = relu(acc + b2), head partial over this tile's 32 columns ----
            {
                float dm[16], dc[16];
                if (wq == 0) gemm_phase<32>(ring, qq, bar_full, empty_r, dm, dc, P.err, 30, lane, P, t, 0);
                else qq += NCH;
                stage_acc<32>(accs, dm, dc, wq, sp, lane);
            }
            if (et == 0) STAMP(2);
            float h2[C1];
            acc_ld<C1>(accs, trow, cb1, h2);
            float hp[OUTP];
#pragma unroll
            for (int j = 0; j < OUTP; ++j) hp[j] = 0.f;
#pragma unroll
            for (int j = 0; j < C1; ++j) {
                h2[j] = fmaxf(h2[j] + sp_p[sm.b2 + cb1 + j], 0.f);
                const float* w = sp_p + sm.w3 + (cb1 + j) * OUTP;
#pragma unroll
                for (int jj = 0; jj < OUTP; ++jj) hp[jj] = fmaf(h2[j], w[jj], hp[jj]);
            }
#pragma unroll
            for (int jj = 0; jj < OUTP; ++jj) hp[jj] += __shfl_xor_sync(0xffffffffu, hp[jj], 16);
            if (WQ > 1) {                                       // the WQ warps of a subpartition hold different columns of the same rows
                float* xh = &s_red[0][0];
                if (half == 0 && wq > 0) {
#pragma unroll
                    for (int jj = 0; jj < OUTP; ++jj) xh[((wq - 1) * 64 + trow) * OUTP + jj] = hp[jj];
                }
                epi_bar();
                if (half == 0 && wq == 0) {
#pragma unroll
                    for (int w2 = 1; w2 < WQ; ++w2)
#pragma unroll
                        for (int jj = 0; jj < OUTP; ++jj) hp[jj] += xh[((w2 - 1) * 64 + trow) * OUTP + jj];
                }
            }
            float outv[OUTP];
#pragma unroll
            for (int jj = 0; jj < OUTP; ++jj) outv[jj] = sp_p[sm.b3 + jj];
            // hop B inside the cluster (8 CTAs = the column blocks of this row block): push the partial rows into every
            // peer's landing zone, one remote mbarrier arrival per peer, then wait for the 8 arrivals on the own barrier
            if (et == 0) {
                STAMP(3);
                mbar_expect_tx(&bar_b, 8u * 64u * OUTP * (uint32_t)sizeof(float));
            }
            if (half == 0 && wq == 0) {
                const uint32_t mine = smem_u32(land + ((size_t)b * 64 + trow) * OUTP);
                const uint32_t bb_ = smem_u32(&bar_b);
#pragma unroll
                for (int r = 0; r < 8; ++r) {
                    const uint32_t ra = mapa_u32(mine, r), rb = mapa_u32(bb_, r);
                    st_async4(ra, make_float4(hp[0], hp[1], hp[2], hp[3]), rb);
                    st_async4(ra + 16, make_float4(hp[4], hp[5], hp[6], hp[7]), rb);
                }
            }
            if (!mbar_wait_cluster(&bar_b, t & 1, WAIT_CYCLES)) fail(P.err, 31);
            __syncwarp();
            if (et == 0) STAMP(4);
#pragma unroll
            for (int bb = 0; bb < 8; ++bb) {
                const float* src = land + ((size_t)bb * 64 + trow) * OUTP;
                const float4 v0 = *reinterpret_cast<const float4*>(src);
                const float4 v1 = *reinterpret_cast<const float4*>(src + 4);
                outv[0] += v0.x; outv[1] += v0.y; outv[2] += v0.z; outv[3] += v0.w;
                outv[4] += v1.x; outv[5] += v1.y; outv[6] += v1.z; outv[7] += v1.w;
            }
            // ---- loss gradient at the head (ppo_lag.py:152-212): dd[j] = d loss / d head_j --------------
            float dd[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) dd[j] = 0.f;
            float st_a = 0.f, st_b = 0.f, st_c = 0.f, st_d = 0.f;
            {
                const float invB = 1.0f / (float)MB;
                if (net == 0) {
                    float g_mu[8], g_ls[8];
                    ppo_actor_row(u, outv, p_act, p_ls, p_rsg, p_lpo, p_adv0, p_adv1, mean, rstd, invB, g_mu, g_ls,
                                  st_a, st_b, st_c);
#pragma unroll
                    for (int j = 0; j < 8; ++j) { dd[j] = g_mu[j]; dd[8 + j] = g_ls[j]; }    // log sigma columns: 8 ..
                } else {
                    dd[0] = ppo_value_row(u, outv[0], p_ret, p_val, invB, st_d);
                }
            }
            if (et == 0) STAMP(26);
            // ---- dz2 tile = (dOut W3^T) * relu'(h2): images DZA / DZT; partial db2, dW3, db3 ----------------
            const int nfeed = (net == 0) ? A : 1;              // head columns that feed W3 (mu only)
            float dz[C1];
#pragma unroll
            for (int j = 0; j < C1; ++j) {
                const float* w = sp_p + sm.w3 + (cb1 + j) * OUTP;
                float g = 0.f;
#pragma unroll
                for (int jj = 0; jj < OUTP; ++jj) if (jj < nfeed) g = fmaf(dd[jj], w[jj], g);
                dz[j] = h2[j] > 0.f ? g : 0.f;
            }
            {
                float hi[C1], lo[C1];
                float* a_hi = wsn + (size_t)I_DZA_HI * IMG + (size_t)a * 16384 + (size_t)trow * 4;
#pragma unroll
                for (int q = 0; q < C1 / 4; ++q) {
#pragma unroll
                    for (int e = 0; e < 4; ++e) tf32_split(dz[4 * q + e], hi[4 * q + e], lo[4 * q + e]);
                    const size_t plane = (size_t)(8 * b + (cb1 >> 2) + q) * 256;
                    *reinterpret_cast<float4*>(a_hi + plane) = make_float4(hi[4 * q], hi[4 * q + 1], hi[4 * q + 2], hi[4 * q + 3]);
                    *reinterpret_cast<float4*>(a_hi + IMG + plane) = make_float4(lo[4 * q], lo[4 * q + 1], lo[4 * q + 2], lo[4 * q + 3]);
                }
                // DZT (MN = o, K = r): block b / 2, columns 32 (b & 1) ..
                store_transposed<C1, 32>(scratch, hi, lo, trow, cb1, et, wsn + (size_t)I_DZT_HI * IMG + (size_t)(b >> 1) * 16384, 64 * a, 32 * (b & 1));
            }
            if (et == 0) STAMP(27);
            // partial sums over this tile's 64 rows: half-warp butterflies (16 rows of a subpartition), one shared
            // memory exchange, then 4-way sums.  s_red row: [0,32) db2 | [32,32+32 nfeed) dW3 | [288,304) db3, dlog sigma | [304,308) loss sums
            {
                float* row = &s_red[sp][0];
#pragma unroll
                for (int j = 0; j < C1; ++j) {
                    const float sdz = half_sum(dz[j]);
                    if (r16 == 0) row[cb1 + j] = sdz;
                }
#pragma unroll
                for (int jj = 0; jj < OUTP; ++jj) {
                    if (jj < nfeed) {
#pragma unroll
                        for (int j = 0; j < C1; ++j) {
                            const float sv = half_sum(h2[j] * dd[jj]);
                            if (r16 == 0) row[32 + 32 * jj + cb1 + j] = sv;
                        }
                    }
                }
                if (b == 0 && wq == 0) {                            // per-row quantities: one warp of each subpartition
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        const float sv = half_sum(dd[j]);
                        if (lane == 0) row[288 + j] = sv;
                    }
                    const float sa = half_sum(st_a), sb = half_sum(st_b), sc = half_sum(st_c), sdv = half_sum(st_d);
                    if (lane == 0) { row[304] = sa; row[305] = sb; row[306] = sc; row[307] = sdv; }
                }
            }
            epi_bar();
            if (et == 0) STAMP(28);
            for (int i = et; i < 32 + 32 * nfeed; i += NEPI) {
                const float tot = ((s_red[0][i] + s_red[1][i]) + s_red[2][i]) + s_red[3][i];
                if (i < 32) wsn[DB2P_OFF + a * H + 32 * b + i] = tot;
                else wsn[DW3P_OFF + ((size_t)a * H + 32 * b + ((i - 32) & 31)) * OUTP + ((i - 32) >> 5)] = tot;
            }
            if (b == 0) {                                       // db3 | d log sigma partial, loss statistics
                if (et < 20) {
                    const int i = 288 + et;
                    const float tot = ((s_red[0][i] + s_red[1][i]) + s_red[2][i]) + s_red[3][i];
                    if (et < 16) wsn[DB3P_OFF + a * 16 + et] = tot;
                    else {
                        float* stat = u.stats + (size_t)slot * FSRL_PPO_STATS;
                        if (net == 0) { if (et == 16) atomicAdd(stat + ST_ACTOR_REW, tot); if (et == 17) atomicAdd(stat + ST_ACTOR_SAFETY, tot); if (et == 18) atomicAdd(stat + ST_KL, tot); }
                        else if (et == 19) atomicAdd(stat + ST_VF0 + (net - 1), tot);
                    }
                }
                if (net == 0 && a == 0 && et == 20) u.stats[(size_t)slot * FSRL_PPO_STATS + ST_ENTROPY] = ppo_entropy(sp_p + sm.b3 + 8, A);
            }
            fence_proxy_async_smem();                                // scratch stores before the next bulk copies into the ring
            epi_bar();
            if (et == 0) { STAMP(5); flag_add_release(fl_net + F_C * FLAG_LINE); }

            // ---- G2 / G3 epilogue ---------------------------------------------------------------------------
            // G2: what does not depend on the accumulators is requested BEFORE waiting for them -- the ReLU mask of
            // this lane's h1 entries (image H1A, complete since flag A) and this thread's share of the 64 x D
            // observation block of row block q4.  Neither stays in registers across the GEMM, whose accumulators need
            // them: the mask is kept as C2 bits, the block is staged in the hop-B landing zone, idle until the next step
            // (row r at r * dp4 + 4 (r >> 5), dp4 = D rounded up to a multiple of 4: 16-byte aligned rows for the dW1
            // loop's vector reads, and the two half-warps read different banks).
            unsigned mbits = 0;
            if (is_g2) {
                const int k = 64 * ka + trow;
                const float* msk = wsn + (size_t)I_H1A_HI * IMG + (size_t)q4 * 16384 + (size_t)(k >> 2) * 256 + (k & 3);
                float mreg[C2];
#pragma unroll
                for (int jq = 0; jq < C2; ++jq) mreg[jq] = __ldcg(msk + (size_t)(cb2 + jq) * 4);
                float xr[(64 * MAXD + NEPI - 1) / NEPI];
                const int nx = (64 * D + NEPI - 1) / NEPI;
                const float* xb = u.obs + (row0 + 64 * q4) * D;
#pragma unroll
                for (int q = 0; q < (64 * MAXD + NEPI - 1) / NEPI; ++q)
                    xr[q] = (q < nx && et + q * NEPI < 64 * D) ? __ldg(xb + et + q * NEPI) : 0.f;
#pragma unroll
                for (int jq = 0; jq < C2; ++jq) mbits |= (mreg[jq] > 0.f ? 1u : 0u) << jq;
#pragma unroll
                for (int q = 0; q < (64 * MAXD + NEPI - 1) / NEPI; ++q) {
                    const int e = et + q * NEPI;
                    if (q < nx && e < 64 * D) { const int r = e / D; land[r * ((D + 3) & ~3) + 4 * (r >> 5) + (e - r * D)] = xr[q]; }
                }
            }
            // reducers: warpgroup 1 would only wait for warpgroup 0's GEMM -- it sums the b2 / W3 / b3 / log sigma
            // partials of slice b (complete since flag C) into sp_g meanwhile.  Each element: its 4 row-block partials
            // in order a = 0 .. 3, starting from 0.
            if (red_cta() && wq == 1) {
                const int tw = et - 128;
                if (tw == 0) {
                    if (!flag_wait_ge(fl_net + F_C * FLAG_LINE, 32u * (t + 1), WAIT_CYCLES)) fail(P.err, 35);
                    STAMP(15);
                }
                asm volatile("bar.sync 6, 128;" ::: "memory");
                for (int i0 = sm.b2 + tw; i0 < sm.n; i0 += 4 * 128) {     // 4 elements x 4 partials in flight per thread
                    float pv[4][4];
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const int i = i0 + e * 128;
                        const float* src = wsn;
                        size_t stride = 0;
                        bool real = false;
                        if (i < sm.n) {
                            if (i < sm.w3) { src = wsn + DB2P_OFF + 32 * b + (i - sm.b2); stride = H; real = true; }
                            else if (i < sm.b3) {
                                const int oo = (i - sm.w3) / OUTP, jj = (i - sm.w3) % OUTP;
                                real = jj < out;
                                src = wsn + DW3P_OFF + ((size_t)32 * b + oo) * OUTP + jj; stride = (size_t)H * OUTP;
                            } else {
                                const int jj = i - sm.b3;
                                real = (jj < out) || (net == 0 && jj >= 8 && jj < 8 + A);
                                src = wsn + DB3P_OFF + jj; stride = 16;
                            }
                        }
#pragma unroll
                        for (int q = 0; q < 4; ++q) pv[e][q] = real ? __ldcg(src + q * stride) : 0.f;
                    }
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const int i = i0 + e * 128;
                        if (i < sm.n) {
                            float gsum = 0.f;
#pragma unroll
                            for (int q = 0; q < 4; ++q) gsum += pv[e][q];          // fixed order
                            sp_g[i] = gsum;
                        }
                    }
                }
                if (tw == 0) STAMP(16);
            }
            {
                float dm[32], dc[32];
                if (wq == 0) gemm_phase<64>(ring, qq, bar_full, empty_r, dm, dc, P.err, 32, lane, P, t, 1);
                else qq += NCH;
                stage_acc<64>(accs, dm, dc, wq, sp, lane);
            }
            if (et == 0) STAMP(6);
            float sq = 0.f;
            if (is_g2) {
                // lane: k = 64 ka + trow ; rows cb2 + j of row block q4; partial set 2 q4 + wq (WQ sets per row block).
                // The partials stay in this CTA's operand ring, [wq][D + 1][64 k]: every chunk of this step's G2 has
                // landed and been consumed, and no peer copies into the ring again before flag A of the next step.
                float v[C2];
                acc_ld<C2>(accs, trow, cb2, v);
#pragma unroll
                for (int jq = 0; jq < C2; ++jq) v[jq] = ((mbits >> jq) & 1u) ? v[jq] : 0.f;
                epi_bar();
                if (et == 0) STAMP(22);
                // 4 of the D independent sums at a time, so that their FMA chains interleave: each d keeps its own
                // accumulator, fed in jq order from 0, and one 16-byte read gives the 4 d of row cb2 + jq.  The last
                // batch may run past D into the row's padding; those sums are not stored.
                const int dp4 = (D + 3) & ~3;
                const float* xh = land + (size_t)cb2 * dp4 + 4 * half;
                float* dst = reinterpret_cast<float*>(ring) + (size_t)wq * (D + 1) * 64 + trow;
                for (int d0 = 0; d0 < D; d0 += 4) {
                    float sacc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                    for (int jq = 0; jq < C2; ++jq) {
                        const float4 x = *reinterpret_cast<const float4*>(xh + jq * dp4 + d0);
                        sacc[0] = fmaf(x.x, v[jq], sacc[0]);
                        sacc[1] = fmaf(x.y, v[jq], sacc[1]);
                        sacc[2] = fmaf(x.z, v[jq], sacc[2]);
                        sacc[3] = fmaf(x.w, v[jq], sacc[3]);
                    }
#pragma unroll
                    for (int i = 0; i < 4; ++i) sacc[i] += __shfl_xor_sync(0xffffffffu, sacc[i], 16);
                    if (half == 0) {
#pragma unroll
                        for (int i = 0; i < 4; ++i)
                            if (d0 + i < D) dst[(d0 + i) * 64] = sacc[i];
                    }
                }
                float sb1 = 0.f;
#pragma unroll
                for (int jq = 0; jq < C2; ++jq) sb1 += v[jq];
                sb1 += __shfl_xor_sync(0xffffffffu, sb1, 16);
                if (half == 0) dst[D * 64] = sb1;                 // db1
                if (et == 0) STAMP(23);
                epi_bar();
                // the reducers of column blocks 2 ka and 2 ka + 1 (cluster ranks = column blocks) may read them now
                if (et == 0) mbar_arrive_release_cluster2(mapa_u32(smem_u32(&bar_w1), 2 * ka), mapa_u32(smem_u32(&bar_w1), 2 * ka + 1));
            } else {
                float g[C2];
                acc_ld<C2>(accs, trow, cb2, g);
                if (DP) {
                    dp_tile_send(dp_ctx(t), (size_t)(net * 16 + (c - 16)) * TILE_FLOATS + (size_t)et * 4, accs, trow, cb2, et);
                    if (et == 0) STAMP(32);
                } else {
#pragma unroll
                    for (int jq = 0; jq < C2; ++jq) sq = fmaf(g[jq], g[jq], sq);
                }
            }
            if (et == 0) STAMP(7);
            // ---- small-parameter gradients (reducers): W1 / b1 = fixed-order sums of the 8 partials q = WQ rb + wq in the
            // rings of the G2 CTAs 4 (b >> 1) + rb (cluster ranks (4 (b >> 1) + rb) & 7), read over distributed shared memory
            if (red_cta()) {
                if (!mbar_wait_cluster(&bar_w1, t & 1, WAIT_CYCLES)) fail(P.err, 33);
                if (et == 0) STAMP(8);
                const uint32_t ring_s = smem_u32(ring);
                const int kb = 32 * (b & 1);                           // the slice's first k inside k block b >> 1
                for (int i0 = et; i0 < sm.b2; i0 += 2 * NEPI) {       // 2 elements x 8 partials in flight per thread
                    float pv[2][4 * WQ];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int i = i0 + e * NEPI;
                        const uint32_t off = 4u * (uint32_t)((i / 32) * 64 + kb + (i % 32));
#pragma unroll
                        for (int rb = 0; rb < 4; ++rb) {
                            const uint32_t src = mapa_u32(ring_s + off, (uint32_t)((4 * (b >> 1) + rb) & 7));
#pragma unroll
                            for (int w = 0; w < WQ; ++w)
                                pv[e][WQ * rb + w] = i < sm.b2 ? ld_cluster(src + 4u * (uint32_t)(w * (D + 1) * 64)) : 0.f;
                        }
                    }
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int i = i0 + e * NEPI;
                        if (i < sm.b2) {
                            float gsum = 0.f;
#pragma unroll
                            for (int q = 0; q < 4 * WQ; ++q) gsum += pv[e][q];          // fixed order
                            sp_g[i] = gsum;
                        }
                    }
                }
                epi_bar();                                    // sp_g complete (warpgroup 1 summed b2 .. n before the G2 epilogue)
                if (et == 0) STAMP(17);
            }
            if (DP) {
                const DpCtx d = dp_ctx(t);
                const size_t off_t = (size_t)(net * 16 + (c - 16)) * TILE_FLOATS + (size_t)et * 4;
                sq += dp_tail(d, off_t, (size_t)u.n_nets * 16 * TILE_FLOATS + (size_t)(net * 8 + b) * SLICE_PK * 4, accs, sp_g, sm.n,
                              trow, cb2, et, !is_g2, red_cta());
                if (et == 0) STAMP(41);
                epi_bar();                                    // sp_g holds the ranks' mean before the norm reads it
            }
            if (red_cta()) {
                // every small parameter is counted once in the norm: the W1/b1/b2/W3 slices by their reducers, b3 / log sigma
                // by the reducer of b = 0.  The slice goes out to the other CTAs of the column block with it.
                for (int i = et; i < sm.n; i += NEPI) {
                    bool real = true;
                    if (i >= sm.w3 && i < sm.b3) real = ((i - sm.w3) % OUTP) < out;
                    else if (i >= sm.b3) { const int jj = i - sm.b3; real = (jj < out) || (net == 0 && jj >= 8 && jj < 8 + A); }
                    if (real && (i < sm.b3 || b == 0)) sq = fmaf(sp_g[i], sp_g[i], sq);
                    wsn[SLICE_OFF + (size_t)b * NSMAX + i] = sp_g[i];   // final gradient slice of column block b
                }
            }
            // ---- global gradient norm: per-CTA partials -> device-wide hop -> same summation order everywhere.  Slot
            // 32 net + b holds column block b's slice (written by its reducer), slots 32 net + 16 .. 31 the W2 tiles; slots
            // 32 net + 8 .. 15 stay +0 (zeroed at launch), so only 24 CTAs per network arrive.
            if (red_cta() || !is_g2) {
                sq = warp_sum(sq);
                if (lane == 0) s_misc[warp] = sq;
                epi_bar();
                if (et == 0) {
                    float tot = 0.f;
#pragma unroll
                    for (int w2 = 0; w2 < NEPI / 32; ++w2) tot += s_misc[w2];
                    sumsq_g[blockIdx.x - (red_cta() ? 8 * a : 0)] = tot;
                    STAMP(9);
                    flag_add_release(fl_d2);
                }
            }
            // the next step's h1 rows travel while the CTA waits for D2 and steps its parameters
            if (is_g2 && t + 1 < P.n_mb) stage_rows(xs, u.obs, row0 + MB, a, D, et);
            if (et == 0) {
                if (!flag_wait_ge(fl_d2, 24u * (unsigned)u.n_nets * (t + 1), WAIT_CYCLES)) fail(P.err, 34);
                STAMP(10);
            }
            epi_bar();
            float nq[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) nq[q] = (lane + 32 * q < n_cta) ? __ldcg(sumsq_g + lane + 32 * q) : 0.f;
            // the other CTAs of the column block fetch its final slice in the same round trip (each thread the elements
            // it steps below: same i = et + k NEPI mapping, no barrier needed).  <DP = true> reads it inside the Adam loop
            // instead: a separate pass there raises the register pressure of the whole step and with it the spills.
            if (!DP && !red_cta())
                for (int i = et; i < sm.n; i += NEPI) sp_g[i] = __ldcg(wsn + SLICE_OFF + (size_t)b * NSMAX + i);
            float nsq = ((nq[0] + nq[1]) + nq[2]) + nq[3];                          // identical order in every warp of the grid
            nsq = warp_sum(nsq);
            float gscale = 1.0f;
            if (u.max_grad_norm > 0.f) gscale = fminf(u.max_grad_norm / (sqrtf(nsq) + 1e-6f), 1.0f);
            if (blockIdx.x == 0 && et == 0) u.stats[(size_t)slot * FSRL_PPO_STATS + ST_GRADNORM] = sqrtf(nsq);
            const AdamS ad = s_adam;
            if (et == 0) STAMP(24);
            // ---- clip + Adam: replicated small slices, then the owned W2 tile (registers) ------------------------
            for (int i = et; i < sm.n; i += NEPI) {
                float m = sp_m[i], v = sp_v[i];
                const float g = (DP && !red_cta()) ? __ldcg(wsn + SLICE_OFF + (size_t)b * NSMAX + i) : sp_g[i];
                sp_p[i] = adam_one(sp_p[i], g * gscale, m, v, ad);
                sp_m[i] = m; sp_v[i] = v;
            }
            if (et == 0) STAMP(25);
            if (!is_g2) {
                float g[C2];
                acc_ld<C2>(accs, trow, cb2, g);            // data-parallel runs: the ranks' mean (dp_tile_*)
#pragma unroll
                for (int j = 0; j < C2; ++j) w2p[j] = adam_one(w2p[j], g[j] * gscale, w2m[j], w2v[j], ad);
            } else {
                __pipeline_wait_prior(0);                 // the next step's h1 rows (stage_rows) landed
                if (et == 0) STAMP(18);
            }
            epi_bar();     // slices and h1 rows final before the next h1 tile / head reads them; s_adam may be rewritten
            if (et == 0) STAMP(11);
        }

        // ---- write the parameters and Adam moments back to the arena ------------------------------------------
        if (a == 0) {
            for (int i = et; i < sm.n; i += NEPI) {
                long long dst = -1;
                if (i < sm.b2) { const int d = i / 32, kk = i % 32; dst = (d < D) ? o_w1 + (long long)d * H + 32 * b + kk : o_b1 + 32 * b + kk; }
                else if (i < sm.w3) dst = o_b2 + 32 * b + (i - sm.b2);
                else if (i < sm.b3) { const int oo = (i - sm.w3) / OUTP, jj = (i - sm.w3) % OUTP; if (jj < out) dst = o_w3 + (long long)(32 * b + oo) * out + jj; }
                else if (b == 0) { const int jj = i - sm.b3; if (jj < out) dst = o_b3 + jj; else if (net == 0 && jj >= 8 && jj < 8 + A) dst = o_ls + (jj - 8); }
                if (dst >= 0) { u.theta[dst] = sp_p[i]; u.adam_m[dst] = sp_m[i]; u.adam_v[dst] = sp_v[i]; }
            }
        }
        if (!is_g2) {
            const int o = 64 * q4 + trow;
#pragma unroll
            for (int j = 0; j < C2; ++j) {
                const long long idx = o_w2 + (long long)(64 * ka + cb2 + j) * H + o;
                u.theta[idx] = w2p[j]; u.adam_m[idx] = w2m[j]; u.adam_v[idx] = w2v[j];
            }
        }
    }
    __syncthreads();
    cluster_sync_all();
}

static size_t smem_bytes(int D) {
    return (size_t)NSLOT * SLOT_BYTES + sizeof(float) * 64 * ACC_LD + 4 * sizeof(float) * SliceMap(D).n +
           sizeof(float) * 8 * 64 * OUTP;
}

// 32 CTAs per network in clusters of 8 (the column blocks of one row block); `at` holds the cluster attribute
static cudaLaunchConfig_t cluster_launch(int n_nets, size_t smem, cudaStream_t s, cudaLaunchAttribute* at) {
    at->id = cudaLaunchAttributeClusterDimension;
    at->val.clusterDim.x = 8; at->val.clusterDim.y = 1; at->val.clusterDim.z = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(32 * n_nets); cfg.blockDim = dim3(TPB); cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cfg.attrs = at; cfg.numAttrs = 1;
    return cfg;
}

// The instantiation for world > 1 (dp) or a single GPU, with its dynamic shared memory opted in once for the largest D
// the gate admits, and how many of its clusters of 8 can be co-resident (0 if the opt-in fails).  The count is the same
// at every D: the shared memory of one CTA rules out a second on the same SM.
struct Instance {
    void (*kern)(const Args);
    int max_clusters;
};
static const Instance& instance(bool dp) {
    static Instance inst[2] = {};
    Instance& in = inst[dp];
    if (!in.kern) {
        in.kern = dp ? ppo_persist_kernel<true> : ppo_persist_kernel<false>;
        cudaLaunchAttribute at;
        const cudaLaunchConfig_t cfg = cluster_launch(1, smem_bytes(MAXD), nullptr, &at);
        if (cudaFuncSetAttribute(in.kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cfg.dynamicSmemBytes) != cudaSuccess ||
            cudaOccupancyMaxActiveClusters(&in.max_clusters, in.kern, &cfg) != cudaSuccess) {
            cudaGetLastError();
            in.max_clusters = 0;
        }
    }
    return in;
}

}  // namespace pp

size_t ppo_persist_ws_floats(int n_nets, int D, int H) {
    (void)D; (void)H;
    return (size_t)n_nets * pp::NET_WS + pp::SUMSQ_FLOATS + (size_t)(n_nets * pp::F_PER_NET + 1) * pp::FLAG_LINE + 32 +
           2 * (size_t)pp::MAX_MB + 2 * (size_t)32 * n_nets * pp::DBG_N;
}

size_t ppo_persist_p2p_floats(int n_nets) { return (size_t)(FSRL_P2P_MAX_RANKS + 1) * n_nets * pp::XG_PER_NET + 64; }

bool ppo_persist_supported(const fsrl_ppo_update_t& u, long long n_total, int batch_size) {
    if (u.H != 256 || batch_size != pp::MB || n_total % pp::MB != 0 || n_total < pp::MB || n_total / pp::MB > pp::MAX_MB) return false;
    if (u.world > 1 && !(u.p2p_on && u.world <= FSRL_P2P_MAX_RANKS && (size_t)u.p2p_stride >= ppo_persist_p2p_floats(u.n_nets))) return false;
    if (u.D < 1 || u.D > pp::MAXD || u.A > 8 || u.n_nets < 1 || u.n_nets > 3) return false;
    if (u.persist_ws == nullptr || (size_t)u.persist_ws_floats < ppo_persist_ws_floats(u.n_nets, u.D, u.H)) return false;
    if (32 * u.n_nets > sm_count()) return false;
    // the CTAs of a step wait for each other: every cluster of the grid must be resident at once
    return pp::instance(u.world > 1).max_clusters >= 4 * u.n_nets;
}

// ug: descriptor whose batch pointers are the gathered (contiguous) arrays; mb_stats filled.
int ppo_persist_run(const fsrl_ppo_update_t& ug, int n_mb, int stats_slot0, long long adam_t0, cudaStream_t s) {
    pp::Args a;
    a.u = ug;
    a.n_mb = n_mb; a.slot0 = stats_slot0; a.adam_t0 = adam_t0;
    a.ws = ug.persist_ws;
    const size_t fl_off = (size_t)ug.n_nets * pp::NET_WS + pp::SUMSQ_FLOATS;
    a.flags = reinterpret_cast<unsigned*>(ug.persist_ws + fl_off);
    const size_t n_flag_words = (size_t)(ug.n_nets * pp::F_PER_NET + 1) * pp::FLAG_LINE;
    a.err = reinterpret_cast<int*>(a.flags + n_flag_words);
    // the per-CTA sums of squares (slots no CTA writes read +0), the flag lines and the error word
    FSRL_CUDA(cudaMemsetAsync(ug.persist_ws + fl_off - pp::SUMSQ_FLOATS, 0, (pp::SUMSQ_FLOATS + n_flag_words + 32) * sizeof(float), s));
    // Adam bias corrections of every step, computed like torch.optim.Adam does (python doubles)
    float* tab_dev = reinterpret_cast<float*>(a.err + 32);
    static std::vector<float> tab;
    tab.resize(2 * (size_t)n_mb);
    for (int t = 0; t < n_mb; ++t) {
        const double tt = (double)(adam_t0 + t + 1);
        const double bc1 = 1.0 - pow(ug.beta1, tt), bc2 = 1.0 - pow(ug.beta2, tt);
        tab[2 * t] = (float)(1.0 / sqrt(bc2));
        tab[2 * t + 1] = (float)(-(ug.lr / bc1));
    }
    FSRL_CUDA(cudaMemcpyAsync(tab_dev, tab.data(), tab.size() * sizeof(float), cudaMemcpyHostToDevice, s));
    a.adam_tab = tab_dev;
    // tag of the exchange packets: ranks run their persistent launches in lock step, so the count agrees everywhere
    static unsigned dp_seq = 0;
    if (ug.world > 1) dp_seq = (dp_seq % 65535u) + 1u;
    a.dp_seq = dp_seq;
    a.dp_direct = ug.world <= 2;
    if (const char* e = getenv("FSRL_PPO_DP_DIRECT")) a.dp_direct = atoi(e) != 0;      // (experiments; must agree on all ranks)
    a.dbg = nullptr; a.dbg_step = -1;
    if (const char* e = getenv("FSRL_PPO_PERSIST_DBG")) {
        a.dbg = reinterpret_cast<long long*>(tab_dev + 2 * (size_t)pp::MAX_MB);
        a.dbg_step = atoi(e);
    }
    cudaLaunchAttribute at;
    const cudaLaunchConfig_t cfg = pp::cluster_launch(ug.n_nets, pp::smem_bytes(ug.D), s, &at);
    FSRL_CUDA(cudaLaunchKernelEx(&cfg, pp::instance(ug.world > 1).kern, a));
    ++g_launches;
    return FSRL_OK;
}

}  // namespace fsrl
