// sm_90a building blocks for the persistent PPO update (csrc/ppo_persist.cu): warpgroup tensor core
// MMAs (wgmma.mma_async kind tf32, accumulators in registers), bulk asynchronous copies (TMA unit,
// cp.async.bulk) completing on mbarriers, and the device-scope flag barriers that chain the
// CTAs of the persistent grid.  Inline PTX only -- no CUTLASS / CuTe dependency.
//
// Operand layout ("plane layout", no swizzle).  A matrix X[mn][k] of fp32 words is stored as
//       X_img[k / 4][mn][k % 4]            (planes of R rows x 16 bytes, R = MN extent of the block)
// which is the canonical K-major INTERLEAVE (no swizzle) layout of wgmma (CUTLASS cute/atom/mma_traits_sm90_gmma.hpp,
// make_gmma_desc): 8 x 16 B core matrices are 8 consecutive rows of one plane,
//         SBO (next 8 rows) = 128 B,   LBO (next 4 k = next plane) = 16 * R bytes,
// and one MMA instruction consumes K = 8 tf32 values = 2 planes.  wgmma reads tf32 operands K-major only, so an
// operand that is contracted over its other index is published by its producer as a second, transposed K-major image.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace fsrl {
namespace wg {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier ---------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// arrival on an mbarrier of any CTA of the cluster (shared::cluster address from mapa), default semantics (release at
// CTA scope).  Used to release a ring slot once wgmma.wait_group has retired the MMAs that read it; a cluster-scope
// release would add a fence to every arrival (on H100 it cost an earlier version of the persistent PPO kernel about
// 14 k cycles per minibatch step).
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_addr) {
    asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
// bounded wait: a barrier that never completes must not hang the GPU (returns false on timeout)
__device__ __forceinline__ bool mbar_wait(uint64_t* bar, uint32_t parity, long long timeout_cycles = 4000000000LL) {
    if (mbar_try_wait(bar, parity)) return true;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > timeout_cycles) return false;
    }
    return true;
}

// ---- bulk asynchronous copy global -> shared (TMA unit; SASS UBLKCP), completes on an mbarrier --
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
        ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// the same copy into the same shared-memory offset of every CTA of `cta_mask` (cluster ranks), each completing its
// bytes on the mbarrier at the same offset in that CTA
__device__ __forceinline__ void bulk_g2s_multicast(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar, uint16_t cta_mask) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;"
        ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)), "h"(cta_mask) : "memory");
}
// orders this thread's earlier generic-proxy operations on global memory (the acquire of a flag) before its later
// async-proxy operations (bulk copies reading what another SM wrote with ordinary stores).  Restricted to global
// memory: the unqualified fence.proxy.async also carries a GPU-scope memory barrier (MEMBAR.ALL.GPU in the SASS).
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
// orders this thread's earlier generic stores to shared memory before later async-proxy writes to the same bytes
// (scratch in the operand ring that the next phase's bulk copies overwrite)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- wgmma.mma_async kind tf32, operands from shared memory --------------------------------------
// shared-memory matrix descriptor, no swizzle (cute::GMMA::GmmaDescriptor: start >> 4 at [0,14), LBO >> 4 at [16,30),
// SBO >> 4 at [32,46), base offset 0, layout_type 0 = INTERLEAVE at [62,64))
__device__ __forceinline__ uint64_t smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((saddr >> 4) & 0x3fffu) | ((uint64_t)((lbo_bytes >> 4) & 0x3fffu) << 16) |
           ((uint64_t)((sbo_bytes >> 4) & 0x3fffu) << 32);
}
// D[64 x N] += A[64 x 8] B[N x 8]^T for the executing warpgroup, N = 32 or 64.  Fragment of thread (warp w of the
// warpgroup, lane l): d[4 i + e] = D[16 w + l / 4 + 8 (e >> 1)][8 i + 2 (l % 4) + (e & 1)],  i = 0 .. N / 8 - 1
__device__ __forceinline__ void mma_m64n32k8_tf32(float (&d)[16], uint64_t adesc, uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(adesc), "l"(bdesc), "n"(1));
}
__device__ __forceinline__ void mma_m64n64k8_tf32(float (&d)[32], uint64_t adesc, uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "n"(1));
}
// before the first wgmma that reads accumulator registers written by ordinary instructions
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// at most N committed groups of this warp still in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses to accumulator registers across wgmma_wait
template <int N>
__device__ __forceinline__ void reg_fence(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ---- device-scope flag barriers between the CTAs of a co-resident grid ---------------------------
__device__ __forceinline__ void flag_add_release(unsigned* ctr, unsigned v = 1u) {
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(ctr), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned flag_ld_acquire(const unsigned* ctr) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
    return v;
}
// spin until *ctr >= target; false after `timeout_cycles` (caller raises the error flag and leaves).  BACKOFF: sleep
// ~20 ns between polls, so that the pollers do not compete with the warps that share their scheduler and with the
// flag's L2 slice.
template <bool BACKOFF = true>
__device__ __forceinline__ bool flag_wait_ge(const unsigned* ctr, unsigned target, long long timeout_cycles = 4000000000LL) {
    if (flag_ld_acquire(ctr) >= target) return true;
    const long long t0 = clock64();
    while (flag_ld_acquire(ctr) < target) {
        if (clock64() - t0 > timeout_cycles) return false;
        if (BACKOFF) __nanosleep(20);
    }
    return true;
}

// fp32 -> (hi, lo) tf32 pair with the 13 low mantissa bits cleared (round to nearest, ties away):
// x ~= hi + lo to ~2^-22 relative; whatever the tensor core does with the low bits is irrelevant
__device__ __forceinline__ float tf32_round(float x) {
    return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u);
}
__device__ __forceinline__ void tf32_split(float x, float& hi, float& lo) {
    hi = tf32_round(x);
    lo = tf32_round(x - hi);
}

}  // namespace wg
}  // namespace fsrl
