// Shared device/host helpers for the fsrl_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace fsrl {

// ---- error plumbing for the C-ABI (thread-local message, int return codes) ----------
void set_error(const char* fmt, ...);
#define FSRL_OK 0
#define FSRL_EINVAL (-1)
#define FSRL_ECUDA (-2)
#define FSRL_EWORKSPACE (-3)

#define FSRL_REQUIRE(cond, ...)                                                        \
    do {                                                                               \
        if (!(cond)) {                                                                 \
            ::fsrl::set_error(__VA_ARGS__);                                            \
            return FSRL_EINVAL;                                                        \
        }                                                                              \
    } while (0)

#define FSRL_CUDA(call)                                                                \
    do {                                                                               \
        cudaError_t e__ = (call);                                                      \
        if (e__ != cudaSuccess) {                                                      \
            ::fsrl::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #call,             \
                              cudaGetErrorString(e__));                                \
            return FSRL_ECUDA;                                                         \
        }                                                                              \
    } while (0)

#define FSRL_LAUNCH_CHECK()                                                            \
    do {                                                                               \
        ++::fsrl::g_launches;                                                          \
        cudaError_t e__ = cudaGetLastError();                                          \
        if (e__ != cudaSuccess) {                                                      \
            ::fsrl::set_error("%s:%d kernel launch -> %s", __FILE__, __LINE__,         \
                              cudaGetErrorString(e__));                                \
            return FSRL_ECUDA;                                                         \
        }                                                                              \
    } while (0)

extern unsigned long long g_launches;  // kernels launched by this library (host-side count)

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

int sm_count();  // cached cudaDevAttrMultiProcessorCount of the current device (132 on an H100 SXM)

// ---- device helpers -------------------------------------------------------------------
__device__ __forceinline__ double shfl_up_f64(double v, int d) {
    return __shfl_up_sync(0xffffffffu, v, d);
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Sum over a block of NWARPS warps, returned to every thread: warp sums, then the warp partials
// added in warp order.  red holds NWARPS values; the leading barrier lets a caller reuse it.
template <int NWARPS, class T>
__device__ __forceinline__ T block_sum(T v, T* red) {
    v = warp_sum(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    T t = 0;
#pragma unroll
    for (int i = 0; i < NWARPS; ++i) t += red[i];
    return t;
}

constexpr float LOG_SQRT_2PI = 0.9189385332046727f;   // log(sqrt(2 pi)) of the Gaussian log-density

// streaming (read-once) loads: keep them out of L1
__device__ __forceinline__ float4 ldg_stream4(const float* p) {
    return __ldcs(reinterpret_cast<const float4*>(p));
}
__device__ __forceinline__ void stg_stream4(float* p, float4 v) {
    __stcs(reinterpret_cast<float4*>(p), v);
}

// ---- Philox4x32-10 counter RNG (documented stream; CPU twin in oracle/philox.py) -------
struct Philox {
    static constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
    static constexpr uint32_t W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
    __host__ __device__ static inline void round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
        uint64_t p0 = (uint64_t)M0 * c[0];
        uint64_t p1 = (uint64_t)M1 * c[2];
        uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0;
        uint32_t hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
        uint32_t n0 = hi1 ^ c[1] ^ k0;
        uint32_t n1 = lo1;
        uint32_t n2 = hi0 ^ c[3] ^ k1;
        uint32_t n3 = lo0;
        c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
    }
    // counter = (c0,c1,c2,c3), key = (k0,k1) -> 4 x u32
    __host__ __device__ static inline void gen(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                               uint32_t k0, uint32_t k1, uint32_t (&out)[4]) {
        uint32_t c[4] = {c0, c1, c2, c3};
#pragma unroll
        for (int i = 0; i < 10; ++i) {
            round(c, k0, k1);
            k0 += W0;
            k1 += W1;
        }
        out[0] = c[0]; out[1] = c[1]; out[2] = c[2]; out[3] = c[3];
    }
};

// Box-Muller in f64 from two Philox words (CPU twin: oracle/philox.py normal_pair)
__device__ __forceinline__ void gauss_pair(uint32_t a, uint32_t b, float& n0, float& n1) {
    const double u1 = ((double)a + 1.0) * (1.0 / 4294967296.0);
    const double u2 = (double)b * (1.0 / 4294967296.0);
    const double r = sqrt(-2.0 * log(u1));
    const double ang = 2.0 * 3.141592653589793 * u2;
    n0 = (float)(r * cos(ang));
    n1 = (float)(r * sin(ang));
}

// u32 -> uniform in (0,1]: (x + 1) * 2^-32 computed in f32 via the 24 top bits
__host__ __device__ inline float u01(uint32_t x) {
    return ((float)(x >> 8) + 1.0f) * (1.0f / 16777216.0f);
}

}  // namespace fsrl
