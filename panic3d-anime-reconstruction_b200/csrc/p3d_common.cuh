// Shared device/host helpers for the p3d CUDA library (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <math.h>
#include <atomic>
#include <string>

#include "../../include/p3d_render.h"

namespace p3d {

// ---------------------------------------------------------------- errors
void set_error(const char* fmt, ...);
extern std::atomic<uint64_t> g_launches;
inline void count_launch(int n = 1) { g_launches.fetch_add((uint64_t)n, std::memory_order_relaxed); }

#define P3D_CUDA_TRY(expr)                                                                   \
    do {                                                                                     \
        cudaError_t _e = (expr);                                                             \
        if (_e != cudaSuccess) {                                                             \
            ::p3d::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return P3D_ECUDA;                                                                \
        }                                                                                    \
    } while (0)

#define P3D_REQUIRE(cond, ...)                                                               \
    do {                                                                                     \
        if (!(cond)) {                                                                       \
            ::p3d::set_error(__VA_ARGS__);                                                   \
            return P3D_EINVAL;                                                               \
        }                                                                                    \
    } while (0)

// Optional per-kernel device timing (bench.py's roofline leg): when enabled, launch sites bracket
// their kernel with CUDA events on the launching stream; p3d_profile_read() sums them per slot.
enum ProfileSlot { PROF_SAMPLE_DECODE = 0, PROF_IMPORTANCE = 1, PROF_COMPOSITE = 2, PROF_LAYOUT = 3, PROF_RAYGEN = 4,
                   PROF_FUSED = 5, PROF_OTHER = 6, PROF_MODCONV = 7, PROF_SLOTS = 8 };
bool profile_enabled();
void profile_begin(int slot, cudaStream_t stream);
void profile_end(int slot, cudaStream_t stream);
struct ProfileScope {
    int slot; cudaStream_t st; bool on;
    ProfileScope(int s, cudaStream_t stream) : slot(s), st(stream), on(profile_enabled()) { if (on) profile_begin(slot, st); }
    ~ProfileScope() { if (on) profile_end(slot, st); }
};

#define P3D_LAUNCH_CHECK()                                                                   \
    do {                                                                                     \
        ::p3d::count_launch();                                                               \
        P3D_CUDA_TRY(cudaGetLastError());                                                    \
    } while (0)

// ---------------------------------------------------------------- math (torch semantics)
// F.softplus(beta=1, threshold=20): x if x > 20 else log1p(exp(x))
__device__ __forceinline__ float softplus_t(float x) { return x > 20.f ? x : log1pf(expf(x)); }
__device__ __forceinline__ float sigmoid_t(float x) { return 1.f / (1.f + expf(-x)); }

// MUFU-based fast math (1 instruction each; ftz).  ex2/lg2: rel/abs error ~2^-22.
__device__ __forceinline__ float ex2_approx(float x) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float lg2_approx(float x) { float r; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float rcp_approx(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
// softplus in base 2: log2(1 + 2^x); equals x beyond the torch threshold (20 nats) to fp32 precision
__device__ __forceinline__ float softplus2(float x2) { return x2 > 28.853900817779268f ? x2 : lg2_approx(1.f + ex2_approx(x2)); }
// natural softplus through the base-2 one
__device__ __forceinline__ float softplus_mufu(float x) { return 0.6931471805599453f * softplus2(1.4426950408889634f * x); }

// Order-preserving float <-> uint mapping for atomicMin/Max on floats of either sign.
__device__ __forceinline__ unsigned int float_to_ordered(float f) {
    unsigned int u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float ordered_to_float(unsigned int u) {
    unsigned int v = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
#ifdef __CUDA_ARCH__
    return __uint_as_float(v);
#else
    float f;
    memcpy(&f, &v, 4);
    return f;
#endif
}

// ---------------------------------------------------------------- Philox4x32-10 (Salmon et al. 2011)
struct Philox4 {
    unsigned int x, y, z, w;
};
__device__ __forceinline__ Philox4 philox4x32_10(uint64_t seed, uint64_t counter, unsigned int stream) {
    unsigned int k0 = (unsigned int)seed, k1 = (unsigned int)(seed >> 32);
    unsigned int c0 = (unsigned int)counter, c1 = (unsigned int)(counter >> 32), c2 = stream, c3 = 0x1BD11BDAu;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        unsigned int hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        unsigned int hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        unsigned int n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    return Philox4{c0, c1, c2, c3};
}
// uniform in [0,1) with 24 random bits (same support as torch.rand for fp32)
__device__ __forceinline__ float u01(unsigned int bits) { return (float)(bits >> 8) * (1.0f / 16777216.0f); }
__device__ __forceinline__ float philox_uniform(uint64_t seed, uint64_t index, unsigned int stream) {
    Philox4 r = philox4x32_10(seed, index >> 2, stream);
    unsigned int v = (index & 3) == 0 ? r.x : (index & 3) == 1 ? r.y : (index & 3) == 2 ? r.z : r.w;
    return u01(v);
}

// ---------------------------------------------------------------- warp helpers
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// inclusive scans across the 32 lanes
__device__ __forceinline__ float warp_scan_add(float v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        float t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += t;
    }
    return v;
}
__device__ __forceinline__ float warp_scan_mul(float v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        float t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v *= t;
    }
    return v;
}

// 128-bit read-only global load
__device__ __forceinline__ float4 ldg128(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

}  // namespace p3d
