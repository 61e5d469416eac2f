// Shared helpers for libr3dp_b200 (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include "../../include/r3dp_b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libr3dp_b200 is written for sm_90a (H100) only"
#endif

namespace r3dp {

// ---- error plumbing -------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
inline int fail(const char* msg) { set_error("%s", msg); return 1; }

#define R3DP_REQUIRE(cond, ...)                       \
    do {                                              \
        if (!(cond)) {                                \
            ::r3dp::set_error(__VA_ARGS__);           \
            return 1;                                 \
        }                                             \
    } while (0)

#define R3DP_CUDA(expr)                                                                            \
    do {                                                                                           \
        cudaError_t _e = (expr);                                                                   \
        if (_e != cudaSuccess) {                                                                   \
            ::r3dp::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return 1;                                                                              \
        }                                                                                          \
    } while (0)

// every API function calls this once per kernel it enqueued; r3dp_launch_count() reports the running total
void count_launches(int n);
#define R3DP_LAUNCH_CHECK() R3DP_CUDA(cudaGetLastError())

inline cudaStream_t as_stream(r3dp_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }
int sm_count();

// ---- device helpers -------------------------------------------------------------------------------------------
// Order-preserving float <-> uint32 map so that float min/max can use integer atomics (handles negatives).
__device__ __forceinline__ unsigned f2ord(float f) {
    unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned u) {
    return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

__device__ __forceinline__ float4 ldg_nc_f4(const float* p) {
    float4 r;
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
// streaming (evict-first) 128-bit store: output that is never re-read must not displace the planes in L2
__device__ __forceinline__ void stg_cs_f4(float* p, float4 v) {
    asm volatile("st.global.cs.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// torch.nn.Softplus(beta=1, threshold=20) with MUFU ex2/lg2: |err| < 2e-7 absolute on the whole range
__device__ __forceinline__ float softplus_fast(float x) {
    float e = exp2f(x * 1.4426950408889634f);          // ex2.approx (compiled with -use_fast_math off: exp2f is still MUFU-based, <=2 ulp)
    float r = 0.6931471805599453f * __log2f(1.0f + e);
    return x > 20.0f ? x : r;
}
__device__ __forceinline__ float sigmoid_fast(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }

__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

}  // namespace r3dp
