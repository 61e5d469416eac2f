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

// Bilinear up-resize (F.interpolate, align_corners=False; antialias is the identity for scale >= 1).  Every resize kernel goes through
// these two helpers.  The multiply-adds are spelled out with intrinsics: left to the compiler, `a * (1 - t) + b * t` is contracted into
// fma(a, 1 - t, b * t) in one kernel and fma(b, t, a * (1 - t)) in another, and two kernels that must agree bit for bit would not.
// bilinear_coord: output index o of an n -> size resize -> source indices i0, i1 and weight t of i1.
__device__ __forceinline__ void bilinear_coord(int o, int n, int size, int& i0, int& i1, float& t) {
    const float s = fmaxf(__fmaf_rn((float)o + 0.5f, (float)n / (float)size, -0.5f), 0.f);
    i0 = min((int)s, n - 1);
    i1 = min(i0 + 1, n - 1);
    t = s - (float)i0;
}
// a<row><col>: the four source values at (y0,x0), (y1,x0), (y0,x1), (y1,x1)
__device__ __forceinline__ float bilinear_mix(float a00, float a10, float a01, float a11, float ty, float tx) {
    const float r0 = __fmaf_rn(a00, 1.f - ty, __fmul_rn(a10, ty));
    const float r1 = __fmaf_rn(a01, 1.f - ty, __fmul_rn(a11, ty));
    return __fmaf_rn(r0, 1.f - tx, __fmul_rn(r1, tx));
}

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
