// The reference's default 'concat_debug' video frames on sm_90a (real3d_infer.py:494-521; DESIGN.md, "Debug video"): each frame is a
// 512 x 2560 uint8 RGB strip of five 512^2 panels, source | driving SECC | raw render (x8 nearest) | clip-normalised depth (x8 nearest) | final.
//   debug_panels_kernel   one block per (row, panel, frame), 4 pixels per thread: panels 0, 1, 2 and 4 from fp32 inputs
//   depth_minmax_kernel   min and max of the clip's depth images as ordered-uint atomics (the encoding ray_limits_kernel uses)
//   depth_panel_kernel    panel 3 of every frame of the clip, from the reduced min and max
// The reference concatenates four float32 panels with one float64 panel (the SECC image comes back from numpy), so torch.cat promotes and
// the clamp and the ((x + 1) / 2 * 255).int() conversion of EVERY panel run in float64; every step here is spelled out with _rn intrinsics
// in the precision the reference computes it in, so that no contraction or reordering changes a byte.
#include "common.cuh"

namespace r3dp {
namespace debugf {

constexpr int kS = 512;                        // panel size
constexpr int kRes = 64;                       // the render's resolution: panels 2 and 3 replicate each pixel 8 x 8
constexpr int kPanelBytes = kS * 3;            // bytes of one panel row
constexpr int kRowBytes = 5 * kPanelBytes;     // bytes of one strip row
constexpr int kThreads = kS / 4;               // one block per panel row, 4 pixels per thread

// imgs.clamp(-1, 1) and ((x + 1) / 2 * 255).int().astype(np.uint8) in float64.  NaN survives the clamp and .int() makes it INT_MIN, whose
// low byte is 0.  After the clamp the value lies in [0, 255], where truncation toward zero is exact.
__device__ __forceinline__ unsigned to_byte(double x) {
    if (x != x) return 0u;
    x = x < -1.0 ? -1.0 : (x > 1.0 ? 1.0 : x);
    return (unsigned)__double2int_rz(__dmul_rn(__ddiv_rn(__dadd_rn(x, 1.0), 2.0), 255.0));
}

// panel 1: q = ((secc + 1) * 127.5).int() in float32 (real3d_infer.py:502), then q / 127.5 - 1 in float64 (:510)
__device__ __forceinline__ unsigned secc_byte(float s) {
    const int q = __float2int_rz(__fmul_rn(__fadd_rn(s, 1.f), 127.5f));
    return to_byte(__dsub_rn(__ddiv_rn((double)q, 127.5), 1.0));
}

// panel 3: ((d - mn) / (mx - mn)) * 2 - 1 in float32, clamped (:506-508); 0 / 0 (a constant clip) is NaN
__device__ __forceinline__ unsigned depth_byte(float d, float mn, float mx) {
    const float x = __fsub_rn(__fmul_rn(__fdiv_rn(__fsub_rn(d, mn), __fsub_rn(mx, mn)), 2.f), 1.f);
    return to_byte((double)x);
}

// 4 pixels x 3 channels -> 12 bytes at p: three 32-bit stores when the strip is 4-byte aligned, byte stores otherwise
template <bool kAligned>
__device__ __forceinline__ void store12(unsigned char* p, const unsigned (&b)[12]) {
    if (kAligned) {
        unsigned* w = reinterpret_cast<unsigned*>(p);
#pragma unroll
        for (int i = 0; i < 3; ++i) w[i] = b[4 * i] | (b[4 * i + 1] << 8) | (b[4 * i + 2] << 16) | (b[4 * i + 3] << 24);
    } else {
#pragma unroll
        for (int i = 0; i < 12; ++i) p[i] = (unsigned char)b[i];
    }
}

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }

// grid (512 rows, 4 panels: 0, 1, 2, 4, B frames).  ref_gt [3,512,512] (every frame), secc / image [B,3,512,512], feat [B,4096,C] with rgb in
// channels 0-2.  dst: byte 0 of frame 0's strip; frames frame_stride bytes apart, rows row_pitch bytes apart
template <bool kAligned>
__global__ void __launch_bounds__(kThreads) debug_panels_kernel(const float* __restrict__ ref_gt, const float* __restrict__ secc,
                                                                const float* __restrict__ feat, int C, const float* __restrict__ image,
                                                                unsigned char* __restrict__ dst, long long frame_stride, long long row_pitch) {
    const int y = blockIdx.x, b = blockIdx.z, x = threadIdx.x * 4;
    const int panel = blockIdx.y < 3 ? blockIdx.y : 4;
    const size_t plane = (size_t)kS * kS, pix = (size_t)y * kS + x;
    unsigned v[12];
    if (panel == 2) {
        // F.interpolate(imgs_raw, (512, 512)) nearest: source pixel dst // 8, the same for all 4 pixels of the thread
        const float* f = feat + ((size_t)b * kRes * kRes + (size_t)(y >> 3) * kRes + (x >> 3)) * C;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const unsigned u = to_byte((double)f[c]);          // image_raw's float32 clamp is exact, so the float64 clamp covers it
#pragma unroll
            for (int i = 0; i < 4; ++i) v[3 * i + c] = u;
        }
    } else {
        const float* src = panel == 0 ? ref_gt : panel == 1 ? secc + (size_t)b * 3 * plane : image + (size_t)b * 3 * plane;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float4 q = ld4(src + c * plane + pix);
            const float a[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) v[3 * i + c] = panel == 1 ? secc_byte(a[i]) : to_byte((double)a[i]);
        }
    }
    store12<kAligned>(dst + b * frame_stride + y * row_pitch + panel * kPanelBytes + x * 3, v);
}

// minmax[0] / [1]: f2ord of the min / max over n floats (initialised to 0xffffffff / 0 by the caller).  Ordered uints keep NaN: a NaN
// encodes above +inf or below -inf, so it reaches the max or the min, and every pixel of panel 3 becomes NaN, as torch's min / max make it.
__global__ void __launch_bounds__(256) depth_minmax_kernel(const float* __restrict__ depth, long long n, unsigned* __restrict__ minmax) {
    unsigned lo = 0xffffffffu, hi = 0u;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const unsigned u = f2ord(depth[i]);
        lo = min(lo, u);
        hi = max(hi, u);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
        hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    }
    __shared__ unsigned s_lo[8], s_hi[8];
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) { s_lo[w] = lo; s_hi[w] = hi; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int i = 1; i < (int)(blockDim.x >> 5); ++i) { lo = min(lo, s_lo[i]); hi = max(hi, s_hi[i]); }
        atomicMin(minmax, lo);
        atomicMax(minmax + 1, hi);
    }
}

// grid (512 rows, F frames).  depth [F,64,64]; the one channel is repeated three times
template <bool kAligned>
__global__ void __launch_bounds__(kThreads) depth_panel_kernel(const float* __restrict__ depth, const unsigned* __restrict__ minmax,
                                                               unsigned char* __restrict__ dst, long long frame_stride, long long row_pitch) {
    const int y = blockIdx.x, f = blockIdx.y, x = threadIdx.x * 4;
    const float mn = ord2f(minmax[0]), mx = ord2f(minmax[1]);
    const unsigned u = depth_byte(depth[(size_t)f * kRes * kRes + (size_t)(y >> 3) * kRes + (x >> 3)], mn, mx);
    unsigned v[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) v[i] = u;
    store12<kAligned>(dst + f * frame_stride + y * row_pitch + 3 * kPanelBytes + x * 3, v);
}

inline bool aligned4(const void* p, long long a, long long b) { return (((uintptr_t)p | (uintptr_t)a | (uintptr_t)b) & 3u) == 0; }

}  // namespace debugf
}  // namespace r3dp

using namespace r3dp;
using namespace r3dp::debugf;

extern "C" int r3dp_debug_panels(const float* ref_gt, const float* secc, const float* feat, int feat_c, const float* image, int B,
                                 unsigned char* dst, long long frame_stride, long long row_pitch, r3dp_stream_t stream) {
    R3DP_REQUIRE(ref_gt && secc && feat && image && dst, "debug_panels: null pointer");
    R3DP_REQUIRE(B >= 1 && B <= 65535, "debug_panels: need 1 <= B <= 65535, got %d", B);
    R3DP_REQUIRE(feat_c >= 3, "debug_panels: the render's features need at least 3 channels, got %d", feat_c);
    R3DP_REQUIRE(row_pitch >= kRowBytes && (B == 1 || frame_stride >= kS * row_pitch),
                 "debug_panels: row_pitch must be >= %d bytes and frame_stride >= 512 rows", kRowBytes);
    R3DP_REQUIRE(((uintptr_t)ref_gt | (uintptr_t)secc | (uintptr_t)image) % 16 == 0, "debug_panels: ref_gt, secc and image must be 16-byte aligned");
    const dim3 grid(kS, 4, B);
    if (aligned4(dst, frame_stride, row_pitch))
        debug_panels_kernel<true><<<grid, kThreads, 0, as_stream(stream)>>>(ref_gt, secc, feat, feat_c, image, dst, frame_stride, row_pitch);
    else
        debug_panels_kernel<false><<<grid, kThreads, 0, as_stream(stream)>>>(ref_gt, secc, feat, feat_c, image, dst, frame_stride, row_pitch);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_debug_depth_panel(const float* depth, int F, unsigned* minmax, unsigned char* dst, long long frame_stride, long long row_pitch,
                                      r3dp_stream_t stream) {
    R3DP_REQUIRE(depth && minmax && dst, "debug_depth_panel: null pointer");
    R3DP_REQUIRE(F >= 1 && F <= 65535, "debug_depth_panel: need 1 <= F <= 65535, got %d", F);
    R3DP_REQUIRE(row_pitch >= kRowBytes && (F == 1 || frame_stride >= kS * row_pitch),
                 "debug_depth_panel: row_pitch must be >= %d bytes and frame_stride >= 512 rows", kRowBytes);
    cudaStream_t st = as_stream(stream);
    R3DP_CUDA(cudaMemsetAsync(minmax, 0xff, sizeof(unsigned), st));
    R3DP_CUDA(cudaMemsetAsync(minmax + 1, 0, sizeof(unsigned), st));
    const long long n = (long long)F * kRes * kRes;
    const long long want = (n + 255) / 256, cap = 4LL * sm_count();
    const unsigned grid = (unsigned)(want < cap ? want : cap);
    depth_minmax_kernel<<<grid, 256, 0, st>>>(depth, n, minmax);
    R3DP_LAUNCH_CHECK();
    if (aligned4(dst, frame_stride, row_pitch))
        depth_panel_kernel<true><<<dim3(kS, F), kThreads, 0, st>>>(depth, minmax, dst, frame_stride, row_pitch);
    else
        depth_panel_kernel<false><<<dim3(kS, F), kThreads, 0, st>>>(depth, minmax, dst, frame_stride, row_pitch);
    R3DP_LAUNCH_CHECK();
    count_launches(2);
    return 0;
}
