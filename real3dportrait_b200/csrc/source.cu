// Source images on sm_90a: the torso head's per-clip images (ref_head_img, ref_torso_img, bg_img) from the source image and its segmap,
// as real3d_infer.py:243-260 builds them with _seg_out_img_with_segmap, inpaint_torso_job and extract_background (DESIGN.md, "Source images").
//   src_inpaint_kernel   one warp per column: the column's head / neck / torso bits by ballot (32 words, H <= 1024), the vertical 3-row
//                        dilation of the neck on those words, the top torso and top dilated-neck rows and the dilated-neck count, then every
//                        pixel of the column once: head zeroed, torso (9 rows) and neck (53 rows) darkened copies with numpy's index wrap,
//                        neck after torso -> img2 (uint8 HWC) and a flag byte (1: kept in torso_img, 2: neck-inpainted, i.e. blurred)
//   src_compose_kernel   one thread per pixel: cv2's 5x5 GaussianBlur(sigma 4) at neck-inpainted pixels as its exact integer form, the torso
//                        mask, and the float32 NCHW ((u - 127.5) / 127.5) of ref_torso_img and ref_head_img
//   edt_cols_kernel      exact squared EDT, phase 1: one thread per (column, frame), the signed row offset to the column's nearest source
//                        (the upper one on a tie); sources are a frame's non-bg pixels (s0 == 0) or the pixels with max d^2 > 100
//   edt_max_kernel       phase 2 for the selected frames: one block per row, the row's offsets in shared memory, every pixel's
//                        min_u (x - u)^2 + g(u)^2 by an outward search that stops once (x - u)^2 exceeds the best; frames in order within
//                        the block, so the running max and its first argmax need no atomics
//   edt_fill_kernel      phase 2 over the d^2 > 100 set with the feature (nearest source; ties: smallest column, then smallest row) and
//                        the colour gather: bg = frame argmax[f] at f = nearest source of the pixel (the pixel itself when it is a source)
#include "common.cuh"
#include <stdint.h>

namespace r3dp {
namespace source {

constexpr int kMinSize = 64, kMaxSize = 1024;     // H <= 1024: a column's bits fit 32 words of 32; W <= 1024: a row fits shared memory
constexpr int kTorsoRows = 9, kNeckRows = 53;      // inpaint_torso_job: L = 8 + 1 and 48 + push_down + 1
constexpr int kPushDown = 4;
constexpr short kNone = 0x7fff;                    // no source in the column
constexpr int kInfD2 = 1 << 30;
constexpr int kRowThreads = 256;
constexpr unsigned kFull = 0xffffffffu;

inline unsigned blocks(long long n, int t) { return (unsigned)((n + t - 1) / t); }

template <typename T>
__device__ __forceinline__ float segv(const T* seg, long long plane, int ch, long long p) { return (float)seg[ch * plane + p]; }

// (s1 + s3 + s5) in float32, in that order (inpaint_torso_job's head mask tests != 0, _seg_out_img_with_segmap's > 0.5)
template <typename T>
__device__ __forceinline__ float head_sum(const T* seg, long long plane, long long p) {
    return __fadd_rn(__fadd_rn(segv(seg, plane, 1, p), segv(seg, plane, 3, p)), segv(seg, plane, 5, p));
}

__device__ __forceinline__ unsigned char darken(unsigned char v, double s) { return (unsigned char)__double2int_rz(__dmul_rn((double)v, s)); }

__device__ __forceinline__ float normalise(unsigned char v) { return __fdiv_rn(__fsub_rn((float)v, 127.5f), 127.5f); }

// ---- inpaint_torso_job up to the blur ---------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) src_inpaint_kernel(const unsigned char* __restrict__ img, const T* __restrict__ seg, int H, int W,
                                                          const double* __restrict__ tab_torso, const double* __restrict__ tab_neck,
                                                          unsigned char* __restrict__ img2, unsigned char* __restrict__ flags) {
    const int lane = threadIdx.x, c = blockIdx.x * blockDim.y + threadIdx.y;
    if (c >= W) return;                            // whole warps leave together
    const long long plane = (long long)H * W;
    const int nwords = (H + 31) >> 5;
    unsigned hw = 0, nw = 0, tw = 0;               // word `lane` (rows 32 lane ..) of the head, neck and torso bits
    for (int j = 0; j < nwords; ++j) {
        const int r = 32 * j + lane;
        bool h = false, n = false, t = false;
        if (r < H) {
            const long long p = (long long)r * W + c;
            h = head_sum(seg, plane, p) != 0.f;
            n = segv(seg, plane, 2, p) != 0.f;
            t = segv(seg, plane, 4, p) != 0.f;
        }
        const unsigned bh = __ballot_sync(kFull, h), bn = __ballot_sync(kFull, n), bt = __ballot_sync(kFull, t);
        if (lane == j) { hw = bh; nw = bn; tw = bt; }
    }
    // binary_dilation with a vertical [1,1,1] structure, iterations=3, zero border = OR of the neck bits of rows r-3 .. r+3
    const unsigned prev = __shfl_up_sync(kFull, nw, 1), next = __shfl_down_sync(kFull, nw, 1);
    const unsigned below = lane == 0 ? 0u : prev, above = lane == 31 ? 0u : next;
    unsigned dw = nw;
#pragma unroll
    for (int d = 1; d <= 3; ++d) dw |= (nw >> d) | (above << (32 - d)) | (nw << d) | (below >> (32 - d));
    const int valid = H - 32 * lane;               // rows of this word inside the image
    dw = valid >= 32 ? dw : valid <= 0 ? 0u : dw & ((1u << valid) - 1u);
    const int n_dil = __reduce_add_sync(kFull, __popc(dw));
    // the column's top dilated-neck and torso rows; H when it has none
    const int top_dil = (int)__reduce_min_sync(kFull, dw ? (unsigned)(32 * lane + __ffs(dw) - 1) : (unsigned)H);
    const int top_torso = (int)__reduce_min_sync(kFull, tw ? (unsigned)(32 * lane + __ffs(tw) - 1) : (unsigned)H);
    auto bit = [&](unsigned word, int r) { return (__shfl_sync(kFull, word, r >> 5) >> (r & 31)) & 1u; };
    // the top pixel is kept when the pixel above it (numpy's wrap: row -1 is row H-1) is head
    const bool torso_on = top_torso < H && bit(hw, (top_torso + H - 1) % H);
    const bool neck_on = top_dil < H && bit(hw, (top_dil + H - 1) % H);
    const int anchor = neck_on ? top_dil + min(n_dil - 1, kPushDown) : 0;
    unsigned char tc[3] = {0, 0, 0}, nc[3] = {0, 0, 0};
    for (int ch = 0; ch < 3; ++ch) {
        if (torso_on) tc[ch] = img[((long long)top_torso * W + c) * 3 + ch];
        if (neck_on) nc[ch] = img[((long long)anchor * W + c) * 3 + ch];
    }
    for (int j = 0; j < nwords; ++j) {
        const int r = 32 * j + lane;
        const unsigned h = bit(hw, min(r, H - 1)), t = bit(tw, min(r, H - 1)), d = bit(dw, min(r, H - 1));
        if (r >= H) continue;
        const long long p = (long long)r * W + c;
        const int kn = (anchor - r + H) % H, kt = (top_torso - r + H) % H;
        const bool in_neck = neck_on && kn < kNeckRows, in_torso = torso_on && kt < kTorsoRows;
        unsigned char o[3];
        for (int ch = 0; ch < 3; ++ch)
            o[ch] = in_neck ? darken(nc[ch], tab_neck[kn]) : in_torso ? darken(tc[ch], tab_torso[kt]) : h ? 0 : img[p * 3 + ch];
        for (int ch = 0; ch < 3; ++ch) img2[p * 3 + ch] = o[ch];
        flags[p] = (unsigned char)(((d | t) || in_neck || in_torso ? 1 : 0) | (in_neck ? 2 : 0));
    }
}

// ---- blur at the neck-inpainted pixels, torso mask, normalised outputs ----------------------------------------------------------------
__device__ __forceinline__ int reflect101(int i, int n) { return i < 0 ? -i : i >= n ? 2 * n - 2 - i : i; }

template <typename T>
__global__ void __launch_bounds__(256) src_compose_kernel(const unsigned char* __restrict__ img, const T* __restrict__ seg,
                                                          const unsigned char* __restrict__ img2, const unsigned char* __restrict__ flags,
                                                          int H, int W, float* __restrict__ head_f32, float* __restrict__ torso_f32,
                                                          unsigned char* __restrict__ torso_u8) {
    const long long plane = (long long)H * W;
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= plane) return;
    const int r = (int)(p / W), c = (int)(p - (long long)r * W);
    const int f = flags[p];
    unsigned char t[3];
    if (!(f & 1)) {
        t[0] = t[1] = t[2] = 0;
    } else if (f & 2) {                            // cv2.GaussianBlur(img, (5, 5), sigmaX=4) on uint8: integer taps, one rounding
        const int w5[5] = {48, 53, 54, 53, 48};
        int acc[3] = {0, 0, 0};
        for (int dy = 0; dy < 5; ++dy) {
            const long long row = (long long)reflect101(r + dy - 2, H) * W;
            int a[3] = {0, 0, 0};
            for (int dx = 0; dx < 5; ++dx) {
                const unsigned char* q = img2 + (row + reflect101(c + dx - 2, W)) * 3;
                for (int ch = 0; ch < 3; ++ch) a[ch] += w5[dx] * q[ch];
            }
            for (int ch = 0; ch < 3; ++ch) acc[ch] += w5[dy] * a[ch];
        }
        for (int ch = 0; ch < 3; ++ch) t[ch] = (unsigned char)((acc[ch] + (1 << 15)) >> 16);
    } else {
        for (int ch = 0; ch < 3; ++ch) t[ch] = img2[p * 3 + ch];
    }
    if (torso_f32)
        for (int ch = 0; ch < 3; ++ch) torso_f32[ch * plane + p] = normalise(t[ch]);
    if (torso_u8)
        for (int ch = 0; ch < 3; ++ch) torso_u8[p * 3 + ch] = t[ch];
    if (head_f32) {
        const bool head = head_sum(seg, plane, p) > 0.5f;
        for (int ch = 0; ch < 3; ++ch) head_f32[ch * plane + p] = normalise(head ? img[p * 3 + ch] : (unsigned char)0);
    }
}

// ---- exact squared EDT --------------------------------------------------------------------------------------------------------------
// phase 1: g[f][r][c] = (row of the column's nearest source) - r, the upper source on a tie; kNone when the column has none.  mode 0: the
// sources of frame f are its pixels with seg[f][0] == 0, and has_src[f] = 1 when any column has one; mode 1: the pixels with maxd2 > 100,
// and has_src[0] = 1 + the raster index of the last of them (0: none).
template <typename T>
__global__ void __launch_bounds__(128) edt_cols_kernel(const T* __restrict__ seg, long long seg_stride, const int* __restrict__ maxd2, int mode,
                                                       int H, int W, short* __restrict__ g, int* __restrict__ has_src) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x, f = blockIdx.y;
    if (c >= W) return;
    const T* s = seg ? seg + f * seg_stride : nullptr;
    short* gf = g + (long long)f * H * W;
    auto src = [&](int r) { return mode == 0 ? (float)s[(long long)r * W + c] == 0.f : maxd2[(long long)r * W + c] > 100; };
    int last = -1;
    for (int r = 0; r < H; ++r) {
        if (src(r)) last = r;
        gf[(long long)r * W + c] = last < 0 ? kNone : (short)(last - r);
    }
    if (last >= 0) {                               // mode 1: has_src = 1 + the last source pixel in raster order (see edt_fill_kernel)
        if (mode == 0) has_src[f] = 1;
        else atomicMax(has_src, last * W + c + 1);
    }
    int nxt = -1;
    for (int r = H - 1; r >= 0; --r) {
        if (src(r)) nxt = r;
        const short up = gf[(long long)r * W + c];
        const bool use_up = up != kNone && (nxt < 0 || -up <= nxt - r);
        gf[(long long)r * W + c] = use_up ? up : nxt < 0 ? kNone : (short)(nxt - r);
    }
}

__device__ __forceinline__ int col_d2(short g) { return g == kNone ? kInfD2 : (int)g * g; }

// phase 2 for the selected frames f0 .. f0+n-1 of a chunk: running max of d^2 over frames and the first frame attaining it
__global__ void __launch_bounds__(kRowThreads) edt_max_kernel(const short* __restrict__ g, int H, int W, int f0, int n, int* __restrict__ maxd2,
                                                              int* __restrict__ argmax) {
    __shared__ int d2[kMaxSize];
    constexpr int kPer = kMaxSize / kRowThreads;
    const int r = blockIdx.x;
    int best[kPer], arg[kPer];
#pragma unroll
    for (int i = 0; i < kPer; ++i) {
        const int x = threadIdx.x + i * kRowThreads;
        best[i] = -1;
        arg[i] = 0;
        if (f0 > 0 && x < W) {
            best[i] = maxd2[(long long)r * W + x];
            arg[i] = argmax[(long long)r * W + x];
        }
    }
    for (int f = 0; f < n; ++f) {
        __syncthreads();
        for (int u = threadIdx.x; u < W; u += kRowThreads) d2[u] = col_d2(g[((long long)f * H + r) * W + u]);
        __syncthreads();
#pragma unroll
        for (int i = 0; i < kPer; ++i) {
            const int x = threadIdx.x + i * kRowThreads;
            if (x >= W) continue;
            int m = kInfD2;
            for (int k = 0; k * k <= m && (x - k >= 0 || x + k < W); ++k) {
                if (x - k >= 0) m = min(m, k * k + d2[x - k]);
                if (x + k < W) m = min(m, k * k + d2[x + k]);
            }
            if (m > best[i]) { best[i] = m; arg[i] = f0 + f; }
        }
    }
#pragma unroll
    for (int i = 0; i < kPer; ++i) {
        const int x = threadIdx.x + i * kRowThreads;
        if (x < W) {
            maxd2[(long long)r * W + x] = best[i];
            argmax[(long long)r * W + x] = arg[i];
        }
    }
}

// phase 2 over the d^2 > 100 set: each pixel's nearest source (smallest column, then smallest row, among the nearest) and its colour
__global__ void __launch_bounds__(kRowThreads) edt_fill_kernel(const short* __restrict__ g, const int* __restrict__ argmax,
                                                               const int* __restrict__ last_bc, const unsigned char* __restrict__ frames,
                                                               long long frame_stride, int H, int W, unsigned char* __restrict__ bg_u8,
                                                               float* __restrict__ bg_f32) {
    __shared__ int d2[kMaxSize];
    __shared__ short off[kMaxSize];
    const int r = blockIdx.x;
    for (int u = threadIdx.x; u < W; u += kRowThreads) {
        const short o = g[(long long)r * W + u];
        off[u] = o;
        d2[u] = col_d2(o);
    }
    __syncthreads();
    const long long plane = (long long)H * W;
    for (int x = threadIdx.x; x < W; x += kRowThreads) {
        int m = kInfD2, bu = -1;
        for (int k = 0; k * k <= m && (x - k >= 0 || x + k < W); ++k) {
            const int lo = x - k, hi = x + k;
            if (lo >= 0) {
                const int v = k * k + d2[lo];
                if (v < m || (v == m && lo < bu)) { m = v; bu = lo; }
            }
            if (hi < W && k > 0) {
                const int v = k * k + d2[hi];
                if (v < m) { m = v; bu = hi; }       // a tie keeps the smaller column found so far
            }
        }
        unsigned char col[3] = {0, 0, 0};
        if (m < kInfD2) {                          // no source anywhere: the call is rejected after the launch; write zeros
            // extract_background assigns imgs[bc_ids, np.nonzero(bc_pixs)] with the [HW,1] mask's nonzero tuple, which also writes pixel 0
            // once per source pixel: pixel 0 ends with the colour of the frame chosen at the LAST source pixel in raster order
            const long long q = (long long)(r + off[bu]) * W + bu;
            const int fr = q == 0 ? argmax[*last_bc - 1] : argmax[q];
            const unsigned char* px = frames + (long long)fr * frame_stride + q * 3;
            col[0] = px[0]; col[1] = px[1]; col[2] = px[2];
        }
        const long long p = (long long)r * W + x;
        if (bg_u8)
            for (int ch = 0; ch < 3; ++ch) bg_u8[p * 3 + ch] = col[ch];
        if (bg_f32)
            for (int ch = 0; ch < 3; ++ch) bg_f32[ch * plane + p] = normalise(col[ch]);
    }
}

bool size_ok(int H, int W) { return H >= kMinSize && H <= kMaxSize && W >= kMinSize && W <= kMaxSize; }

}  // namespace source
}  // namespace r3dp

using namespace r3dp;
using namespace r3dp::source;

extern "C" int r3dp_src_inpaint(const unsigned char* img, const void* seg, int seg_u8, int H, int W, const double* tab_torso,
                                const double* tab_neck, unsigned char* img2, unsigned char* flags, r3dp_stream_t stream) {
    R3DP_REQUIRE(img && seg && tab_torso && tab_neck && img2 && flags, "src_inpaint: null pointer");
    R3DP_REQUIRE(size_ok(H, W), "src_inpaint: H and W must lie in [%d, %d], got %d x %d", kMinSize, kMaxSize, H, W);
    const dim3 block(32, 8), grid(blocks(W, 8));
    if (seg_u8)
        src_inpaint_kernel<<<grid, block, 0, as_stream(stream)>>>(img, (const unsigned char*)seg, H, W, tab_torso, tab_neck, img2, flags);
    else
        src_inpaint_kernel<<<grid, block, 0, as_stream(stream)>>>(img, (const float*)seg, H, W, tab_torso, tab_neck, img2, flags);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_src_compose(const unsigned char* img, const void* seg, int seg_u8, const unsigned char* img2, const unsigned char* flags,
                                int H, int W, float* head_f32, float* torso_f32, unsigned char* torso_u8, r3dp_stream_t stream) {
    R3DP_REQUIRE(img && seg && img2 && flags, "src_compose: null pointer");
    R3DP_REQUIRE(head_f32 || torso_f32 || torso_u8, "src_compose: no output");
    R3DP_REQUIRE(size_ok(H, W), "src_compose: H and W must lie in [%d, %d], got %d x %d", kMinSize, kMaxSize, H, W);
    const unsigned grid = blocks((long long)H * W, 256);
    if (seg_u8)
        src_compose_kernel<<<grid, 256, 0, as_stream(stream)>>>(img, (const unsigned char*)seg, img2, flags, H, W, head_f32, torso_f32, torso_u8);
    else
        src_compose_kernel<<<grid, 256, 0, as_stream(stream)>>>(img, (const float*)seg, img2, flags, H, W, head_f32, torso_f32, torso_u8);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_src_bg_distance(const void* segs, int seg_u8, long long seg_stride, int F, int H, int W, short* g, int chunk, int* maxd2,
                                    int* argmax, int* has_fg, r3dp_stream_t stream) {
    R3DP_REQUIRE(segs && g && maxd2 && argmax && has_fg, "src_bg_distance: null pointer");
    R3DP_REQUIRE(size_ok(H, W), "src_bg_distance: H and W must lie in [%d, %d], got %d x %d", kMinSize, kMaxSize, H, W);
    R3DP_REQUIRE(F >= 1 && chunk >= 1 && chunk <= 65535, "src_bg_distance: need F >= 1 and 1 <= chunk <= 65535");
    cudaStream_t st = as_stream(stream);
    R3DP_CUDA(cudaMemsetAsync(has_fg, 0, sizeof(int) * F, st));
    for (int f0 = 0; f0 < F; f0 += chunk) {
        const int n = min(chunk, F - f0);
        const dim3 grid(blocks(W, 128), n);
        if (seg_u8)
            edt_cols_kernel<<<grid, 128, 0, st>>>((const unsigned char*)segs + f0 * seg_stride, seg_stride, nullptr, 0, H, W, g, has_fg + f0);
        else
            edt_cols_kernel<<<grid, 128, 0, st>>>((const float*)segs + f0 * seg_stride, seg_stride, nullptr, 0, H, W, g, has_fg + f0);
        R3DP_LAUNCH_CHECK();
        edt_max_kernel<<<H, kRowThreads, 0, st>>>(g, H, W, f0, n, maxd2, argmax);
        R3DP_LAUNCH_CHECK();
        count_launches(2);
    }
    return 0;
}

extern "C" int r3dp_src_bg_fill(const unsigned char* frames, long long frame_stride, const int* maxd2, const int* argmax, int H, int W, short* g,
                                int* has_bc, unsigned char* bg_u8, float* bg_f32, r3dp_stream_t stream) {
    R3DP_REQUIRE(frames && maxd2 && argmax && g && has_bc, "src_bg_fill: null pointer");
    R3DP_REQUIRE(bg_u8 || bg_f32, "src_bg_fill: no output");
    R3DP_REQUIRE(size_ok(H, W), "src_bg_fill: H and W must lie in [%d, %d], got %d x %d", kMinSize, kMaxSize, H, W);
    cudaStream_t st = as_stream(stream);
    R3DP_CUDA(cudaMemsetAsync(has_bc, 0, sizeof(int), st));
    edt_cols_kernel<float><<<dim3(blocks(W, 128), 1), 128, 0, st>>>(nullptr, 0, maxd2, 1, H, W, g, has_bc);
    R3DP_LAUNCH_CHECK();
    edt_fill_kernel<<<H, kRowThreads, 0, st>>>(g, argmax, has_bc, frames, frame_stride, H, W, bg_u8, bg_f32);
    R3DP_LAUNCH_CHECK();
    count_launches(2);
    return 0;
}
