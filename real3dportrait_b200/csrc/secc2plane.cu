// SegFormerSECC2PlaneBackbone (modules/real3d/segformer.py:673-733, MiT-b0) on sm_90a: the kernels around the token GEMMs.
//   sp_prenet_kernel        the prenet's 1x1 conv (Conv2dLayer, networks_stylegan2.py:139-183) on the per-clip channels: the constant image
//   sp_embed_kernel         prenet (constant image + tgt part, or the whole input) fused with patch_embed1's 7x7 stride-4 conv (segformer.py:206-232)
//   layernorm_rows_kernel   (layernorm.cuh) optional residual add, then LayerNorm of each C <= 1024 row in fp32 (one warp per row)
//   sp_patches_kernel       k x k stride-s dilation-d patches of an NHWC fp16 image as GEMM rows: the 3x3/2 patch embeds of stages 2-4 and
//                           the spatial-reduction conv (k = stride = sr_ratio, segformer.py:126-128); Img2PlaneModel's strided and dilated convs
//   sp_attention_kernel     softmax(q k^T * scale) v for head_dim 32 and <= 256 keys (segformer.py:130-150), exact fp32 softmax
//   sp_dwconv_gelu_kernel   DWConv 3x3 + bias + exact GELU (segformer.py:82-84,459-468)
//   sp_head_fuse_kernel     SegFormerHead with linear_c* and the BN'd linear_fuse folded into the per-level maps G_i (the caller's GEMMs):
//                           sum_i resize_i(G_i c_i) + b, ReLU (segformer.py:525-537)
//   sp_leaky_kernel         nn.LeakyReLU(0.01) in place, for the to_plane_cnn convs that do not run on r3dp_sr_tc_conv
//   sp_upsample2_flip       nn.UpsamplingBilinear2d(x2) (align_corners=True), written row-mirrored and row+column-mirrored (segformer.py:722-730)
// The GEMMs themselves (q, kv, proj, fc1, fc2, patch embeds 2-4, sr, G_i, the last conv) run on r3dp_mf_conv3d; to_plane_cnn.0/2/4 on
// r3dp_sr_tc_conv.  Activations fp16, residual stream / LayerNorm / softmax / GELU in fp32.
// precision='tc_exact' runs the *_split entry points at the end of this file: each activation the `tc` path stores as fp16 is stored as fp32
// (the GEMM outputs the attention and the DWConv read) or as split rows [hi C | lo C], hi = fp16(v), lo = fp16(v - hi), which the split
// r3dp_mf_conv3d / r3dp_sr_tcx_conv read as three MMAs per product.
#include "common.cuh"
#include "layernorm.cuh"
#include <cuda_fp16.h>
#include <math.h>

namespace r3dp {
namespace sp {

constexpr int kEmbedC = 32;              // MiT-b0 embed_dims[0]
constexpr int kHd = 32;                  // head_dim of every MiT-b0 stage
constexpr int kMaxKeys = 256;

__global__ void sp_prenet_kernel(const float* __restrict__ x, int N, int cin, int HW, const float* __restrict__ w, const float* __restrict__ b,
                                 float* __restrict__ y) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * HW) return;
    const int n = (int)(idx / HW), p = (int)(idx % HW);
    for (int c = 0; c < 3; ++c) {
        float v = b[c];
        for (int j = 0; j < cin; ++j) v = fmaf(w[c * cin + j], x[((size_t)n * cin + j) * HW + p], v);
        y[((size_t)n * 3 + c) * HW + p] = v;
    }
}

// One thread per output token.  smem: the patch-embed weights as [ky*7+kx][c][co] (broadcast reads), the prenet's [3][cin].
__global__ void __launch_bounds__(128) sp_embed_kernel(const float* __restrict__ x, int N, int cin, int H, int W, const float* __restrict__ wpre,
                                                       const float* __restrict__ base, const float* __restrict__ bpre,
                                                       const float* __restrict__ wpe, const float* __restrict__ bpe, float* __restrict__ y) {
    __shared__ float sw[49 * 3 * kEmbedC];
    __shared__ float spre[3 * 9];
    for (int i = threadIdx.x; i < 49 * 3 * kEmbedC; i += blockDim.x) {
        const int co = i % kEmbedC, c = (i / kEmbedC) % 3, tap = i / (3 * kEmbedC);
        sw[i] = wpe[(co * 3 + c) * 49 + tap];
    }
    for (int i = threadIdx.x; i < 3 * cin; i += blockDim.x) spre[i] = wpre[i];
    __syncthreads();
    const int Ho = (H - 1) / 4 + 1, Wo = (W - 1) / 4 + 1;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * Ho * Wo) return;
    const int ox = (int)(idx % Wo), oy = (int)((idx / Wo) % Ho), n = (int)(idx / ((long long)Wo * Ho));
    float acc[kEmbedC];
#pragma unroll
    for (int co = 0; co < kEmbedC; ++co) acc[co] = bpe[co];
    const size_t HW = (size_t)H * W;
    for (int ky = 0; ky < 7; ++ky) {
        const int iy = oy * 4 - 3 + ky;
        if (iy < 0 || iy >= H) continue;                          // the conv's zero padding of the prenet OUTPUT
        for (int kx = 0; kx < 7; ++kx) {
            const int ix = ox * 4 - 3 + kx;
            if (ix < 0 || ix >= W) continue;
            const size_t pix = (size_t)iy * W + ix;
            float p[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) p[c] = base ? base[c * HW + pix] : bpre[c];
            for (int j = 0; j < cin; ++j) {
                const float xv = x[((size_t)n * cin + j) * HW + pix];
#pragma unroll
                for (int c = 0; c < 3; ++c) p[c] = fmaf(spre[c * cin + j], xv, p[c]);
            }
            const float* wt = sw + (ky * 7 + kx) * 3 * kEmbedC;
#pragma unroll
            for (int c = 0; c < 3; ++c)
#pragma unroll
                for (int co = 0; co < kEmbedC; ++co) acc[co] = fmaf(wt[c * kEmbedC + co], p[c], acc[co]);
        }
    }
    float4* out = reinterpret_cast<float4*>(y + idx * kEmbedC);
#pragma unroll
    for (int i = 0; i < kEmbedC / 4; ++i) out[i] = make_float4(acc[4 * i], acc[4 * i + 1], acc[4 * i + 2], acc[4 * i + 3]);
}

// y[(n, oy, ox)][(ky*k + kx)*C + c] = x[n, oy*s - p + ky*d, ox*s - p + kx*d, c] (0 outside), rows of ldy halves with columns from k*k*C
// on zero; 8 channels per thread.
__global__ void sp_patches_kernel(const __half* __restrict__ x, int N, int H, int W, int C, int k, int s, int p, int d, int Ho, int Wo, int ldy,
                                  __half* __restrict__ y) {
    const int c8 = C / 8, l8 = ldy / 8;
    const long long total = (long long)N * Ho * Wo * l8;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    long long t = idx;
    const int j = (int)(t % l8); t /= l8;
    const int ox = (int)(t % Wo); t /= Wo;
    const int oy = (int)(t % Ho); const int n = (int)(t / Ho);
    const int tap = j / c8, cc = j - tap * c8;
    const int iy = oy * s - p + (tap / k) * d, ix = ox * s - p + (tap % k) * d;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (tap < k * k && iy >= 0 && iy < H && ix >= 0 && ix < W) v = *reinterpret_cast<const uint4*>(x + (((size_t)n * H + iy) * W + ix) * C + cc * 8);
    *reinterpret_cast<uint4*>(y + idx * 8) = v;
}

__device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_f32(float v) { return v; }

// hi = fp16(v) at y[0], lo = fp16(v - hi) at y[lo]: one value of a split row
__device__ __forceinline__ void put_split(__half* y, int lo, float v) {
    const __half h = __float2half_rn(v);
    y[0] = h;
    y[lo] = __float2half_rn(v - __half2float(h));
}

// grid (ceil(Tq / 128), heads, N), one thread per query.  K and V of the (frame, head) sit in shared memory as fp32; pass 1 finds the row
// maximum, pass 2 accumulates exp(s - max) and exp(s - max) v, so the softmax is the exact full-row one.  T: the element type of q and kv
// (fp16, or fp32 in tc_exact); SPLIT: o is written as split rows, lo at olo (tc_exact), else fp16.
template <typename T, bool SPLIT>
__global__ void __launch_bounds__(128) sp_attention_kernel(const T* __restrict__ q, int qs, const T* __restrict__ kv, int kvs, int Tq,
                                                           int Tk, int C, float scale, __half* __restrict__ o, int os, int olo) {
    extern __shared__ float4 skv[];                               // [Tk][8] keys then [Tk][8] values (float4 = 4 dims)
    const int h = blockIdx.y, n = blockIdx.z;
    for (int i = threadIdx.x; i < Tk * kHd; i += blockDim.x) {
        const int j = i / kHd, d = i % kHd;
        const T* r = kv + ((size_t)n * Tk + j) * kvs + h * kHd + d;
        reinterpret_cast<float*>(skv)[i] = to_f32(r[0]);
        reinterpret_cast<float*>(skv)[Tk * kHd + i] = to_f32(r[C]);
    }
    __syncthreads();
    const int tq = blockIdx.x * blockDim.x + threadIdx.x;
    if (tq >= Tq) return;
    float qv[kHd];
    const T* qr = q + ((size_t)n * Tq + tq) * qs + h * kHd;
#pragma unroll
    for (int d = 0; d < kHd; ++d) qv[d] = to_f32(qr[d]) * scale;
    const float4* sk = skv;
    const float4* sv = skv + Tk * (kHd / 4);
    float mx = -INFINITY;
    for (int j = 0; j < Tk; ++j) {
        float s = 0.f;
#pragma unroll
        for (int d4 = 0; d4 < kHd / 4; ++d4) {
            const float4 kk = sk[j * (kHd / 4) + d4];
            s = fmaf(qv[4 * d4], kk.x, s); s = fmaf(qv[4 * d4 + 1], kk.y, s); s = fmaf(qv[4 * d4 + 2], kk.z, s); s = fmaf(qv[4 * d4 + 3], kk.w, s);
        }
        mx = fmaxf(mx, s);
    }
    float acc[kHd];
#pragma unroll
    for (int d = 0; d < kHd; ++d) acc[d] = 0.f;
    float l = 0.f;
    for (int j = 0; j < Tk; ++j) {
        float s = 0.f;
#pragma unroll
        for (int d4 = 0; d4 < kHd / 4; ++d4) {
            const float4 kk = sk[j * (kHd / 4) + d4];
            s = fmaf(qv[4 * d4], kk.x, s); s = fmaf(qv[4 * d4 + 1], kk.y, s); s = fmaf(qv[4 * d4 + 2], kk.z, s); s = fmaf(qv[4 * d4 + 3], kk.w, s);
        }
        const float pj = expf(s - mx);
        l += pj;
#pragma unroll
        for (int d4 = 0; d4 < kHd / 4; ++d4) {
            const float4 vv = sv[j * (kHd / 4) + d4];
            acc[4 * d4] = fmaf(pj, vv.x, acc[4 * d4]); acc[4 * d4 + 1] = fmaf(pj, vv.y, acc[4 * d4 + 1]);
            acc[4 * d4 + 2] = fmaf(pj, vv.z, acc[4 * d4 + 2]); acc[4 * d4 + 3] = fmaf(pj, vv.w, acc[4 * d4 + 3]);
        }
    }
    const float inv = 1.f / l;
    __half* ob = o + ((size_t)n * Tq + tq) * os + h * kHd;
    if constexpr (SPLIT) {
#pragma unroll
        for (int d = 0; d < kHd; ++d) put_split(ob + d, olo, acc[d] * inv);
    } else {
        __half2* orow = reinterpret_cast<__half2*>(ob);
#pragma unroll
        for (int d = 0; d < kHd / 2; ++d) orow[d] = __floats2half2_rn(acc[2 * d] * inv, acc[2 * d + 1] * inv);
    }
}

// one thread per (pixel, channel pair); weights [C][9] fp32
__global__ void sp_dwconv_gelu_kernel(const __half* __restrict__ x, int N, int H, int W, int C, const float* __restrict__ w,
                                      const float* __restrict__ b, __half* __restrict__ y) {
    const int c2 = C / 2;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * H * W * c2) return;
    const int c = (int)(idx % c2) * 2;
    const long long pix = idx / c2;
    const int xx = (int)(pix % W), yy = (int)((pix / W) % H), n = (int)(pix / ((long long)W * H));
    float a0 = b[c], a1 = b[c + 1];
    for (int dy = -1; dy <= 1; ++dy) {
        const int iy = yy + dy;
        if (iy < 0 || iy >= H) continue;
        for (int dx = -1; dx <= 1; ++dx) {
            const int ix = xx + dx;
            if (ix < 0 || ix >= W) continue;
            const float2 v = __half22float2(*reinterpret_cast<const __half2*>(x + (((size_t)n * H + iy) * W + ix) * C + c));
            const int tap = (dy + 1) * 3 + dx + 1;
            a0 = fmaf(w[c * 9 + tap], v.x, a0);
            a1 = fmaf(w[(c + 1) * 9 + tap], v.y, a1);
        }
    }
    a0 = 0.5f * a0 * (1.f + erff(a0 * 0.70710678118654752f));
    a1 = 0.5f * a1 * (1.f + erff(a1 * 0.70710678118654752f));
    *reinterpret_cast<__half2*>(y + pix * C + c) = __floats2half2_rn(a0, a1);
}

// The split form (tc_exact): x fp32 NHWC [N,H,W,C] (fc1's fp32 output), y split rows [N*H*W][hi C | lo C]; the same taps, order and GELU
__global__ void sp_dwconv_gelu_split_kernel(const float* __restrict__ x, int N, int H, int W, int C, const float* __restrict__ w,
                                            const float* __restrict__ b, __half* __restrict__ y) {
    const int c2 = C / 2;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * H * W * c2) return;
    const int c = (int)(idx % c2) * 2;
    const long long pix = idx / c2;
    const int xx = (int)(pix % W), yy = (int)((pix / W) % H), n = (int)(pix / ((long long)W * H));
    float a0 = b[c], a1 = b[c + 1];
    for (int dy = -1; dy <= 1; ++dy) {
        const int iy = yy + dy;
        if (iy < 0 || iy >= H) continue;
        for (int dx = -1; dx <= 1; ++dx) {
            const int ix = xx + dx;
            if (ix < 0 || ix >= W) continue;
            const float2 v = *reinterpret_cast<const float2*>(x + (((size_t)n * H + iy) * W + ix) * C + c);
            const int tap = (dy + 1) * 3 + dx + 1;
            a0 = fmaf(w[c * 9 + tap], v.x, a0);
            a1 = fmaf(w[(c + 1) * 9 + tap], v.y, a1);
        }
    }
    a0 = 0.5f * a0 * (1.f + erff(a0 * 0.70710678118654752f));
    a1 = 0.5f * a1 * (1.f + erff(a1 * 0.70710678118654752f));
    const __half2 hi = __floats2half2_rn(a0, a1);
    const float2 hf = __half22float2(hi);
    __half* row = y + pix * 2 * C + c;
    *reinterpret_cast<__half2*>(row) = hi;
    *reinterpret_cast<__half2*>(row + C) = __floats2half2_rn(a0 - hf.x, a1 - hf.y);
}

// The split form of sp_patches_kernel (tc_exact): x split pixels [N,H,W][hi C | lo C], y rows [hi k*k*C | lo k*k*C] (d = 1, no padding
// columns), the layout r3dp_mf_conv3d reads with xs = 2K, xlo = K; 8 halves per thread.
__global__ void sp_patches_split_kernel(const __half* __restrict__ x, int N, int H, int W, int C, int k, int s, int p, int Ho, int Wo,
                                        __half* __restrict__ y) {
    const int c8 = C / 8, k8 = k * k * c8;                        // 8-half chunks per tap, per half-row
    const long long total = (long long)N * Ho * Wo * 2 * k8;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    long long t = idx;
    int j = (int)(t % (2 * k8)); t /= 2 * k8;
    const int ox = (int)(t % Wo); t /= Wo;
    const int oy = (int)(t % Ho); const int n = (int)(t / Ho);
    const int half = j >= k8 ? 1 : 0;
    j -= half * k8;
    const int tap = j / c8, cc = j - tap * c8;
    const int iy = oy * s - p + tap / k, ix = ox * s - p + tap % k;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = *reinterpret_cast<const uint4*>(x + (((size_t)n * H + iy) * W + ix) * 2 * C + half * C + cc * 8);
    *reinterpret_cast<uint4*>(y + idx * 8) = v;
}

// In-place nn.LeakyReLU on split rows [P][hi C | lo C]: v = hi + lo, then hi, lo of max(v, slope v); one thread per (pixel, channel pair)
__global__ void sp_leaky_split_kernel(__half* x, long long P, int C, float slope) {
    const int c2 = C / 2;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P * c2) return;
    __half* r = x + (idx / c2) * 2 * C + (int)(idx % c2) * 2;
    float2 v = __half22float2(*reinterpret_cast<const __half2*>(r));
    const float2 l = __half22float2(*reinterpret_cast<const __half2*>(r + C));
    v.x += l.x;
    v.y += l.y;
    v.x = fmaxf(v.x, v.x * slope);
    v.y = fmaxf(v.y, v.y * slope);
    const __half2 hi = __floats2half2_rn(v.x, v.y);
    const float2 hf = __half22float2(hi);
    *reinterpret_cast<__half2*>(r) = hi;
    *reinterpret_cast<__half2*>(r + C) = __floats2half2_rn(v.x - hf.x, v.y - hf.y);
}

// F.interpolate(bilinear, align_corners=False) source taps along one axis (PyTorch's area_pixel_compute_source_index + clamp at 0)
__device__ __forceinline__ void bilin_src(int o, int in, int out, int& i0, int& i1, float& l1) {
    float s = ((float)o + 0.5f) * ((float)in / (float)out) - 0.5f;
    s = fmaxf(s, 0.f);
    i0 = min((int)s, in - 1);
    i1 = min(i0 + 1, in - 1);
    l1 = s - (float)i0;
}

struct HeadLevels { const float* g[4]; int hw[4]; };

// one thread per (pixel, 4 channels) of the H1 x H1 output; levels NHWC fp32 [N, hw_i, hw_i, 256].  SPLIT (tc_exact): y split rows
// [N*H1*H1][hi 256 | lo 256], else fp16 [N*H1*H1][256]
template <bool SPLIT>
__global__ void sp_head_fuse_kernel(HeadLevels lv, int N, int H1, const float* __restrict__ bias, __half* __restrict__ y) {
    constexpr int E = 256;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * H1 * H1 * (E / 4)) return;
    const int c = (int)(idx % (E / 4)) * 4;
    const long long pix = idx / (E / 4);
    const int xx = (int)(pix % H1), yy = (int)((pix / H1) % H1), n = (int)(pix / ((long long)H1 * H1));
    float4 a = *reinterpret_cast<const float4*>(bias + c);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int h = lv.hw[i];
        int y0, y1, x0, x1; float ly, lx;
        bilin_src(yy, h, H1, y0, y1, ly);
        bilin_src(xx, h, H1, x0, x1, lx);
        const float* base = lv.g[i] + (size_t)n * h * h * E + c;
        const float4 v00 = *reinterpret_cast<const float4*>(base + ((size_t)y0 * h + x0) * E);
        const float4 v01 = *reinterpret_cast<const float4*>(base + ((size_t)y0 * h + x1) * E);
        const float4 v10 = *reinterpret_cast<const float4*>(base + ((size_t)y1 * h + x0) * E);
        const float4 v11 = *reinterpret_cast<const float4*>(base + ((size_t)y1 * h + x1) * E);
        const float w00 = (1.f - ly) * (1.f - lx), w01 = (1.f - ly) * lx, w10 = ly * (1.f - lx), w11 = ly * lx;
        a.x += w00 * v00.x + w01 * v01.x + w10 * v10.x + w11 * v11.x;
        a.y += w00 * v00.y + w01 * v01.y + w10 * v10.y + w11 * v11.y;
        a.z += w00 * v00.z + w01 * v01.z + w10 * v10.z + w11 * v11.z;
        a.w += w00 * v00.w + w01 * v01.w + w10 * v10.w + w11 * v11.w;
    }
    if constexpr (SPLIT) {
        __half* out = y + pix * 2 * E + c;
        put_split(out, E, fmaxf(a.x, 0.f));
        put_split(out + 1, E, fmaxf(a.y, 0.f));
        put_split(out + 2, E, fmaxf(a.z, 0.f));
        put_split(out + 3, E, fmaxf(a.w, 0.f));
    } else {
        __half2* out = reinterpret_cast<__half2*>(y + pix * E + c);
        out[0] = __floats2half2_rn(fmaxf(a.x, 0.f), fmaxf(a.y, 0.f));
        out[1] = __floats2half2_rn(fmaxf(a.z, 0.f), fmaxf(a.w, 0.f));
    }
}

__global__ void sp_leaky_kernel(__half2* x, long long n2, float slope) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n2) return;
    float2 v = __half22float2(x[i]);
    v.x = fmaxf(v.x, v.x * slope);
    v.y = fmaxf(v.y, v.y * slope);
    x[i] = __floats2half2_rn(v.x, v.y);
}

// one thread per (output pixel of the 2h x 2w grid, 8 channels); the value at (Y, X) goes to (2h-1-Y, X) of y_r and (2h-1-Y, 2w-1-X) of y_rc
__global__ void sp_upsample2_flip_kernel(const __half* __restrict__ x, int N, int h, int w, int C, __half* __restrict__ yr,
                                         __half* __restrict__ yrc) {
    const int H = 2 * h, W = 2 * w, c8 = C / 8;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * H * W * c8) return;
    const int cc = (int)(idx % c8);
    const long long pix = idx / c8;
    const int X = (int)(pix % W), Y = (int)((pix / W) % H), n = (int)(pix / ((long long)W * H));
    const float sy = (float)Y * ((float)(h - 1) / (float)(H - 1)), sx = (float)X * ((float)(w - 1) / (float)(W - 1));
    const int y0 = min((int)sy, h - 1), x0 = min((int)sx, w - 1);
    const int y1 = min(y0 + 1, h - 1), x1 = min(x0 + 1, w - 1);
    const float ly = sy - (float)y0, lx = sx - (float)x0;
    const __half* b = x + (size_t)n * h * w * C + cc * 8;
    const uint4 q00 = *reinterpret_cast<const uint4*>(b + ((size_t)y0 * w + x0) * C), q01 = *reinterpret_cast<const uint4*>(b + ((size_t)y0 * w + x1) * C);
    const uint4 q10 = *reinterpret_cast<const uint4*>(b + ((size_t)y1 * w + x0) * C), q11 = *reinterpret_cast<const uint4*>(b + ((size_t)y1 * w + x1) * C);
    const __half2* h00 = reinterpret_cast<const __half2*>(&q00); const __half2* h01 = reinterpret_cast<const __half2*>(&q01);
    const __half2* h10 = reinterpret_cast<const __half2*>(&q10); const __half2* h11 = reinterpret_cast<const __half2*>(&q11);
    uint4 res;
    __half2* r = reinterpret_cast<__half2*>(&res);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float2 a = __half22float2(h00[j]), bb = __half22float2(h01[j]), c = __half22float2(h10[j]), d = __half22float2(h11[j]);
        const float t0x = a.x + (bb.x - a.x) * lx, t0y = a.y + (bb.y - a.y) * lx;
        const float t1x = c.x + (d.x - c.x) * lx, t1y = c.y + (d.y - c.y) * lx;
        r[j] = __floats2half2_rn(t0x + (t1x - t0x) * ly, t0y + (t1y - t0y) * ly);
    }
    const size_t row_r = (size_t)n * H + (H - 1 - Y);
    *reinterpret_cast<uint4*>(yr + (row_r * W + X) * C + cc * 8) = res;
    *reinterpret_cast<uint4*>(yrc + (row_r * W + (W - 1 - X)) * C + cc * 8) = res;
}

// The split form (tc_exact): x, yr, yrc split pixels [hi C | lo C]; each tap is hi + lo in fp32, the same weights and order, and the
// interpolated value is written as hi, lo.  One thread per (output pixel, 4 channels)
__global__ void sp_upsample2_flip_split_kernel(const __half* __restrict__ x, int N, int h, int w, int C, __half* __restrict__ yr,
                                               __half* __restrict__ yrc) {
    const int H = 2 * h, W = 2 * w, c4 = C / 4;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * H * W * c4) return;
    const int c = (int)(idx % c4) * 4;
    const long long pix = idx / c4;
    const int X = (int)(pix % W), Y = (int)((pix / W) % H), n = (int)(pix / ((long long)W * H));
    const float sy = (float)Y * ((float)(h - 1) / (float)(H - 1)), sx = (float)X * ((float)(w - 1) / (float)(W - 1));
    const int y0 = min((int)sy, h - 1), x0 = min((int)sx, w - 1);
    const int y1 = min(y0 + 1, h - 1), x1 = min(x0 + 1, w - 1);
    const float ly = sy - (float)y0, lx = sx - (float)x0;
    const __half* b = x + (size_t)n * h * w * 2 * C + c;
    const __half* p[4] = {b + ((size_t)y0 * w + x0) * 2 * C, b + ((size_t)y0 * w + x1) * 2 * C, b + ((size_t)y1 * w + x0) * 2 * C,
                          b + ((size_t)y1 * w + x1) * 2 * C};
    float v[4][4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        const uint2 qh = *reinterpret_cast<const uint2*>(p[t]), ql = *reinterpret_cast<const uint2*>(p[t] + C);
        const __half2* hh = reinterpret_cast<const __half2*>(&qh);
        const __half2* hl = reinterpret_cast<const __half2*>(&ql);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const float2 a = __half22float2(hh[j]), l = __half22float2(hl[j]);
            v[t][2 * j] = a.x + l.x;
            v[t][2 * j + 1] = a.y + l.y;
        }
    }
    uint2 rh, rl;
    __half* oh = reinterpret_cast<__half*>(&rh);
    __half* ol = reinterpret_cast<__half*>(&rl);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float t0 = v[0][j] + (v[1][j] - v[0][j]) * lx, t1 = v[2][j] + (v[3][j] - v[2][j]) * lx;
        const float u = t0 + (t1 - t0) * ly;
        oh[j] = __float2half_rn(u);
        ol[j] = __float2half_rn(u - __half2float(oh[j]));
    }
    const size_t row_r = (size_t)n * H + (H - 1 - Y);
    __half* a = yr + (row_r * W + X) * 2 * C + c;
    __half* bb = yrc + (row_r * W + (W - 1 - X)) * 2 * C + c;
    *reinterpret_cast<uint2*>(a) = rh;
    *reinterpret_cast<uint2*>(a + C) = rl;
    *reinterpret_cast<uint2*>(bb) = rh;
    *reinterpret_cast<uint2*>(bb + C) = rl;
}

inline unsigned blocks(long long n, int t) { return (unsigned)((n + t - 1) / t); }

}  // namespace sp
}  // namespace r3dp

using namespace r3dp;
using namespace r3dp::sp;

extern "C" int r3dp_sp_prenet(const float* x, int N, int cin, int H, int W, const float* w, const float* b, float* y, r3dp_stream_t stream) {
    R3DP_REQUIRE(x && w && b && y, "sp_prenet: null pointer");
    R3DP_REQUIRE(N > 0 && cin > 0 && H > 0 && W > 0, "sp_prenet: bad shape");
    const long long n = (long long)N * H * W;
    sp_prenet_kernel<<<blocks(n, 256), 256, 0, as_stream(stream)>>>(x, N, cin, H * W, w, b, y);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_sp_embed(const float* x, int N, int cin, int H, int W, const float* wpre, const float* base, const float* bpre, const float* wpe,
                             const float* bpe, float* y, r3dp_stream_t stream) {
    R3DP_REQUIRE(x && wpre && (base || bpre) && wpe && bpe && y, "sp_embed: null pointer");
    R3DP_REQUIRE(N > 0 && cin > 0 && cin <= 9 && H > 0 && W > 0, "sp_embed: bad shape");
    const long long n = (long long)N * ((H - 1) / 4 + 1) * ((W - 1) / 4 + 1);
    sp_embed_kernel<<<blocks(n, 128), 128, 0, as_stream(stream)>>>(x, N, cin, H, W, wpre, base, bpre, wpe, bpe, y);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_sp_layernorm(const float* x, const float* t, int R, int C, const float* g, const float* b, float eps, float* xo, float* yf,
                                 void* yh_f16, int yhs, r3dp_stream_t stream) {
    R3DP_REQUIRE(x && g && b && (xo || yf || yh_f16), "sp_layernorm: null pointer");
    R3DP_REQUIRE(R > 0 && C % 32 == 0 && C >= 32 && C <= 1024 && (!yh_f16 || yhs >= C), "sp_layernorm: C must be a multiple of 32, at most 1024");
    if (C <= 256)
        layernorm_rows_kernel<8><<<blocks(R, 8), 256, 0, as_stream(stream)>>>(x, t, R, C, g, b, eps, xo, yf, C, reinterpret_cast<__half*>(yh_f16), yhs, 0, 0);
    else
        layernorm_rows_kernel<32><<<blocks(R, 8), 256, 0, as_stream(stream)>>>(x, t, R, C, g, b, eps, xo, yf, C, reinterpret_cast<__half*>(yh_f16), yhs, 0, 0);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_sp_patches_dil(const void* x_f16, int N, int H, int W, int C, int k, int s, int p, int d, void* y_f16, int ldy,
                                   r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && y_f16, "sp_patches: null pointer");
    const int ke = d * (k - 1) + 1;                               // the dilated window's extent
    R3DP_REQUIRE(N > 0 && H > 0 && W > 0 && C % 8 == 0 && C > 0 && k > 0 && s > 0 && p >= 0 && d > 0 && H + 2 * p >= ke && W + 2 * p >= ke &&
                 ldy >= k * k * C && ldy % 8 == 0, "sp_patches: bad shape");
    const int Ho = (H + 2 * p - ke) / s + 1, Wo = (W + 2 * p - ke) / s + 1;
    const long long n = (long long)N * Ho * Wo * (ldy / 8);
    sp_patches_kernel<<<blocks(n, 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<const __half*>(x_f16), N, H, W, C, k, s, p, d, Ho, Wo, ldy,
                                                                     reinterpret_cast<__half*>(y_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_sp_patches(const void* x_f16, int N, int H, int W, int C, int k, int s, int p, void* y_f16, r3dp_stream_t stream) {
    return r3dp_sp_patches_dil(x_f16, N, H, W, C, k, s, p, 1, y_f16, k * k * C, stream);
}

extern "C" int r3dp_sp_attention(const void* q_f16, int qs, const void* kv_f16, int kvs, int N, int Tq, int Tk, int heads, float scale, void* o_f16,
                                 int os, r3dp_stream_t stream) {
    R3DP_REQUIRE(q_f16 && kv_f16 && o_f16, "sp_attention: null pointer");
    const int C = heads * kHd;
    R3DP_REQUIRE(N > 0 && Tq > 0 && Tk > 0 && Tk <= kMaxKeys && heads > 0 && qs >= C && kvs >= 2 * C && os >= C && qs % 2 == 0 && os % 2 == 0,
                 "sp_attention: bad shape (head_dim 32, at most 256 keys)");
    const int smem = 2 * Tk * kHd * (int)sizeof(float);
    // the limit belongs to the current device's function, so it is set on every call (as every other launcher does): a process that drives
    // a second GPU would otherwise launch there with the 48 KB default and be refused at Tk > 192
    R3DP_CUDA(cudaFuncSetAttribute(sp_attention_kernel<__half, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   2 * kMaxKeys * kHd * (int)sizeof(float)));
    const dim3 grid(blocks(Tq, 128), heads, N);
    sp_attention_kernel<__half, false><<<grid, 128, smem, as_stream(stream)>>>(reinterpret_cast<const __half*>(q_f16), qs,
                                                                               reinterpret_cast<const __half*>(kv_f16), kvs, Tq, Tk, C, scale,
                                                                               reinterpret_cast<__half*>(o_f16), os, 0);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_sp_dwconv_gelu(const void* x_f16, int N, int H, int W, int C, const float* w, const float* b, void* y_f16, r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && w && b && y_f16, "sp_dwconv_gelu: null pointer");
    R3DP_REQUIRE(N > 0 && H > 0 && W > 0 && C % 2 == 0, "sp_dwconv_gelu: bad shape");
    const long long n = (long long)N * H * W * (C / 2);
    sp_dwconv_gelu_kernel<<<blocks(n, 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<const __half*>(x_f16), N, H, W, C, w, b,
                                                                         reinterpret_cast<__half*>(y_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_sp_head_fuse(const float* g1, int h1, const float* g2, int h2, const float* g3, int h3, const float* g4, int h4, int N,
                                 const float* bias, void* y_f16, r3dp_stream_t stream) {
    R3DP_REQUIRE(g1 && g2 && g3 && g4 && bias && y_f16, "sp_head_fuse: null pointer");
    R3DP_REQUIRE(N > 0 && h1 > 0 && h2 > 0 && h3 > 0 && h4 > 0, "sp_head_fuse: bad shape");
    HeadLevels lv = {{g1, g2, g3, g4}, {h1, h2, h3, h4}};
    const long long n = (long long)N * h1 * h1 * 64;
    sp_head_fuse_kernel<false><<<blocks(n, 256), 256, 0, as_stream(stream)>>>(lv, N, h1, bias, reinterpret_cast<__half*>(y_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_sp_leaky(void* x_f16, long long n, float slope, r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && n > 0 && n % 2 == 0, "sp_leaky: bad arguments");
    sp_leaky_kernel<<<blocks(n / 2, 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<__half2*>(x_f16), n / 2, slope);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_sp_upsample2_flip(const void* x_f16, int N, int h, int w, int C, void* yr_f16, void* yrc_f16, r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && yr_f16 && yrc_f16, "sp_upsample2_flip: null pointer");
    R3DP_REQUIRE(N > 0 && h > 1 && w > 1 && C % 8 == 0, "sp_upsample2_flip: bad shape");
    const long long n = (long long)N * 4 * h * w * (C / 8);
    sp_upsample2_flip_kernel<<<blocks(n, 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<const __half*>(x_f16), N, h, w, C,
                                                                            reinterpret_cast<__half*>(yr_f16), reinterpret_cast<__half*>(yrc_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

// ---- the split (tc_exact) forms: every activation that crosses a launch as fp16 in `tc` crosses as fp32 or as split rows [hi | lo] ----
extern "C" int r3dp_sp_layernorm_split(const float* x, const float* t, int R, int C, const float* g, const float* b, float eps, float* xo,
                                       void* yh_f16, int yhs, int yhlo, r3dp_stream_t stream) {
    R3DP_REQUIRE(x && t && g && b && yh_f16, "sp_layernorm_split: null pointer (the residual t and the split output are required)");
    R3DP_REQUIRE(R > 0 && C % 32 == 0 && C >= 32 && C <= 1024 && yhlo >= C && yhs >= yhlo + C,
                 "sp_layernorm_split: bad shape (C a multiple of 32, at most 1024; split rows [hi | lo])");
    __half* yh = reinterpret_cast<__half*>(yh_f16);
    if (C <= 256)
        layernorm_rows_kernel<8><<<blocks(R, 8), 256, 0, as_stream(stream)>>>(x, t, R, C, g, b, eps, xo, nullptr, C, yh, yhs, yhlo, 0);
    else
        layernorm_rows_kernel<32><<<blocks(R, 8), 256, 0, as_stream(stream)>>>(x, t, R, C, g, b, eps, xo, nullptr, C, yh, yhs, yhlo, 0);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_sp_patches_split(const void* x_f16, int N, int H, int W, int C, int k, int s, int p, void* y_f16, r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && y_f16, "sp_patches_split: null pointer");
    R3DP_REQUIRE(N > 0 && H > 0 && W > 0 && C % 8 == 0 && C > 0 && k > 0 && s > 0 && p >= 0 && H + 2 * p >= k && W + 2 * p >= k,
                 "sp_patches_split: bad shape");
    const int Ho = (H + 2 * p - k) / s + 1, Wo = (W + 2 * p - k) / s + 1;
    const long long n = (long long)N * Ho * Wo * 2 * k * k * (C / 8);
    sp_patches_split_kernel<<<blocks(n, 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<const __half*>(x_f16), N, H, W, C, k, s, p, Ho, Wo,
                                                                           reinterpret_cast<__half*>(y_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_sp_attention_split(const float* q, int qs, const float* kv, int kvs, int N, int Tq, int Tk, int heads, float scale, void* o_f16,
                                       int os, int olo, r3dp_stream_t stream) {
    R3DP_REQUIRE(q && kv && o_f16, "sp_attention_split: null pointer");
    const int C = heads * kHd;
    R3DP_REQUIRE(N > 0 && Tq > 0 && Tk > 0 && Tk <= kMaxKeys && heads > 0 && qs >= C && kvs >= 2 * C && olo >= C && os >= olo + C,
                 "sp_attention_split: bad shape (head_dim 32, at most 256 keys; split rows [hi | lo])");
    const int smem = 2 * Tk * kHd * (int)sizeof(float);
    R3DP_CUDA(cudaFuncSetAttribute(sp_attention_kernel<float, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   2 * kMaxKeys * kHd * (int)sizeof(float)));
    const dim3 grid(blocks(Tq, 128), heads, N);
    sp_attention_kernel<float, true><<<grid, 128, smem, as_stream(stream)>>>(q, qs, kv, kvs, Tq, Tk, C, scale, reinterpret_cast<__half*>(o_f16),
                                                                             os, olo);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_sp_dwconv_gelu_split(const float* x, int N, int H, int W, int C, const float* w, const float* b, void* y_f16,
                                         r3dp_stream_t stream) {
    R3DP_REQUIRE(x && w && b && y_f16, "sp_dwconv_gelu_split: null pointer");
    R3DP_REQUIRE(N > 0 && H > 0 && W > 0 && C % 2 == 0, "sp_dwconv_gelu_split: bad shape");
    const long long n = (long long)N * H * W * (C / 2);
    sp_dwconv_gelu_split_kernel<<<blocks(n, 256), 256, 0, as_stream(stream)>>>(x, N, H, W, C, w, b, reinterpret_cast<__half*>(y_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_sp_head_fuse_split(const float* g1, int h1, const float* g2, int h2, const float* g3, int h3, const float* g4, int h4, int N,
                                       const float* bias, void* y_f16, r3dp_stream_t stream) {
    R3DP_REQUIRE(g1 && g2 && g3 && g4 && bias && y_f16, "sp_head_fuse_split: null pointer");
    R3DP_REQUIRE(N > 0 && h1 > 0 && h2 > 0 && h3 > 0 && h4 > 0, "sp_head_fuse_split: bad shape");
    HeadLevels lv = {{g1, g2, g3, g4}, {h1, h2, h3, h4}};
    const long long n = (long long)N * h1 * h1 * 64;
    sp_head_fuse_kernel<true><<<blocks(n, 256), 256, 0, as_stream(stream)>>>(lv, N, h1, bias, reinterpret_cast<__half*>(y_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_sp_leaky_split(void* x_f16, long long P, int C, float slope, r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && P > 0 && C > 0 && C % 2 == 0, "sp_leaky_split: bad arguments");
    sp_leaky_split_kernel<<<blocks(P * (C / 2), 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<__half*>(x_f16), P, C, slope);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_sp_upsample2_flip_split(const void* x_f16, int N, int h, int w, int C, void* yr_f16, void* yrc_f16, r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && yr_f16 && yrc_f16, "sp_upsample2_flip_split: null pointer");
    R3DP_REQUIRE(N > 0 && h > 1 && w > 1 && C % 4 == 0, "sp_upsample2_flip_split: bad shape");
    const long long n = (long long)N * 4 * h * w * (C / 4);
    sp_upsample2_flip_split_kernel<<<blocks(n, 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<const __half*>(x_f16), N, h, w, C,
                                                                                  reinterpret_cast<__half*>(yr_f16), reinterpret_cast<__half*>(yrc_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}
