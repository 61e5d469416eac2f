// SegFormerSECC2PlaneBackbone (modules/real3d/segformer.py:673-733, MiT-b0) on sm_90a: the kernels around the token GEMMs.
//   sp_prenet_kernel        the prenet's 1x1 conv (Conv2dLayer, networks_stylegan2.py:139-183) on the per-clip channels: the constant image
//   sp_embed_kernel         prenet (constant image + tgt part, or the whole input) fused with patch_embed1's 7x7 stride-4 conv (segformer.py:206-232)
//   sp_layernorm_kernel     optional residual add, then LayerNorm of each C <= 256 row in fp32 (one warp per row)
//   sp_patches_kernel       k x k stride-s patches of an NHWC fp16 image as GEMM rows: the 3x3/2 patch embeds of stages 2-4 and the
//                           spatial-reduction conv (k = stride = sr_ratio, segformer.py:126-128)
//   sp_attention_kernel     softmax(q k^T * scale) v for head_dim 32 and <= 256 keys (segformer.py:130-150), exact fp32 softmax
//   sp_dwconv_gelu_kernel   DWConv 3x3 + bias + exact GELU (segformer.py:82-84,459-468)
//   sp_head_fuse_kernel     SegFormerHead with linear_c* and the BN'd linear_fuse folded into the per-level maps G_i (the caller's GEMMs):
//                           sum_i resize_i(G_i c_i) + b, ReLU (segformer.py:525-537)
//   sp_leaky_kernel         nn.LeakyReLU(0.01) in place, for the to_plane_cnn convs that do not run on r3dp_sr_tc_conv
//   sp_upsample2_flip       nn.UpsamplingBilinear2d(x2) (align_corners=True), written row-mirrored and row+column-mirrored (segformer.py:722-730)
// The GEMMs themselves (q, kv, proj, fc1, fc2, patch embeds 2-4, sr, G_i, the last conv) run on r3dp_mf_conv3d; to_plane_cnn.0/2/4 on
// r3dp_sr_tc_conv.  Activations fp16, residual stream / LayerNorm / softmax / GELU in fp32.
#include "common.cuh"
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

// One warp per row; lane holds channels lane + 32 i.  Two-pass statistics in fp32 (nn.LayerNorm: biased variance).
__global__ void __launch_bounds__(256) sp_layernorm_kernel(const float* x, const float* __restrict__ t, int R, int C, const float* __restrict__ g,
                                                           const float* __restrict__ b, float eps, float* xo, float* __restrict__ yf,
                                                           __half* __restrict__ yh, int yhs) {
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= R) return;
    const int nv = C / 32;
    float v[8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        if (i < nv) {
            const size_t o = (size_t)row * C + lane + 32 * i;
            v[i] = x[o] + (t ? t[o] : 0.f);
            s += v[i];
        }
    }
#pragma unroll
    for (int m = 16; m; m >>= 1) s += __shfl_xor_sync(0xffffffffu, s, m);
    const float mean = s / C;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i)
        if (i < nv) { const float d = v[i] - mean; q = fmaf(d, d, q); }
#pragma unroll
    for (int m = 16; m; m >>= 1) q += __shfl_xor_sync(0xffffffffu, q, m);
    const float rstd = rsqrtf(q / C + eps);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        if (i >= nv) break;
        const int c = lane + 32 * i;
        const size_t o = (size_t)row * C + c;
        if (xo) xo[o] = v[i];
        const float u = fmaf((v[i] - mean) * rstd, g[c], b[c]);
        if (yf) yf[o] = u;
        if (yh) yh[(size_t)row * yhs + c] = __float2half_rn(u);
    }
}

// y[(n, oy, ox)][(ky*k + kx)*C + c] = x[n, oy*s - p + ky, ox*s - p + kx, c] (0 outside); 8 channels per thread.
__global__ void sp_patches_kernel(const __half* __restrict__ x, int N, int H, int W, int C, int k, int s, int p, int Ho, int Wo,
                                  __half* __restrict__ y) {
    const int c8 = C / 8;
    const long long total = (long long)N * Ho * Wo * k * k * c8;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    long long t = idx;
    const int cc = (int)(t % c8); t /= c8;
    const int tap = (int)(t % (k * k)); t /= (k * k);
    const int ox = (int)(t % Wo); t /= Wo;
    const int oy = (int)(t % Ho); const int n = (int)(t / Ho);
    const int iy = oy * s - p + tap / k, ix = ox * s - p + tap % k;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = *reinterpret_cast<const uint4*>(x + (((size_t)n * H + iy) * W + ix) * C + cc * 8);
    *reinterpret_cast<uint4*>(y + idx * 8) = v;
}

// grid (ceil(Tq / 128), heads, N), one thread per query.  K and V of the (frame, head) sit in shared memory as fp32; pass 1 finds the row
// maximum, pass 2 accumulates exp(s - max) and exp(s - max) v, so the softmax is the exact full-row one.
__global__ void __launch_bounds__(128) sp_attention_kernel(const __half* __restrict__ q, int qs, const __half* __restrict__ kv, int kvs, int Tq,
                                                           int Tk, int C, float scale, __half* __restrict__ o, int os) {
    extern __shared__ float4 skv[];                               // [Tk][8] keys then [Tk][8] values (float4 = 4 dims)
    const int h = blockIdx.y, n = blockIdx.z;
    for (int i = threadIdx.x; i < Tk * kHd; i += blockDim.x) {
        const int j = i / kHd, d = i % kHd;
        const __half* r = kv + ((size_t)n * Tk + j) * kvs + h * kHd + d;
        reinterpret_cast<float*>(skv)[i] = __half2float(r[0]);
        reinterpret_cast<float*>(skv)[Tk * kHd + i] = __half2float(r[C]);
    }
    __syncthreads();
    const int tq = blockIdx.x * blockDim.x + threadIdx.x;
    if (tq >= Tq) return;
    float qv[kHd];
    const __half* qr = q + ((size_t)n * Tq + tq) * qs + h * kHd;
#pragma unroll
    for (int d = 0; d < kHd; ++d) qv[d] = __half2float(qr[d]) * scale;
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
    __half2* orow = reinterpret_cast<__half2*>(o + ((size_t)n * Tq + tq) * os + h * kHd);
#pragma unroll
    for (int d = 0; d < kHd / 2; ++d) orow[d] = __floats2half2_rn(acc[2 * d] * inv, acc[2 * d + 1] * inv);
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

// F.interpolate(bilinear, align_corners=False) source taps along one axis (PyTorch's area_pixel_compute_source_index + clamp at 0)
__device__ __forceinline__ void bilin_src(int o, int in, int out, int& i0, int& i1, float& l1) {
    float s = ((float)o + 0.5f) * ((float)in / (float)out) - 0.5f;
    s = fmaxf(s, 0.f);
    i0 = min((int)s, in - 1);
    i1 = min(i0 + 1, in - 1);
    l1 = s - (float)i0;
}

struct HeadLevels { const float* g[4]; int hw[4]; };

// one thread per (pixel, 4 channels) of the H1 x H1 output; levels NHWC fp32 [N, hw_i, hw_i, 256]
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
    __half2* out = reinterpret_cast<__half2*>(y + pix * E + c);
    out[0] = __floats2half2_rn(fmaxf(a.x, 0.f), fmaxf(a.y, 0.f));
    out[1] = __floats2half2_rn(fmaxf(a.z, 0.f), fmaxf(a.w, 0.f));
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
    R3DP_REQUIRE(R > 0 && C % 32 == 0 && C >= 32 && C <= 256 && (!yh_f16 || yhs >= C), "sp_layernorm: C must be a multiple of 32, at most 256");
    sp_layernorm_kernel<<<blocks(R, 8), 256, 0, as_stream(stream)>>>(x, t, R, C, g, b, eps, xo, yf, reinterpret_cast<__half*>(yh_f16), yhs);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_sp_patches(const void* x_f16, int N, int H, int W, int C, int k, int s, int p, void* y_f16, r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && y_f16, "sp_patches: null pointer");
    R3DP_REQUIRE(N > 0 && H > 0 && W > 0 && C % 8 == 0 && k > 0 && s > 0 && p >= 0 && H + 2 * p >= k && W + 2 * p >= k, "sp_patches: bad shape");
    const int Ho = (H + 2 * p - k) / s + 1, Wo = (W + 2 * p - k) / s + 1;
    const long long n = (long long)N * Ho * Wo * k * k * (C / 8);
    sp_patches_kernel<<<blocks(n, 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<const __half*>(x_f16), N, H, W, C, k, s, p, Ho, Wo,
                                                                     reinterpret_cast<__half*>(y_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_sp_attention(const void* q_f16, int qs, const void* kv_f16, int kvs, int N, int Tq, int Tk, int heads, float scale, void* o_f16,
                                 int os, r3dp_stream_t stream) {
    R3DP_REQUIRE(q_f16 && kv_f16 && o_f16, "sp_attention: null pointer");
    const int C = heads * kHd;
    R3DP_REQUIRE(N > 0 && Tq > 0 && Tk > 0 && Tk <= kMaxKeys && heads > 0 && qs >= C && kvs >= 2 * C && os >= C && qs % 2 == 0 && os % 2 == 0,
                 "sp_attention: bad shape (head_dim 32, at most 256 keys)");
    const int smem = 2 * Tk * kHd * (int)sizeof(float);
    static bool smem_set = false;                                 // once per process (the attribute is per function, not per launch)
    if (!smem_set) {
        R3DP_CUDA(cudaFuncSetAttribute(sp_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * kMaxKeys * kHd * (int)sizeof(float)));
        smem_set = true;
    }
    const dim3 grid(blocks(Tq, 128), heads, N);
    sp_attention_kernel<<<grid, 128, smem, as_stream(stream)>>>(reinterpret_cast<const __half*>(q_f16), qs, reinterpret_cast<const __half*>(kv_f16), kvs,
                                                                Tq, Tk, C, scale, reinterpret_cast<__half*>(o_f16), os);
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
    sp_head_fuse_kernel<<<blocks(n, 256), 256, 0, as_stream(stream)>>>(lv, N, h1, bias, reinterpret_cast<__half*>(y_f16));
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
