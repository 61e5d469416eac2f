// Stage 2 of the torso warper (modules/real3d/facev2v_warp/network2.py:248-301 Generator + model2.py:212-219,260-263 occlusion_2_predictor):
// the kernels around the tensor-core convolutions (those run on conv_tc3, csrc/sr_tc.cu r3dp_tw_conv*).
//   tw_gather3d_kernel       Generator.get_deformed_feature: trilinear grid_sample of the appearance volume -> in_conv's NHWC fp16 A operand
//   tw_affine_relu_kernel    relu(s * x + t) per channel: the pre-activation BatchNorm + ReLU of each "NAC" ResBlock2D (layers.py:96-115)
//   tw_narrow_conv_kernel    the narrow-cout convolutions of the tail (out_conv 7x7 64 -> 3, the predictor's 65 -> 32 -> 32 -> 1) on CUDA cores, fp32
//   tw_hid_to_nchw_kernel    deformed_torso_hid back to the [N,C,H,W] fp32 tensor the caller's facev2v_ret carries
#include "common.cuh"
#include <cuda_fp16.h>

namespace r3dp {
namespace tw {

// F.grid_sample(fs, grid, mode='bilinear' (trilinear on 5-D input), padding_mode='border', align_corners=True) followed by
// .view(N, C*D, H, W).  fs NDHWC fp32 [N][D][H][W][C], grid [N][D][H][W][3] (x -> W, y -> H, z -> D), output NHWC fp16 [N][H][W][cs]
// with channel c*D + d (split: the fp16 remainder at channel C*D + c*D + d).  Thread = (n, h, w, d), d fastest: the D threads of a pixel
// store D consecutive halves per channel.  fs_shared: fs holds ONE volume read by every image (the per-clip cache).  The corner weights and their order are those of torch's grid_sampler_3d kernel.
__global__ void __launch_bounds__(256) tw_gather3d_kernel(const float* __restrict__ fs, const float* __restrict__ grid, int N, int C, int D, int H,
                                                          int W, int cs, int split, int fs_shared, __half* __restrict__ y) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * H * W * D) return;
    const int d = (int)(idx % D);
    const long long pix = idx / D;                                             // n*H*W + h*W + w
    const int w = (int)(pix % W), h = (int)((pix / W) % H), n = (int)(pix / ((long long)W * H));
    const float* g = grid + ((((size_t)n * D + d) * H + h) * W + w) * 3;
    // unnormalize (align_corners) then clip to the border
    const float ix = fminf(fmaxf((g[0] + 1.f) * 0.5f * (float)(W - 1), 0.f), (float)(W - 1));
    const float iy = fminf(fmaxf((g[1] + 1.f) * 0.5f * (float)(H - 1), 0.f), (float)(H - 1));
    const float iz = fminf(fmaxf((g[2] + 1.f) * 0.5f * (float)(D - 1), 0.f), (float)(D - 1));
    const int x0 = (int)floorf(ix), y0 = (int)floorf(iy), z0 = (int)floorf(iz);
    const float fx1 = (float)(x0 + 1) - ix, fx0 = ix - (float)x0;              // weights of the x0 / x0+1 corners
    const float fy1 = (float)(y0 + 1) - iy, fy0 = iy - (float)y0;
    const float fz1 = (float)(z0 + 1) - iz, fz0 = iz - (float)z0;
    float wt[8]; const float* src[8]; int ok[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int dz = k >> 2, dy = (k >> 1) & 1, dx = k & 1;
        const int zz = z0 + dz, yy = y0 + dy, xx = x0 + dx;
        wt[k] = (dx ? fx0 : fx1) * (dy ? fy0 : fy1) * (dz ? fz0 : fz1);
        ok[k] = zz < D && yy < H && xx < W;                                    // only the +1 corners can leave the volume (weight 0 there)
        src[k] = fs + ((((size_t)(fs_shared ? 0 : n) * D + (ok[k] ? zz : z0)) * H + (ok[k] ? yy : y0)) * W + (ok[k] ? xx : x0)) * C;
    }
    __half* out = y + (size_t)pix * cs + d;
    const int lo = C * D;
    for (int c0 = 0; c0 < C; c0 += 4) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            if (!ok[k]) continue;
            const float4 v = __ldg(reinterpret_cast<const float4*>(src[k] + c0));
            acc.x = fmaf(v.x, wt[k], acc.x); acc.y = fmaf(v.y, wt[k], acc.y); acc.z = fmaf(v.z, wt[k], acc.z); acc.w = fmaf(v.w, wt[k], acc.w);
        }
        const float r[4] = {acc.x, acc.y, acc.z, acc.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const __half hi = __float2half_rn(r[j]);
            out[(c0 + j) * D] = hi;
            if (split) out[lo + (c0 + j) * D] = __float2half_rn(r[j] - __half2float(hi));
        }
    }
}

// y = relu(x * s[c] + t[c]) on NHWC fp16 [P][cs] (channels 0..C-1; split: value = x[c] + x[lo + c], result split again, lo = C)
__global__ void tw_affine_relu_kernel(const __half* __restrict__ x, const float* __restrict__ s, const float* __restrict__ t, long long P, int C, int cs,
                                      int split, __half* __restrict__ y) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P * C) return;
    const int c = (int)(idx % C);
    const size_t e = (size_t)(idx / C) * cs + c;
    float v = __half2float(x[e]);
    if (split) v += __half2float(x[e + C]);
    v = fmaxf(fmaf(v, s[c], t[c]), 0.f);
    const __half hi = __float2half_rn(v);
    y[e] = hi;
    if (split) y[e + C] = __float2half_rn(v - __half2float(hi));
}

// Direct KxK convolution (stride 1, zero padding K/2) to CO <= 32 channels on CUDA cores, fp32 accumulation; one thread per output pixel.
// Input channels, in this order: xa (NHWC fp16, pixel stride sa, ca channels, split: + the remainder at channel lo_a) or xf (NHWC fp32, pixel
// stride sf, cf channels), then optionally ONE channel bilinearly resized on the fly from ex [N,1,eh,ew] fp32 to HxW (F.interpolate,
// align_corners=False: the concat of model2.py:262 without materialising it).  Weights wk fp32 [K*K][cin][CO] (tap-major), bias [CO].
// act 0 linear, 1 ReLU, 2 sigmoid.  Output fp32: NCHW [N][CO][H][W] (nchw != 0) or NHWC [N][H][W][CO].
constexpr int kNarrowThreads = 128;
template <int CO>
__global__ void __launch_bounds__(kNarrowThreads) tw_narrow_conv_kernel(const __half* __restrict__ xa, int sa, int ca, int lo_a,
                                                                        const float* __restrict__ xf, int sf, int cf, const float* __restrict__ ex,
                                                                        int eh, int ew, const float* __restrict__ wk, const float* __restrict__ bias,
                                                                        int N, int H, int W, int K, int act, int nchw, float* __restrict__ out) {
    extern __shared__ float s_w[];                                              // [K*K][cin][CO]
    const int cx = xa ? ca : cf, cin = cx + (ex ? 1 : 0);
    const int nw = K * K * cin * CO;
    for (int e = threadIdx.x; e < nw; e += blockDim.x) s_w[e] = wk[e];
    __syncthreads();
    const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= (long long)N * H * W) return;
    const int X = (int)(pix % W), Y = (int)((pix / W) % H), n = (int)(pix / ((long long)W * H));
    float acc[CO];
#pragma unroll
    for (int o = 0; o < CO; ++o) acc[o] = bias[o];
    const int r = K / 2;
    for (int ky = 0; ky < K; ++ky) {
        const int yy = Y + ky - r;
        if (yy < 0 || yy >= H) continue;
        for (int kx = 0; kx < K; ++kx) {
            const int xx = X + kx - r;
            if (xx < 0 || xx >= W) continue;
            const float* wt = s_w + (size_t)(ky * K + kx) * cin * CO;
            const size_t p = ((size_t)n * H + yy) * W + xx;
            if (xa) {
                const __half* xp = xa + p * sa;
                for (int c0 = 0; c0 < ca; c0 += 8) {
                    const uint4 hv = __ldg(reinterpret_cast<const uint4*>(xp + c0));
                    const __half2* h2 = reinterpret_cast<const __half2*>(&hv);
                    float v[8];
#pragma unroll
                    for (int j = 0; j < 4; ++j) { const float2 f = __half22float2(h2[j]); v[2 * j] = f.x; v[2 * j + 1] = f.y; }
                    if (lo_a) {
                        const uint4 lv = __ldg(reinterpret_cast<const uint4*>(xp + lo_a + c0));
                        const __half2* l2 = reinterpret_cast<const __half2*>(&lv);
#pragma unroll
                        for (int j = 0; j < 4; ++j) { const float2 f = __half22float2(l2[j]); v[2 * j] += f.x; v[2 * j + 1] += f.y; }
                    }
#pragma unroll
                    for (int j = 0; j < 8; ++j)
#pragma unroll
                        for (int o = 0; o < CO; ++o) acc[o] = fmaf(v[j], wt[(c0 + j) * CO + o], acc[o]);
                }
            } else {
                const float* xp = xf + p * sf;
                for (int c0 = 0; c0 < cf; c0 += 4) {
                    const float4 f = __ldg(reinterpret_cast<const float4*>(xp + c0));
                    const float v[4] = {f.x, f.y, f.z, f.w};
#pragma unroll
                    for (int j = 0; j < 4; ++j)
#pragma unroll
                        for (int o = 0; o < CO; ++o) acc[o] = fmaf(v[j], wt[(c0 + j) * CO + o], acc[o]);
                }
            }
            if (ex) {
                int y0, y1, x0, x1; float ty, tx;
                bilinear_coord(yy, eh, H, y0, y1, ty);
                bilinear_coord(xx, ew, W, x0, x1, tx);
                const float* ep = ex + (size_t)n * eh * ew;
                const float v = bilinear_mix(ep[y0 * ew + x0], ep[y1 * ew + x0], ep[y0 * ew + x1], ep[y1 * ew + x1], ty, tx);
#pragma unroll
                for (int o = 0; o < CO; ++o) acc[o] = fmaf(v, wt[cx * CO + o], acc[o]);
            }
        }
    }
#pragma unroll
    for (int o = 0; o < CO; ++o) {
        float v = acc[o];
        if (act == 1) v = fmaxf(v, 0.f);
        else if (act == 2) v = 1.f / (1.f + expf(-v));
        if (nchw) out[(((size_t)n * CO + o) * H + Y) * W + X] = v;
        else out[(size_t)pix * CO + o] = v;
    }
}

// NHWC fp16 [N][H][W][cs] (channels 0..C-1, + the split remainder at channel lo + c when lo > 0) -> NCHW fp32 [N][C][H][W]
__global__ void tw_hid_to_nchw_kernel(const __half* __restrict__ x, int N, int C, int H, int W, int cs, int lo, float* __restrict__ y) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * C * H * W) return;
    const int c = (int)(idx % C);
    const long long p = idx / C;                                                // n*H*W + pixel
    const int n = (int)(p / ((long long)H * W));
    const long long hw = p - (long long)n * H * W;
    float v = __half2float(x[(size_t)p * cs + c]);
    if (lo) v += __half2float(x[(size_t)p * cs + lo + c]);
    y[((size_t)n * C + c) * H * W + hw] = v;
}

}  // namespace tw
}  // namespace r3dp

using namespace r3dp;
using namespace r3dp::tw;

extern "C" int r3dp_tw_gather3d(const float* fs_ndhwc, int fs_shared, const float* grid, int N, int C, int D, int H, int W, void* y_f16, int split,
                                r3dp_stream_t stream) {
    R3DP_REQUIRE(fs_ndhwc && grid && y_f16, "tw_gather3d: null pointer");
    R3DP_REQUIRE(N > 0 && C > 0 && C % 4 == 0 && D > 1 && H > 1 && W > 1, "tw_gather3d: bad shape");
    const long long total = (long long)N * H * W * D;
    const int cs = C * D * (split ? 2 : 1);
    tw_gather3d_kernel<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(fs_ndhwc, grid, N, C, D, H, W, cs, split, fs_shared, reinterpret_cast<__half*>(y_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_tw_affine_relu(const void* x_f16, const float* scale, const float* shift, int N, int H, int W, int C, int split, void* y_f16,
                                   r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && scale && shift && y_f16, "tw_affine_relu: null pointer");
    R3DP_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0, "tw_affine_relu: bad shape");
    const long long P = (long long)N * H * W;
    tw_affine_relu_kernel<<<(unsigned)((P * C + 255) / 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<const __half*>(x_f16), scale, shift, P, C,
                                                                                         C * (split ? 2 : 1), split, reinterpret_cast<__half*>(y_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_tw_narrow_conv(const void* xa_f16, int sa, int ca, int lo_a, const float* xf, int sf, int cf, const float* ex, int eh, int ew,
                                   const float* wk, const float* bias, int N, int H, int W, int K, int CO, int act, int nchw, float* out,
                                   r3dp_stream_t stream) {
    R3DP_REQUIRE(wk && bias && out && ((xa_f16 != nullptr) != (xf != nullptr)), "tw_narrow_conv: null pointer / exactly one of xa, xf");
    R3DP_REQUIRE(N > 0 && H > 0 && W > 0 && (K == 1 || K == 3 || K == 5 || K == 7) && act >= 0 && act <= 2, "tw_narrow_conv: bad shape / options");
    R3DP_REQUIRE(xa_f16 ? (ca > 0 && ca % 8 == 0 && sa % 8 == 0 && lo_a % 8 == 0) : (cf > 0 && cf % 4 == 0 && sf % 4 == 0), "tw_narrow_conv: channel alignment");
    R3DP_REQUIRE(!ex || (eh > 0 && ew > 0), "tw_narrow_conv: extra channel shape");
    const int cin = (xa_f16 ? ca : cf) + (ex ? 1 : 0);
    const size_t smem = (size_t)K * K * cin * CO * sizeof(float);
    R3DP_REQUIRE(smem <= 200 * 1024, "tw_narrow_conv: weights over the shared-memory budget");
    const long long P = (long long)N * H * W;
    const unsigned grid = (unsigned)((P + kNarrowThreads - 1) / kNarrowThreads);
    cudaStream_t st = as_stream(stream);
    const __half* xa = reinterpret_cast<const __half*>(xa_f16);
#define R3DP_TW_NARROW(CO_)                                                                                                                 \
    R3DP_CUDA(cudaFuncSetAttribute(tw_narrow_conv_kernel<CO_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));                   \
    tw_narrow_conv_kernel<CO_><<<grid, kNarrowThreads, smem, st>>>(xa, sa, ca, lo_a, xf, sf, cf, ex, eh, ew, wk, bias, N, H, W, K, act, nchw, out)
    switch (CO) {
        case 1: R3DP_TW_NARROW(1); break;
        case 3: R3DP_TW_NARROW(3); break;
        case 32: R3DP_TW_NARROW(32); break;
        default: R3DP_REQUIRE(false, "tw_narrow_conv: CO must be 1, 3 or 32");
    }
#undef R3DP_TW_NARROW
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_tw_hid_to_nchw(const void* x_f16, int N, int C, int H, int W, int cs, int lo, float* y, r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && y, "tw_hid_to_nchw: null pointer");
    R3DP_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0 && lo >= 0 && cs >= (lo ? lo : 0) + C, "tw_hid_to_nchw: bad shape");
    const long long total = (long long)N * C * H * W;
    tw_hid_to_nchw_kernel<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<const __half*>(x_f16), N, C, H, W, cs, lo, y);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}
