// Exact-fp32 super-resolution building blocks (CUDA-core path).  This is the parity anchor for the SR stack: same
// arithmetic as the reference's fp32 modules (SURVEY.md App. A.8), NCHW fp32 activations, no tensor cores.  The
// tensor-core path (sr_tc.cu) is checked against the same oracle with its own, looser, stated tolerance.
#include "common.cuh"

namespace r3dp {

// ---- styles = affine(w) (networks_stylegan2.py:113-127) -----------------------------------------------------------
__global__ void sr_styles_kernel(const float* __restrict__ w_lat, const float* __restrict__ A, const float* __restrict__ a,
                                 int N, int w_dim, int Cin, float gain, float post, float* __restrict__ styles) {
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (gw >= N * Cin) return;
    const int n = gw / Cin, i = gw - n * Cin;
    float acc = 0.f;
    for (int k = lane; k < w_dim; k += 32) acc = fmaf(w_lat[(size_t)n * w_dim + k], __fmul_rn(A[(size_t)i * w_dim + k], gain), acc);
#pragma unroll
    for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) styles[gw] = (acc + a[i]) * post;
}

// ---- per-sample modulated (+demodulated) weights (networks_stylegan2.py:63-70) ------------------------------------
__global__ void sr_fold_kernel(const float* __restrict__ W, const float* __restrict__ styles, int O, int I, int kk,
                               int demod, float* __restrict__ wf) {
    const int n = blockIdx.y, o = blockIdx.x, tid = threadIdx.x;
    const int len = I * kk;
    const float* w = W + (size_t)o * len;
    const float* s = styles + (size_t)n * I;
    float* out = wf + ((size_t)n * O + o) * len;
    __shared__ float red[32];
    float sq = 0.f;
    for (int e = tid; e < len; e += blockDim.x) {
        const float v = __fmul_rn(w[e], s[e / kk]);
        out[e] = v;
        sq = fmaf(v, v, sq);
    }
    if (!demod) return;
#pragma unroll
    for (int off = 16; off; off >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, off);
    if ((tid & 31) == 0) red[tid >> 5] = sq;
    __syncthreads();
    if (tid < 32) {
        float v = tid < (blockDim.x >> 5) ? red[tid] : 0.f;
#pragma unroll
        for (int off = 16; off; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
        if (tid == 0) red[0] = 1.0f / sqrtf(v + 1e-8f);
    }
    __syncthreads();
    const float d = red[0];
    for (int e = tid; e < len; e += blockDim.x) out[e] *= d;     // same thread wrote out[e] above
}

// ---- bilinear up-resize (F.interpolate align_corners=False; antialias is the identity for scale >= 1) -------------
__global__ void sr_resize_kernel(const float* __restrict__ x, int NC, int h, int w, int size, float* __restrict__ y) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)NC * size * size) return;
    const int ox = (int)(idx % size), oy = (int)((idx / size) % size); const long long nc = idx / ((long long)size * size);
    int y0, y1, x0, x1;
    float ty, tx;
    bilinear_coord(oy, h, size, y0, y1, ty);
    bilinear_coord(ox, w, size, x0, x1, tx);
    const float* p = x + nc * h * w;
    y[idx] = bilinear_mix(p[y0 * w + x0], p[y1 * w + x0], p[y0 * w + x1], p[y1 * w + x1], ty, tx);
}

// ---- direct convolution over a tap list ---------------------------------------------------------------------------
// out position (I,J) of the (sub-)grid accumulates  sum_{ci,tap} x[ci][I+dy_tap][J+dx_tap] * wf[co][ci][widx_tap];
// 3x3 correlation (pad 1): 9 taps, dy=ky-1; transposed-conv phase (a,b): taps with ky%2==a, kx%2==b, dy=-(ky>>1).
struct ConvTaps {
    int n;
    int dy[9], dx[9], widx[9];
};
struct ConvArgs {
    const float* x; const float* wf; float* y;
    int I, O, H, W;            // input channels / output channels / input height / width
    int gh, gw;                // size of the (sub-)grid of output positions this launch covers
    int oy_mul, oy_off, ox_mul, ox_off, OH, OW;   // output pixel = (I*oy_mul+oy_off, J*ox_mul+ox_off) in an OH x OW image
    const float* bias;         // fused bias + lrelu(0.2)*sqrt(2) if non-null (up == 1 path)
    ConvTaps taps;
};

constexpr int kCT_TW = 32, kCT_TH = 16, kCT_CO = 32, kCT_CI = 8;

__global__ void __launch_bounds__(256) conv_taps_kernel(const ConvArgs a) {
    __shared__ float s_in[kCT_CI][kCT_TH + 2][kCT_TW + 2];
    __shared__ __align__(16) float s_w[kCT_CI][9][kCT_CO];
    const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;   // ty 0..7, rows ty and ty+8
    const int tiles_x = (a.gw + kCT_TW - 1) / kCT_TW;
    const int J0 = (blockIdx.x % tiles_x) * kCT_TW, I0 = (blockIdx.x / tiles_x) * kCT_TH;
    const int co0 = blockIdx.y * kCT_CO, n = blockIdx.z;
    const float* xn = a.x + (size_t)n * a.I * a.H * a.W;
    const float* wn = a.wf + (size_t)n * a.O * a.I * 9;
    float acc0[kCT_CO], acc1[kCT_CO];
#pragma unroll
    for (int c = 0; c < kCT_CO; ++c) { acc0[c] = 0.f; acc1[c] = 0.f; }

    for (int ci0 = 0; ci0 < a.I; ci0 += kCT_CI) {
        __syncthreads();
        for (int e = tid; e < kCT_CI * (kCT_TH + 2) * (kCT_TW + 2); e += 256) {
            const int c = e / ((kCT_TH + 2) * (kCT_TW + 2)), r = e % ((kCT_TH + 2) * (kCT_TW + 2));
            const int yy = I0 - 1 + r / (kCT_TW + 2), xx = J0 - 1 + r % (kCT_TW + 2);
            float v = 0.f;
            if (ci0 + c < a.I && (unsigned)yy < (unsigned)a.H && (unsigned)xx < (unsigned)a.W) v = xn[((size_t)(ci0 + c) * a.H + yy) * a.W + xx];
            (&s_in[0][0][0])[e] = v;
        }
        for (int e = tid; e < kCT_CI * a.taps.n * kCT_CO; e += 256) {
            const int co = e % kCT_CO, t = (e / kCT_CO) % a.taps.n, c = e / (kCT_CO * a.taps.n);
            float v = 0.f;
            if (ci0 + c < a.I && co0 + co < a.O) v = wn[((size_t)(co0 + co) * a.I + ci0 + c) * 9 + a.taps.widx[t]];
            s_w[c][t][co] = v;
        }
        __syncthreads();
#pragma unroll 1
        for (int c = 0; c < kCT_CI; ++c) {
#pragma unroll 1
            for (int t = 0; t < a.taps.n; ++t) {
                const float v0 = s_in[c][ty + 1 + a.taps.dy[t]][tx + 1 + a.taps.dx[t]];
                const float v1 = s_in[c][ty + 9 + a.taps.dy[t]][tx + 1 + a.taps.dx[t]];
                const float4* w4 = reinterpret_cast<const float4*>(&s_w[c][t][0]);
#pragma unroll
                for (int q = 0; q < kCT_CO / 4; ++q) {
                    const float4 w = w4[q];
                    acc0[4 * q + 0] = fmaf(v0, w.x, acc0[4 * q + 0]); acc1[4 * q + 0] = fmaf(v1, w.x, acc1[4 * q + 0]);
                    acc0[4 * q + 1] = fmaf(v0, w.y, acc0[4 * q + 1]); acc1[4 * q + 1] = fmaf(v1, w.y, acc1[4 * q + 1]);
                    acc0[4 * q + 2] = fmaf(v0, w.z, acc0[4 * q + 2]); acc1[4 * q + 2] = fmaf(v1, w.z, acc1[4 * q + 2]);
                    acc0[4 * q + 3] = fmaf(v0, w.w, acc0[4 * q + 3]); acc1[4 * q + 3] = fmaf(v1, w.w, acc1[4 * q + 3]);
                }
            }
        }
    }
    const int J = J0 + tx;
    if (J >= a.gw) return;
    const int X = J * a.ox_mul + a.ox_off;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        const int I = I0 + ty + half * 8;
        if (I >= a.gh) continue;
        const int Y = I * a.oy_mul + a.oy_off;
#pragma unroll
        for (int c = 0; c < kCT_CO; ++c) {
            if (co0 + c >= a.O) continue;
            float v = half ? acc1[c] : acc0[c];
            if (a.bias) {
                v += a.bias[co0 + c];
                v = (v < 0.f ? v * 0.2f : v) * 1.4142135623730951f;       // bias_act lrelu, def_gain sqrt(2)
            }
            a.y[(((size_t)n * a.O + co0 + c) * a.OH + Y) * a.OW + X] = v;
        }
    }
}

// ---- FIR (upfirdn2d pad 1, gain 4) + bias + lrelu after the transposed conv ----------------------------------------
__global__ void fir_bias_lrelu_kernel(const float* __restrict__ yb, const float* __restrict__ bias, int NO, int O, int OH, int OW,
                                      float* __restrict__ y) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)NO * OH * OW) return;
    const int ox = (int)(idx % OW), oy = (int)((idx / OW) % OH); const long long no = idx / ((long long)OH * OW);
    const int BH = OH + 1, BW = OW + 1;
    const float* p = yb + no * BH * BW;
    const float k[4] = {0.25f, 0.75f, 0.75f, 0.25f};                       // [1,3,3,1]/4 per axis: (f (x) f / 64) * gain 4
    float acc = 0.f;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int yy = oy + u - 1;
        if ((unsigned)yy >= (unsigned)BH) continue;
        float row = 0.f;
#pragma unroll
        for (int v = 0; v < 4; ++v) {
            const int xx = ox + v - 1;
            if ((unsigned)xx < (unsigned)BW) row = fmaf(k[v], p[(size_t)yy * BW + xx], row);
        }
        acc = fmaf(k[u], row, acc);
    }
    acc += bias[(int)(no % O)];
    y[idx] = (acc < 0.f ? acc * 0.2f : acc) * 1.4142135623730951f;
}

// ---- ToRGB (1x1 modulated conv, no demod) + bias + FIR-upsampled skip image ----------------------------------------
__global__ void __launch_bounds__(256) torgb_kernel(const float* __restrict__ x, const float* __restrict__ wf, const float* __restrict__ bias,
                                                    const float* __restrict__ img_in, int I, int H, int W, float* __restrict__ img_out) {
    extern __shared__ float s_w[];                                         // [3][I]
    const int n = blockIdx.y;
    for (int e = threadIdx.x; e < 3 * I; e += blockDim.x) s_w[e] = wf[(size_t)n * 3 * I + e];
    __syncthreads();
    const int pix = blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= H * W) return;
    const int Y = pix / W, X = pix - Y * W;
    const float* xp = x + (size_t)n * I * H * W + pix;
    float r = 0.f, g = 0.f, b = 0.f;
    for (int i = 0; i < I; ++i) {
        const float v = xp[(size_t)i * H * W];
        r = fmaf(v, s_w[i], r); g = fmaf(v, s_w[I + i], g); b = fmaf(v, s_w[2 * I + i], b);
    }
    float out[3] = {r + bias[0], g + bias[1], b + bias[2]};
    if (img_in) {
        // upsample2d: z = zero-insert x2 (z[2i][2j] = img[i][j]); out[Y][X] += sum_{u,v} k[u]k[v] z[Y+u-2][X+v-2]
        const int h = H / 2, w = W / 2;
        const float k[4] = {0.25f, 0.75f, 0.75f, 0.25f};
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float* ip = img_in + ((size_t)n * 3 + c) * h * w;
            float acc = 0.f;
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int zy = Y + u - 2;
                if (zy < 0 || (zy & 1) || (zy >> 1) >= h) continue;
                float row = 0.f;
#pragma unroll
                for (int v = 0; v < 4; ++v) {
                    const int zx = X + v - 2;
                    if (zx < 0 || (zx & 1) || (zx >> 1) >= w) continue;
                    row = fmaf(k[v], ip[(size_t)(zy >> 1) * w + (zx >> 1)], row);
                }
                acc = fmaf(k[u], row, acc);
            }
            out[c] += acc;
        }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) img_out[((size_t)n * 3 + c) * H * W + pix] = out[c];
}

static int launch_conv(const ConvArgs& a, int N, cudaStream_t st) {
    const int tiles = ((a.gw + kCT_TW - 1) / kCT_TW) * ((a.gh + kCT_TH - 1) / kCT_TH);
    dim3 grid(tiles, (a.O + kCT_CO - 1) / kCT_CO, N);
    conv_taps_kernel<<<grid, 256, 0, st>>>(a);
    count_launches(1);
    R3DP_LAUNCH_CHECK();
    return 0;
}

}  // namespace r3dp

using namespace r3dp;

extern "C" int r3dp_sr_styles(const float* w_lat, const float* affine_w, const float* affine_b, int N, int w_dim, int Cin,
                              float post_scale, float* styles, r3dp_stream_t stream) {
    R3DP_REQUIRE(w_lat && affine_w && affine_b && styles, "sr_styles: null pointer");
    R3DP_REQUIRE(N > 0 && w_dim > 0 && Cin > 0, "sr_styles: bad shape");
    const int warps = N * Cin;
    sr_styles_kernel<<<(warps * 32 + 255) / 256, 256, 0, as_stream(stream)>>>(w_lat, affine_w, affine_b, N, w_dim, Cin,
                                                                              1.0f / sqrtf((float)w_dim), post_scale, styles);
    count_launches(1);
    R3DP_LAUNCH_CHECK();
    return 0;
}

extern "C" int r3dp_sr_fold_weights(const float* weight, const float* styles, int N, int O, int I, int k, int demodulate,
                                    float* wf, r3dp_stream_t stream) {
    R3DP_REQUIRE(weight && styles && wf, "sr_fold_weights: null pointer");
    R3DP_REQUIRE(N > 0 && O > 0 && I > 0 && (k == 1 || k == 3), "sr_fold_weights: bad shape (k must be 1 or 3)");
    dim3 grid(O, N);
    sr_fold_kernel<<<grid, 256, 0, as_stream(stream)>>>(weight, styles, O, I, k * k, demodulate, wf);
    count_launches(1);
    R3DP_LAUNCH_CHECK();
    return 0;
}

extern "C" int r3dp_sr_resize_bilinear(const float* x, int N, int C, int h, int w, int size, float* y, r3dp_stream_t stream) {
    R3DP_REQUIRE(x && y, "sr_resize_bilinear: null pointer");
    R3DP_REQUIRE(N > 0 && C > 0 && h > 0 && w > 0 && size >= h && size >= w, "sr_resize_bilinear: up-scaling only (%dx%d -> %d)", h, w, size);
    const long long total = (long long)N * C * size * size;
    sr_resize_kernel<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(x, N * C, h, w, size, y);
    count_launches(1);
    R3DP_LAUNCH_CHECK();
    return 0;
}

extern "C" size_t r3dp_sr_layer_scratch_bytes(int N, int O, int H, int W) {
    return (size_t)N * O * (2 * H + 1) * (2 * W + 1) * sizeof(float);
}

extern "C" int r3dp_sr_layer_fp32(const float* x, const float* wf, const float* bias, int N, int I, int O, int H, int W, int up,
                                  float* y, void* scratch, r3dp_stream_t stream) {
    R3DP_REQUIRE(x && wf && bias && y, "sr_layer_fp32: null pointer");
    R3DP_REQUIRE(N > 0 && I > 0 && O > 0 && H > 0 && W > 0, "sr_layer_fp32: bad shape");
    R3DP_REQUIRE(up == 1 || up == 2, "sr_layer_fp32: up must be 1 or 2 (got %d)", up);
    cudaStream_t st = as_stream(stream);
    ConvArgs a;
    a.x = x; a.wf = wf; a.I = I; a.O = O; a.H = H; a.W = W;
    if (up == 1) {
        a.y = y; a.gh = H; a.gw = W; a.oy_mul = a.ox_mul = 1; a.oy_off = a.ox_off = 0; a.OH = H; a.OW = W; a.bias = bias;
        a.taps.n = 9;
        for (int t = 0; t < 9; ++t) { a.taps.dy[t] = t / 3 - 1; a.taps.dx[t] = t % 3 - 1; a.taps.widx[t] = t; }
        return launch_conv(a, N, st);
    }
    R3DP_REQUIRE(scratch, "sr_layer_fp32: up=2 needs scratch (r3dp_sr_layer_scratch_bytes)");
    float* yb = reinterpret_cast<float*>(scratch);
    a.y = yb; a.OH = 2 * H + 1; a.OW = 2 * W + 1; a.bias = nullptr; a.oy_mul = a.ox_mul = 2;
    for (int pa = 0; pa < 2; ++pa)
        for (int pb = 0; pb < 2; ++pb) {
            a.oy_off = pa; a.ox_off = pb; a.gh = pa ? H : H + 1; a.gw = pb ? W : W + 1;
            a.taps.n = 0;
            for (int ky = pa; ky < 3; ky += 2)
                for (int kx = pb; kx < 3; kx += 2) {
                    const int t = a.taps.n++;
                    a.taps.dy[t] = -(ky >> 1); a.taps.dx[t] = -(kx >> 1); a.taps.widx[t] = ky * 3 + kx;
                }
            if (launch_conv(a, N, st)) return 1;
        }
    const long long total = (long long)N * O * (2 * H) * (2 * W);
    fir_bias_lrelu_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(yb, bias, N * O, O, 2 * H, 2 * W, y);
    count_launches(1);
    R3DP_LAUNCH_CHECK();
    return 0;
}

extern "C" int r3dp_sr_torgb_fp32(const float* x, const float* wf_rgb, const float* bias, const float* img_in, int N, int I,
                                  int H, int W, float* img_out, r3dp_stream_t stream) {
    R3DP_REQUIRE(x && wf_rgb && bias && img_out, "sr_torgb_fp32: null pointer");
    R3DP_REQUIRE(N > 0 && I > 0 && H > 0 && W > 0 && (!img_in || (H % 2 == 0 && W % 2 == 0)), "sr_torgb_fp32: bad shape");
    dim3 grid((H * W + 255) / 256, N);
    torgb_kernel<<<grid, 256, 3 * I * sizeof(float), as_stream(stream)>>>(x, wf_rgb, bias, img_in, I, H, W, img_out);
    count_launches(1);
    R3DP_LAUNCH_CHECK();
    return 0;
}
