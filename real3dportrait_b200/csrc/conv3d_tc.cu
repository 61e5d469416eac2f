// The torso warper's motion-field estimator (modules/real3d/facev2v_warp/network2.py:162-244, MotionFieldEstimator('standard')) on sm_90a.
//   conv3d_tc_kernel      3-D implicit-GEMM convolution on wgmma: every conv of the estimator (down / up blocks, the tgt-head encoder, the
//                         fuser and mask convs).  Box taps KD x KH x KW; the nearest-(1,2,2)-up convs run as 4 output-parity phases of
//                         3x2x2 taps on the low-resolution input (one phase per blockIdx.y).
//   mf_input_kernel       heatmap differences + trilinear-deformed compressed source -> the (K+1)*5 input channels (func_utils.py:130-191)
//   mf_pool_kernel        AvgPool3d (1,2,2) on NDHWC fp16 / split (layers.py:58-74)
//   mf_head_input_kernel  2x2 mean of [rgb_256 | weights_256] (the exact-1/2 bilinear resize to 128^2) -> NHWC
//   mf_head_bcast_kernel  2x2 mean of the 128^2 head features, broadcast over depth into the fuser input
//   mf_deform_kernel      softmax over the K+1 mask logits, deformation = sum_k mask_k * sparse_motion_k
//   mf_occlusion_kernel   occlusion_conv / occlusion_conv2: 7x7 2-D convs over the (c*D + d) view of the fuser output, fp32, sigmoid
//
// Activations are NDHWC fp16 with a voxel stride of any multiple of 8 halves; the split (tc_exact) form keeps the fp16 remainder of every
// value at a fixed offset `lo` inside the same voxel ([hi | lo]).  Split weights are stored x 2^10 as [hi | lo] (kSplitScale3).
#include "common.cuh"
#include "tc_prims.cuh"
#include <cuda_fp16.h>

namespace r3dp {
namespace c3 {
using namespace r3dp::tc;

constexpr int kBM = 128;                 // output voxels per CTA (two consumer warpgroups of 64)
constexpr int kBK = 32;                  // channels per K step: one 64-byte row of the 64-byte-swizzled operand tiles
constexpr int kStages = 4;               // ring depth; loads run 2 stages ahead of the MMAs, one MMA group stays in flight
constexpr int kThreads = 256;
constexpr float kSplitScale3 = 1024.0f;

struct Conv3dArgs {
    const __half* x;                     // input NDHWC [N][D][H][W] voxels of xs halves; channels [0, cin) read (split: + lo half at xlo)
    const __half* w;                     // packed [nph][taps][cop][kw] fp16, kw = cin (split: 2 cin = [hi | lo] of w * 2^10)
    const float* bias;                   // [cop]
    const __half* res;                   // residual in the output's layout (voxel stride ys, channel offset yc0, split lo at ylo), or null
    void* y;                             // output: fp16 (split: [hi | lo]) or fp32 (out_f32)
    int N, D, H, W;                      // the GEMM's M space: the INPUT grid (stride-1 convs: also the output grid)
    int xs, xlo, cin;
    int kd, kh, kw, oz, oy, ox;          // taps dz in [-oz, kd - oz) etc.; phase (p, q) shifts the origin to oy - p, ox - q
    int sy, sx;                          // output voxel (d, h * sy + p, w * sx + q) of a grid D x H*sy x W*sx
    int ys, yc0, ylo, cout, cop;
    int relu, out_f32;                   // relu: 0 none, 1 ReLU, 2 exact GELU
    float acc_scale;
};

// byte offset of 16-byte chunk j of row r in a K-major tile of 64-byte rows, 64-byte swizzle (cute Swizzle<2,4,3>)
__device__ __forceinline__ uint32_t sw64(int r, int j) { return (uint32_t)(r * 64 + ((j ^ ((r >> 1) & 3)) << 4)); }

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool ok) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(ok ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void wgmma_m64n16k16(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_m64n32k16(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
          "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b), "r"(acc));
}
template <int BN>
__device__ __forceinline__ void wgmma_n(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    if constexpr (BN == 16) wgmma_m64n16k16(d, a, b, acc);
    else if constexpr (BN == 32) wgmma_m64n32k16(d, a, b, acc);
    else if constexpr (BN == 64) wgmma_m64n64k16(d, a, b, acc);
    else wgmma_m64n128k16(d, a, b, acc);
}

template <int BN, bool SPLIT>
struct Cfg {
    static constexpr int NH = SPLIT ? 2 : 1;                     // operand halves per stage
    static constexpr int A_BYTES = kBM * 64, B_BYTES = BN * 64;
    static constexpr int STAGE = NH * (A_BYTES + B_BYTES);       // a multiple of 1024 (BN >= 16)
    static constexpr int SMEM = kStages * STAGE + 1024;
};

// CTA = 128 consecutive voxels of the M space (n, d, h, w order) x BN couts of one phase.  All 256 threads fill the ring with cp.async
// (zero fill outside the input = the conv's zero padding); warpgroup g runs the MMAs of rows [64 g, 64 g + 64).
// K order: tap-major, 32-channel chunk minor.  Split: per chunk x_hi w_hi + x_lo w_hi + x_hi w_lo.
template <int BN, bool SPLIT>
__global__ void __launch_bounds__(kThreads) conv3d_tc_kernel(const Conv3dArgs a) {
    using C = Cfg<BN, SPLIT>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = align_smem_1024(smem_raw);
    const int tid = threadIdx.x, wg = tid >> 7;
    const int ph = blockIdx.y, p = ph >> 1, q = ph & 1;
    const int n0 = blockIdx.z * BN;
    const long long M = (long long)a.N * a.D * a.H * a.W;
    const int oy = a.oy - p, ox = a.ox - q;
    const int taps = a.kd * a.kh * a.kw, chunks = a.cin / kBK, KI = taps * chunks;
    const __half* wph = a.w + (size_t)ph * taps * a.cop * (SPLIT ? 2 : 1) * a.cin;
    const int kwid = (SPLIT ? 2 : 1) * a.cin;                    // halves per packed weight row

    // this thread's A row and the two 16-byte chunks it copies
    const int ar = tid & 127, aj = (tid >> 7) * 2;
    const long long am = (long long)blockIdx.x * kBM + ar;
    const bool arow_ok = am < M;
    int an = 0, ad = 0, ah = 0, aw = 0;
    if (arow_ok) {
        long long t = am;
        aw = (int)(t % a.W); t /= a.W;
        ah = (int)(t % a.H); t /= a.H;
        ad = (int)(t % a.D); an = (int)(t / a.D);
    }

    auto load_stage = [&](int it, int slot) {
        const int tap = it / chunks, ch = it - tap * chunks;
        const int ix = tap % a.kw, iy = (tap / a.kw) % a.kh, iz = tap / (a.kw * a.kh);
        const int zz = ad + iz - a.oz, yy = ah + iy - oy, xx = aw + ix - ox;
        const bool ok = arow_ok && zz >= 0 && zz < a.D && yy >= 0 && yy < a.H && xx >= 0 && xx < a.W;
        const __half* src = ok ? a.x + ((((size_t)an * a.D + zz) * a.H + yy) * a.W + xx) * a.xs + ch * kBK : a.x;
        const uint32_t base = smem_u32(smem + slot * C::STAGE);
#pragma unroll
        for (int hh = 0; hh < C::NH; ++hh)
#pragma unroll
            for (int j = 0; j < 2; ++j)
                cp_async16(base + hh * C::A_BYTES + sw64(ar, aj + j), ok ? src + hh * a.xlo + (aj + j) * 8 : a.x, ok);
        const uint32_t bbase = base + C::NH * C::A_BYTES;
        const __half* wt = wph + (size_t)tap * a.cop * kwid + ch * kBK;
        for (int e = tid; e < BN * 4 * C::NH; e += kThreads) {
            const int hh = e / (BN * 4), r = (e >> 2) % BN, j = e & 3;
            const int co = n0 + r;
            const bool okb = co < a.cop;
            cp_async16(bbase + hh * C::B_BYTES + sw64(r, j), okb ? wt + (size_t)co * kwid + hh * a.cin + j * 8 : a.w, okb);
        }
    };

    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;

#pragma unroll
    for (int s = 0; s < kStages - 2; ++s) {
        if (s < KI) load_stage(s, s);
        cp_async_commit();
    }
    for (int it = 0; it < KI; ++it) {
        cp_async_wait<kStages - 3>();                             // this thread's copies of stage `it` have landed
        fence_proxy_async();                                      // ... and are visible to the tensor core's async proxy
        __syncthreads();                                          // every thread's copies; every warpgroup is done with the MMAs of it - 2
        if (it + kStages - 2 < KI) load_stage(it + kStages - 2, (it + kStages - 2) % kStages);
        cp_async_commit();
        const uint32_t base = smem_u32(smem + (it % kStages) * C::STAGE);
        const uint32_t sa = base + wg * 64 * 64, sb = base + C::NH * C::A_BYTES;
        wg_fence_acc<BN / 2>(acc);
        wg_fence();
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const uint64_t dah = gmma_desc_sw64(sa + 32 * k), dbh = gmma_desc_sw64(sb + 32 * k);
            wgmma_n<BN>(acc, dah, dbh, (it | k) ? 1u : 0u);
            if constexpr (SPLIT) {
                wgmma_n<BN>(acc, gmma_desc_sw64(sa + C::A_BYTES + 32 * k), dbh, 1u);
                wgmma_n<BN>(acc, dah, gmma_desc_sw64(sb + C::B_BYTES + 32 * k), 1u);
            }
        }
        wg_commit();
        wg_wait<1>();
        wg_fence_acc<BN / 2>(acc);
    }
    wg_wait<0>();
    wg_fence_acc<BN / 2>(acc);
    cp_async_wait<0>();

    // epilogue on the accumulator fragments: bias, ReLU, residual, then the store
#pragma unroll
    for (int i = 0; i < BN / 2; i += 2) {
        const int row = 64 * wg + acc_row(i), col = n0 + acc_col(i);
        const long long m = (long long)blockIdx.x * kBM + row;
        if (m >= M || col >= a.cout) continue;
        long long t = m;
        const int w = (int)(t % a.W); t /= a.W;
        const int h = (int)(t % a.H); t /= a.H;
        const int d = (int)(t % a.D), n = (int)(t / a.D);
        const size_t vox = (((size_t)n * a.D + d) * (a.H * a.sy) + h * a.sy + p) * (a.W * a.sx) + w * a.sx + q;
        const size_t off = vox * a.ys + a.yc0 + col;
        const bool two = col + 1 < a.cout;
        float v[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            float u = SPLIT ? __fmaf_rn(acc[i + e], a.acc_scale, a.bias[col + (two ? e : 0)]) : __fadd_rn(acc[i + e], a.bias[col + (two ? e : 0)]);
            if (a.relu == 1) u = fmaxf(u, 0.f);
            else if (a.relu == 2) u = 0.5f * u * (1.f + erff(u * 0.70710678118654752f));   // nn.GELU() (exact erf form)
            v[e] = u;
        }
        if (a.res) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                if (e && !two) break;
                float r = __half2float(a.res[off + e]);
                if (SPLIT) r += __half2float(a.res[off + a.ylo + e]);
                v[e] += r;
            }
        }
        if (a.out_f32) {
            float* y = reinterpret_cast<float*>(a.y) + off;
            y[0] = v[0];
            if (two) y[1] = v[1];
        } else {
            __half* y = reinterpret_cast<__half*>(a.y) + off;
            const __half h0 = __float2half_rn(v[0]), h1 = __float2half_rn(v[1]);
            if (two) *reinterpret_cast<__half2*>(y) = __halves2half2(h0, h1);
            else y[0] = h0;
            if (SPLIT) {
                const __half l0 = __float2half_rn(v[0] - __half2float(h0)), l1 = __float2half_rn(v[1] - __half2float(h1));
                if (two) *reinterpret_cast<__half2*>(y + a.ylo) = __halves2half2(l0, l1);
                else y[a.ylo] = l0;
            }
        }
    }
}

// ---- the kernels around the convolutions ------------------------------------------------------------------------------------------
__device__ __forceinline__ void put(__half* y, int lo, int split, float v) {
    const __half h = __float2half_rn(v);
    y[0] = h;
    if (split) y[lo] = __float2half_rn(v - __half2float(h));
}
__device__ __forceinline__ float get(const __half* x, int lo, int split) { return __half2float(x[0]) + (split ? __half2float(x[lo]) : 0.f); }
// make_coordinate_grid_3d (func_utils.py:91-103): component 0 runs along W, 1 along H, 2 along D, each 2 * (i / (n - 1)) - 1
__device__ __forceinline__ float grid_coord(int i, int n) { return 2.f * ((float)i / (float)(n - 1)) - 1.f; }

// One thread per voxel (n, d, h, w).  fc: the compressed source [Nf][D][H][W][4] fp32 (Nf = 1: one volume for the clip), kp_s / kp_d [N][K][3].
// Channel k*5 + j of the output (voxel stride ys, split lo at ylo): j = 0 the heatmap difference gauss(kp_d[k-1]) - gauss(kp_s[k-1]) (zeros
// for k = 0), j = 1..4 the compressed source sampled at sparse_motion_k (F.grid_sample trilinear, zeros padding, align_corners=True; k = 0 is
// the identity grid).  Channels (K+1)*5 .. cpad-1 are written as zeros.
__global__ void __launch_bounds__(128) mf_input_kernel(const float* __restrict__ fc, int fc_shared, const float* __restrict__ kp_s,
                                                       const float* __restrict__ kp_d, int N, int K, int D, int H, int W, int cpad, int ys, int ylo,
                                                       int split, __half* __restrict__ y) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * D * H * W) return;
    long long t = idx;
    const int w = (int)(t % W); t /= W;
    const int h = (int)(t % H); t /= H;
    const int d = (int)(t % D), n = (int)(t / D);
    const float gx = grid_coord(w, W), gy = grid_coord(h, H), gz = grid_coord(d, D);
    const float* vol = fc + (size_t)(fc_shared ? 0 : n) * D * H * W * 4;
    __half* out = y + (size_t)idx * ys;
    for (int k = 0; k <= K; ++k) {
        float sx = gx, sy = gy, sz = gz, hm = 0.f;
        if (k > 0) {
            const float* ps = kp_s + ((size_t)n * K + k - 1) * 3;
            const float* pd = kp_d + ((size_t)n * K + k - 1) * 3;
            const float ddx = gx - pd[0], ddy = gy - pd[1], ddz = gz - pd[2];
            const float dsx = gx - ps[0], dsy = gy - ps[1], dsz = gz - ps[2];
            hm = expf(-0.5f * (ddx * ddx + ddy * ddy + ddz * ddz) / 0.01f) - expf(-0.5f * (dsx * dsx + dsy * dsy + dsz * dsz) / 0.01f);
            sx = ddx + ps[0]; sy = ddy + ps[1]; sz = ddz + ps[2];
        }
        put(out + k * 5, ylo, split, hm);
        // grid_sampler_3d, align_corners: unnormalize, 8 corners, out-of-range corners contribute zero
        const float ix = (sx + 1.f) / 2.f * (float)(W - 1), iy = (sy + 1.f) / 2.f * (float)(H - 1), iz = (sz + 1.f) / 2.f * (float)(D - 1);
        const float fx = floorf(ix), fy = floorf(iy), fz = floorf(iz);
        const int x0 = (int)fx, y0 = (int)fy, z0 = (int)fz;
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const int dz = c >> 2, dy = (c >> 1) & 1, dx = c & 1;
            const int xx = x0 + dx, yy = y0 + dy, zz = z0 + dz;
            if (xx < 0 || xx >= W || yy < 0 || yy >= H || zz < 0 || zz >= D) continue;
            const float wt = (dx ? ix - fx : fx + 1.f - ix) * (dy ? iy - fy : fy + 1.f - iy) * (dz ? iz - fz : fz + 1.f - iz);
            const float4 v = __ldg(reinterpret_cast<const float4*>(vol + (((size_t)zz * H + yy) * W + xx) * 4));
            acc[0] += v.x * wt; acc[1] += v.y * wt; acc[2] += v.z * wt; acc[3] += v.w * wt;
        }
#pragma unroll
        for (int c = 0; c < 4; ++c) put(out + k * 5 + 1 + c, ylo, split, acc[c]);
    }
    for (int c = (K + 1) * 5; c < cpad; ++c) put(out + c, ylo, split, 0.f);
}

// AvgPool3d((1,2,2)): x [N*D][2H][2W] voxels of stride xs, C channels (split lo at xlo) -> y [N*D][H][W] of stride ys (lo at ylo)
__global__ void mf_pool_kernel(const __half* __restrict__ x, long long ND, int H, int W, int C, int xs, int xlo, int ys, int ylo, int split,
                               __half* __restrict__ y) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= ND * H * W * C) return;
    const int c = (int)(idx % C);
    long long t = idx / C;
    const int w = (int)(t % W); t /= W;
    const int h = (int)(t % H);
    const long long nd = t / H;
    const __half* p = x + (((size_t)nd * 2 * H + 2 * h) * 2 * W + 2 * w) * xs + c;
    const size_t rs = (size_t)2 * W * xs;
    const float v = ((get(p, xlo, split) + get(p + xs, xlo, split)) + (get(p + rs, xlo, split) + get(p + rs + xs, xlo, split))) * 0.25f;
    put(y + (((size_t)nd * H + h) * W + w) * ys + c, ylo, split, v);
}

// tgt_head_inp = interpolate(cat[rgb, weights], 128, bilinear) at exactly 1/2: mean of each 2x2 block.  rgb [N,3,2H,2W], wts [N,1,2H,2W]
// fp32 -> y [N][H][W] voxels of stride ys: channels 0..3, zeros up to cpad.
__global__ void mf_head_input_kernel(const float* __restrict__ rgb, const float* __restrict__ wts, int N, int H, int W, int cpad, int ys, int ylo,
                                     int split, __half* __restrict__ y) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * H * W) return;
    const int w = (int)(idx % W), h = (int)((idx / W) % H), n = (int)(idx / ((long long)W * H));
    __half* out = y + (size_t)idx * ys;
    for (int c = 0; c < 4; ++c) {
        const float* s = (c < 3 ? rgb + ((size_t)n * 3 + c) * 4 * H * W : wts + (size_t)n * 4 * H * W) + (size_t)(2 * h) * 2 * W + 2 * w;
        put(out + c, ylo, split, ((s[0] + s[1]) + (s[2 * W] + s[2 * W + 1])) * 0.25f);
    }
    for (int c = 4; c < cpad; ++c) put(out + c, ylo, split, 0.f);
}

// the head features x [N][2H][2W] (stride xs, C channels) -> 2x2 mean -> y[n][d][h][w][yc0 + c] for every d < D (the depth repeat)
__global__ void mf_head_bcast_kernel(const __half* __restrict__ x, int N, int D, int H, int W, int C, int xs, int xlo, int ys, int yc0, int ylo,
                                     int split, __half* __restrict__ y) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * H * W * C) return;
    const int c = (int)(idx % C);
    long long t = idx / C;
    const int w = (int)(t % W); t /= W;
    const int h = (int)(t % H), n = (int)(t / H);
    const __half* p = x + (((size_t)n * 2 * H + 2 * h) * 2 * W + 2 * w) * xs + c;
    const size_t rs = (size_t)2 * W * xs;
    const float v = ((get(p, xlo, split) + get(p + xs, xlo, split)) + (get(p + rs, xlo, split) + get(p + rs + xs, xlo, split))) * 0.25f;
    for (int d = 0; d < D; ++d) put(y + ((((size_t)n * D + d) * H + h) * W + w) * ys + yc0 + c, ylo, split, v);
}

// mask = softmax over the K+1 logits (fp32, voxel stride ls); deformation[n][d][h][w][3] = sum_k mask_k * sparse_motion_k
__global__ void mf_deform_kernel(const float* __restrict__ logits, int ls, const float* __restrict__ kp_s, const float* __restrict__ kp_d, int N, int K,
                                 int D, int H, int W, float* __restrict__ def) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * D * H * W) return;
    long long t = idx;
    const int w = (int)(t % W); t /= W;
    const int h = (int)(t % H); t /= H;
    const int d = (int)(t % D), n = (int)(t / D);
    const float* l = logits + (size_t)idx * ls;
    float mx = l[0];
    for (int k = 1; k <= K; ++k) mx = fmaxf(mx, l[k]);
    float den = 0.f;
    for (int k = 0; k <= K; ++k) den += expf(l[k] - mx);
    const float g[3] = {grid_coord(w, W), grid_coord(h, H), grid_coord(d, D)};
    float o[3] = {0.f, 0.f, 0.f};
    for (int k = 0; k <= K; ++k) {
        const float m = expf(l[k] - mx) / den;
        for (int c = 0; c < 3; ++c) {
            const float s = k == 0 ? g[c] : g[c] - kp_d[((size_t)n * K + k - 1) * 3 + c] + kp_s[((size_t)n * K + k - 1) * 3 + c];
            o[c] += s * m;
        }
    }
    for (int c = 0; c < 3; ++c) def[(size_t)idx * 3 + c] = o[c];
}

// occlusion_conv and occlusion_conv2 (7x7, C*D -> 1 each, sigmoid) on x.view(N, C*D, H, W) of the fuser output x [N][D][H][W][C] (stride xs,
// split lo at xlo): input channel c*D + d.  One thread per output pixel, both outputs; the weights of one depth slice [49][C][2] are staged
// in shared memory per pass over d.  wk fp32 [D][49][C][2] (tap-major), bias[2].
constexpr int kOccThreads = 128;
__global__ void __launch_bounds__(kOccThreads) mf_occlusion_kernel(const __half* __restrict__ x, int N, int D, int H, int W, int C, int xs, int xlo,
                                                                   int split, const float* __restrict__ wk, const float* __restrict__ bias,
                                                                   float* __restrict__ occ, float* __restrict__ occ2) {
    extern __shared__ float s_w[];
    const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = pix < (long long)N * H * W;
    const int X = live ? (int)(pix % W) : 0, Y = live ? (int)((pix / W) % H) : 0, n = live ? (int)(pix / ((long long)W * H)) : 0;
    float a0 = 0.f, a1 = 0.f;
    const int nw = 49 * C * 2;
    for (int d = 0; d < D; ++d) {
        __syncthreads();
        for (int e = threadIdx.x; e < nw; e += blockDim.x) s_w[e] = wk[(size_t)d * nw + e];
        __syncthreads();
        if (!live) continue;
        for (int ky = 0; ky < 7; ++ky) {
            const int yy = Y + ky - 3;
            if (yy < 0 || yy >= H) continue;
            for (int kx = 0; kx < 7; ++kx) {
                const int xx = X + kx - 3;
                if (xx < 0 || xx >= W) continue;
                const __half* xp = x + ((((size_t)n * D + d) * H + yy) * W + xx) * xs;
                const float* wt = s_w + (ky * 7 + kx) * C * 2;
                for (int c0 = 0; c0 < C; c0 += 8) {
                    const uint4 hv = __ldg(reinterpret_cast<const uint4*>(xp + c0));
                    const __half2* h2 = reinterpret_cast<const __half2*>(&hv);
                    float v[8];
#pragma unroll
                    for (int j = 0; j < 4; ++j) { const float2 f = __half22float2(h2[j]); v[2 * j] = f.x; v[2 * j + 1] = f.y; }
                    if (split) {
                        const uint4 lv = __ldg(reinterpret_cast<const uint4*>(xp + xlo + c0));
                        const __half2* l2 = reinterpret_cast<const __half2*>(&lv);
#pragma unroll
                        for (int j = 0; j < 4; ++j) { const float2 f = __half22float2(l2[j]); v[2 * j] += f.x; v[2 * j + 1] += f.y; }
                    }
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        a0 = fmaf(v[j], wt[(c0 + j) * 2], a0);
                        a1 = fmaf(v[j], wt[(c0 + j) * 2 + 1], a1);
                    }
                }
            }
        }
    }
    if (!live) return;
    occ[pix] = 1.f / (1.f + expf(-(a0 + bias[0])));
    occ2[pix] = 1.f / (1.f + expf(-(a1 + bias[1])));
}

template <int BN, bool SPLIT>
static int launch_conv(const Conv3dArgs& a, int nph, cudaStream_t st) {
    using C = Cfg<BN, SPLIT>;
    R3DP_CUDA(cudaFuncSetAttribute(conv3d_tc_kernel<BN, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM));
    const long long M = (long long)a.N * a.D * a.H * a.W;
    const dim3 grid((unsigned)((M + kBM - 1) / kBM), (unsigned)nph, (unsigned)((a.cout + BN - 1) / BN));
    conv3d_tc_kernel<BN, SPLIT><<<grid, kThreads, C::SMEM, st>>>(a);
    return 0;
}

}  // namespace c3
}  // namespace r3dp

using namespace r3dp;
using namespace r3dp::c3;

extern "C" int r3dp_mf_conv3d(const void* x_f16, int xs, int xlo, int cin, const void* wp_f16, const float* bias, const void* res_f16, int N, int D,
                              int H, int W, int kd, int kh, int kw, int up, int cout, int cop, int relu, void* y, int ys, int yc0, int ylo, int out_f32,
                              int split, r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && wp_f16 && bias && y, "mf_conv3d: null pointer");
    R3DP_REQUIRE(N > 0 && D > 0 && H > 0 && W > 0 && cin > 0 && cin % kBK == 0 && cout > 0 && cop >= cout, "mf_conv3d: bad shape");
    R3DP_REQUIRE(kd >= 1 && kh >= 1 && kw >= 1 && (kd & 1) && (up ? (kh == 2 && kw == 2) : ((kh & 1) && (kw & 1))) && kd * kh * kw <= 343,
                 "mf_conv3d: taps are an odd box, or (odd, 2, 2) parity phases with up");
    R3DP_REQUIRE(xs % 8 == 0 && xlo % 8 == 0 && xs >= (split ? xlo : 0) + cin, "mf_conv3d: input voxel stride / lo offset");
    R3DP_REQUIRE(ys % 2 == 0 && yc0 % 2 == 0 && ylo % 2 == 0 && ys >= (split ? ylo : 0) + yc0 + cout, "mf_conv3d: output voxel stride / slice");
    R3DP_REQUIRE(!(out_f32 && res_f16), "mf_conv3d: fp32 output takes no residual");
    R3DP_REQUIRE(!split || xlo >= cin, "mf_conv3d: split input needs its lo half past the channels read");
    Conv3dArgs a = {};
    a.x = reinterpret_cast<const __half*>(x_f16); a.w = reinterpret_cast<const __half*>(wp_f16); a.bias = bias;
    a.res = reinterpret_cast<const __half*>(res_f16); a.y = y;
    a.N = N; a.D = D; a.H = H; a.W = W; a.xs = xs; a.xlo = xlo; a.cin = cin;
    a.kd = kd; a.kh = kh; a.kw = kw; a.oz = kd / 2;
    a.oy = up ? 1 : kh / 2; a.ox = up ? 1 : kw / 2;
    a.sy = a.sx = up ? 2 : 1;
    a.ys = ys; a.yc0 = yc0; a.ylo = ylo; a.cout = cout; a.cop = cop; a.relu = relu; a.out_f32 = out_f32;
    a.acc_scale = split ? 1.0f / kSplitScale3 : 1.0f;
    const int nph = up ? 4 : 1;
    cudaStream_t st = as_stream(stream);
    const int bn = cout <= 16 ? 16 : cout <= 32 ? 32 : cout <= 64 ? 64 : 128;
    R3DP_REQUIRE(cop % bn == 0, "mf_conv3d: packed couts must be a multiple of the cout tile (16 | 32 | 64 | 128)");
#define R3DP_MF_CONV(BN_)                                        \
    if ((split ? launch_conv<BN_, true>(a, nph, st) : launch_conv<BN_, false>(a, nph, st)) != 0) return 1
    switch (bn) {
        case 16: R3DP_MF_CONV(16); break;
        case 32: R3DP_MF_CONV(32); break;
        case 64: R3DP_MF_CONV(64); break;
        default: R3DP_MF_CONV(128); break;
    }
#undef R3DP_MF_CONV
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_mf_input(const float* fc, int fc_shared, const float* kp_s, const float* kp_d, int N, int K, int D, int H, int W, int cpad, void* y_f16,
                             int ys, int ylo, int split, r3dp_stream_t stream) {
    R3DP_REQUIRE(fc && kp_s && kp_d && y_f16, "mf_input: null pointer");
    R3DP_REQUIRE(N > 0 && K > 0 && D > 1 && H > 1 && W > 1 && cpad >= (K + 1) * 5 && ys >= (split ? ylo : 0) + cpad && (!split || ylo >= cpad),
                 "mf_input: bad shape");
    const long long total = (long long)N * D * H * W;
    mf_input_kernel<<<(unsigned)((total + 127) / 128), 128, 0, as_stream(stream)>>>(fc, fc_shared, kp_s, kp_d, N, K, D, H, W, cpad, ys, ylo, split,
                                                                                   reinterpret_cast<__half*>(y_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_mf_pool(const void* x_f16, int N, int D, int H, int W, int C, int xs, int xlo, void* y_f16, int ys, int ylo, int split,
                            r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && y_f16, "mf_pool: null pointer");
    R3DP_REQUIRE(N > 0 && D > 0 && H > 0 && W > 0 && C > 0, "mf_pool: bad shape (H, W: the pooled size)");
    R3DP_REQUIRE(split ? (xlo >= C && ylo >= C && xs >= xlo + C && ys >= ylo + C) : (xs >= C && ys >= C), "mf_pool: voxel stride / lo offset");
    const long long total = (long long)N * D * H * W * C;
    mf_pool_kernel<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<const __half*>(x_f16), (long long)N * D, H, W, C, xs,
                                                                                  xlo, ys, ylo, split, reinterpret_cast<__half*>(y_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_mf_head_input(const float* rgb, const float* wts, int N, int H, int W, int cpad, void* y_f16, int ys, int ylo, int split,
                                  r3dp_stream_t stream) {
    R3DP_REQUIRE(rgb && wts && y_f16, "mf_head_input: null pointer");
    R3DP_REQUIRE(N > 0 && H > 0 && W > 0 && cpad >= 4 && ys >= (split ? ylo : 0) + cpad, "mf_head_input: bad shape (H, W: the output size)");
    const long long total = (long long)N * H * W;
    mf_head_input_kernel<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(rgb, wts, N, H, W, cpad, ys, ylo, split,
                                                                                        reinterpret_cast<__half*>(y_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_mf_head_bcast(const void* x_f16, int N, int D, int H, int W, int C, int xs, int xlo, void* y_f16, int ys, int yc0, int ylo, int split,
                                  r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && y_f16, "mf_head_bcast: null pointer");
    R3DP_REQUIRE(N > 0 && D > 0 && H > 0 && W > 0 && C > 0 && yc0 >= 0, "mf_head_bcast: bad shape (H, W: the output size)");
    R3DP_REQUIRE(split ? (xlo >= C && xs >= xlo + C && ylo >= yc0 + C && ys >= ylo + yc0 + C) : (xs >= C && ys >= yc0 + C),
                 "mf_head_bcast: voxel stride / lo offset / channel slice");
    const long long total = (long long)N * H * W * C;
    mf_head_bcast_kernel<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<const __half*>(x_f16), N, D, H, W, C, xs, xlo, ys,
                                                                                        yc0, ylo, split, reinterpret_cast<__half*>(y_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_mf_deform(const float* logits, int ls, const float* kp_s, const float* kp_d, int N, int K, int D, int H, int W, float* deformation,
                              r3dp_stream_t stream) {
    R3DP_REQUIRE(logits && kp_s && kp_d && deformation, "mf_deform: null pointer");
    R3DP_REQUIRE(N > 0 && K > 0 && D > 1 && H > 1 && W > 1 && ls > K, "mf_deform: bad shape");
    const long long total = (long long)N * D * H * W;
    mf_deform_kernel<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(logits, ls, kp_s, kp_d, N, K, D, H, W, deformation);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_mf_occlusion(const void* x_f16, int N, int D, int H, int W, int C, int xs, int xlo, int split, const float* wk, const float* bias,
                                 float* occ, float* occ2, r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && wk && bias && occ && occ2, "mf_occlusion: null pointer");
    R3DP_REQUIRE(N > 0 && D > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && xs % 8 == 0 && xlo % 8 == 0, "mf_occlusion: bad shape / alignment");
    R3DP_REQUIRE(split ? (xlo >= C && xs >= xlo + C) : xs >= C, "mf_occlusion: voxel stride / lo offset");
    const size_t smem = (size_t)49 * C * 2 * sizeof(float);
    R3DP_REQUIRE(smem <= 200 * 1024, "mf_occlusion: weights over the shared-memory budget");
    R3DP_CUDA(cudaFuncSetAttribute(mf_occlusion_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const long long P = (long long)N * H * W;
    mf_occlusion_kernel<<<(unsigned)((P + kOccThreads - 1) / kOccThreads), kOccThreads, smem, as_stream(stream)>>>(
        reinterpret_cast<const __half*>(x_f16), N, D, H, W, C, xs, xlo, split, wk, bias, occ, occ2);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}
