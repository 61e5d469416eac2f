// Img2PlaneModel (modules/img2plane/img2plane_model.py:12-81) on sm_90a: the canonical plane backbone that builds a clip's tri-planes from
// its source image.  The kernels around the GEMMs:
//   ip_flash_attention_kernel  softmax(q k^T / 16) v for head_dim 256 (segformer/base.py:101-122) on wgmma: one TMA producer warp streams
//                              64-key K/V tiles through a two-slot ring, two consumer warpgroups (setmaxnreg) hold 64 queries each, the
//                              online softmax runs in fp32 on the S fragments and P goes to P.V as the register A operand.  No Tq x Tk buffer.
//   ip_input_kernel            rgb + the two coordinate channels (i / H, j / H, meshgrid 'ij') as NHWC fp16, padded to 8 channels
//   ip_maxpool_kernel          nn.MaxPool2d(3, 2, 1) of the ResNet stem (padding is -inf)
//   ip_channel_mean_kernel     AdaptiveAvgPool2d(1) of ASPP's pooling branch (deeplabv3/decoders/my_decoder.py:139-152)
//   ip_broadcast_kernel        the pooling branch's bilinear upsampling of a 1x1 map: one vector per image into a channel slice
//   ip_pixel_shuffle_kernel    nn.PixelShuffle(2) of the ViTs' token map (after the last residual add), into a channel slice
//   ip_upsample2_kernel        nn.UpsamplingBilinear2d(x2), align_corners=True
//   ip_flip_hwpc_kernel        Img2PlaneModel.forward's view + flips (img2plane_model.py:72-81) into the render's hwpc layout
// Convolutions and token GEMMs run on r3dp_mf_conv3d (strided / dilated ones on r3dp_sp_patches rows), LayerNorm on r3dp_sp_layernorm,
// the Mlp's DWConv + GELU on r3dp_sp_dwconv_gelu.
#include "common.cuh"
#include "tc_prims.cuh"
#include <cuda_fp16.h>
#include <math.h>

namespace r3dp {
namespace ip {
using namespace r3dp::tc;

// ---- flash attention, head_dim 256 ---------------------------------------------------------------------------------------------------
constexpr int kHd = 256;
constexpr int kBQ = 64;                    // queries per consumer warpgroup
constexpr int kBKV = 64;                   // keys per ring slot
constexpr int kSlots = 2;
constexpr int kFaThreads = 384;            // producer warpgroup + 2 consumer warpgroups
constexpr int kProducerRegs = 40, kConsumerRegs = 232;
constexpr int kTile = kBKV * kHd * 2;      // one 64 x 256 fp16 tile: 4 column blocks of 64 rows x 128 B (SWIZZLE_128B atoms)
constexpr int kBlk = 64 * 128;             // one column block
constexpr int kFaSmem = 2 * kTile + 2 * kSlots * kTile + 1024 + 64;

// grid (ceil(Tq / 128), heads, N).  Tensor maps: q [N][Tq][qs] and kv [N][Tk][kvs] fp16, boxes of 64 channels x 64 rows, zero fill past Tq / Tk.
__global__ void __launch_bounds__(kFaThreads, 1) ip_flash_attention_kernel(const __grid_constant__ CUtensorMap tmQ,
                                                                          const __grid_constant__ CUtensorMap tmKV, int Tq, int Tk, int C,
                                                                          float scale_log2, __half* __restrict__ o, int os) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = align_smem_1024(smem_raw);
    uint8_t* sQ = smem;                                 // [2 warpgroups][4 column blocks][64 rows][128 B]
    uint8_t* sK = smem + 2 * kTile;                     // [slot][4][64 keys][128 B]
    uint8_t* sV = sK + kSlots * kTile;
    uint64_t* bars = reinterpret_cast<uint64_t*>(sV + kSlots * kTile);
    uint64_t* q_full = bars;
    uint64_t* kv_full = bars + 1;
    uint64_t* kv_empty = bars + 1 + kSlots;
    const int h = blockIdx.y, n = blockIdx.z, q0 = blockIdx.x * 2 * kBQ;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nkv = (Tk + kBKV - 1) / kBKV;
    if (threadIdx.x == 0) {
        mbar_init(q_full, 1);
        for (int i = 0; i < kSlots; ++i) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], 256); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmQ) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmKV) : "memory");
    }
    __syncthreads();

    if (warp < 4) {
        setmaxnreg_dec<kProducerRegs>();
        if (warp == 0 && lane == 0) {
            mbar_expect_tx(q_full, 2 * kTile);
            for (int g = 0; g < 2; ++g)
                for (int b = 0; b < 4; ++b) tma_load_4d(sQ + g * kTile + b * kBlk, &tmQ, q_full, h * kHd + 64 * b, q0 + g * kBQ, n, 0);
            for (int it = 0; it < nkv; ++it) {
                const int s = it % kSlots;
                mbar_wait(&kv_empty[s], ((it / kSlots) & 1) ^ 1);
                mbar_expect_tx(&kv_full[s], 2 * kTile);
                for (int b = 0; b < 4; ++b) {
                    tma_load_4d(sK + s * kTile + b * kBlk, &tmKV, &kv_full[s], h * kHd + 64 * b, it * kBKV, n, 0);
                    tma_load_4d(sV + s * kTile + b * kBlk, &tmKV, &kv_full[s], C + h * kHd + 64 * b, it * kBKV, n, 0);
                }
            }
        }
        return;
    }
    setmaxnreg_inc<kConsumerRegs>();
    const int g = (warp >> 2) - 1;
    // fragment rows acc_row(i) = r0 (+ 8), columns acc_col(i); rmax/rsum over a row: the 4 lanes of a quad
    float oacc[4][32];
#pragma unroll
    for (int b = 0; b < 4; ++b)
#pragma unroll
        for (int i = 0; i < 32; ++i) oacc[b][i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    const uint32_t qb = smem_u32(sQ + g * kTile);
    mbar_wait(q_full, 0);
    for (int it = 0; it < nkv; ++it) {
        const int s = it % kSlots;
        mbar_wait(&kv_full[s], (it / kSlots) & 1);
        const uint32_t kb = smem_u32(sK + s * kTile), vb = smem_u32(sV + s * kTile);
        float sc[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) sc[i] = 0.f;
        wg_fence_acc<32>(sc);
        wg_fence();
#pragma unroll
        for (int j = 0; j < kHd / 16; ++j) {
            const uint32_t off = (j >> 2) * kBlk + (j & 3) * 32;
            wgmma_m64n64k16(sc, desc_sw128(qb + off), desc_sw128(kb + off), j ? 1u : 0u);
        }
        wg_commit();
        wg_wait<0>();
        wg_fence_acc<32>(sc);
        // mask keys past Tk, then the online softmax in the log2 domain
        const int kbase = it * kBKV;
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            const float v = kbase + acc_col(i) < Tk ? sc[i] * scale_log2 : -INFINITY;
            sc[i] = v;
            mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], v);
        }
        float corr[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            const float mn = fmaxf(m[r], mx[r]);            // finite: every tile holds at least one key < Tk
            corr[r] = exp2f(m[r] - mn);
            m[r] = mn;
            l[r] *= corr[r];
        }
        uint32_t pa[4][4];
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
            const int r = (i >> 1) & 1;
            const float p0 = exp2f(sc[i] - m[r]), p1 = exp2f(sc[i + 1] - m[r]);
            l[r] += p0 + p1;
            pa[i >> 3][(i >> 1) & 3] = pack_h2(p0, p1);
        }
#pragma unroll
        for (int b = 0; b < 4; ++b)
#pragma unroll
            for (int i = 0; i < 32; ++i) oacc[b][i] *= corr[(i >> 1) & 1];
#pragma unroll
        for (int b = 0; b < 4; ++b) wg_fence_acc<32>(oacc[b]);
        wg_fence();
#pragma unroll
        for (int t = 0; t < kBKV / 16; ++t)
#pragma unroll
            for (int b = 0; b < 4; ++b) wgmma_rs_m64n64k16_tb(oacc[b], pa[t], desc_sw128(vb + b * kBlk + t * 2048));
        wg_commit();
        wg_wait<0>();
#pragma unroll
        for (int b = 0; b < 4; ++b) wg_fence_acc<32>(oacc[b]);
        mbar_arrive(&kv_empty[s]);
    }
    float inv[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
        l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
        inv[r] = 1.f / l[r];
    }
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
        const int row = q0 + g * kBQ + acc_row(i);
        if (row >= Tq) continue;
        const float iv = inv[(i >> 1) & 1];
        __half* orow = o + ((size_t)n * Tq + row) * os + h * kHd + acc_col(i);
#pragma unroll
        for (int b = 0; b < 4; ++b) *reinterpret_cast<__half2*>(orow + 64 * b) = __floats2half2_rn(oacc[b][i] * iv, oacc[b][i + 1] * iv);
    }
}

// ---- the small kernels ---------------------------------------------------------------------------------------------------------------
// one thread per pixel: x fp32 NCHW [N,3,H,W] -> y fp16 [N,H,W,8] = (r, g, b, i / H, j / H, 0, 0, 0)
__global__ void ip_input_kernel(const float* __restrict__ x, int N, int H, int W, __half* __restrict__ y) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long HW = (long long)H * W;
    if (idx >= N * HW) return;
    const int n = (int)(idx / HW);
    const long long p = idx % HW;
    const int i = (int)(p / W), j = (int)(p % W);
    const float* xn = x + (size_t)n * 3 * HW + p;
    uint4 v;
    __half2* h2 = reinterpret_cast<__half2*>(&v);
    h2[0] = __floats2half2_rn(xn[0], xn[HW]);
    h2[1] = __floats2half2_rn(xn[2 * HW], (float)i / (float)H);
    h2[2] = __floats2half2_rn((float)j / (float)H, 0.f);
    h2[3] = __floats2half2_rn(0.f, 0.f);
    *reinterpret_cast<uint4*>(y + idx * 8) = v;
}

// one thread per (output pixel, 8 channels); window 3x3, stride 2, padding 1 (padding never wins: -inf)
__global__ void ip_maxpool_kernel(const __half* __restrict__ x, int N, int H, int W, int C, int Ho, int Wo, __half* __restrict__ y) {
    const int c8 = C / 8;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * Ho * Wo * c8) return;
    const int cc = (int)(idx % c8);
    long long t = idx / c8;
    const int ox = (int)(t % Wo); t /= Wo;
    const int oy = (int)(t % Ho), n = (int)(t / Ho);
    __half2 mx[4];
    const __half2 ninf = __halves2half2(__ushort_as_half(0xfc00), __ushort_as_half(0xfc00));
#pragma unroll
    for (int k = 0; k < 4; ++k) mx[k] = ninf;
    for (int dy = 0; dy < 3; ++dy) {
        const int iy = 2 * oy - 1 + dy;
        if (iy < 0 || iy >= H) continue;
        for (int dx = 0; dx < 3; ++dx) {
            const int ix = 2 * ox - 1 + dx;
            if (ix < 0 || ix >= W) continue;
            const uint4 v = *reinterpret_cast<const uint4*>(x + (((size_t)n * H + iy) * W + ix) * C + cc * 8);
            const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
            for (int k = 0; k < 4; ++k) mx[k] = __hmax2(mx[k], h[k]);
        }
    }
    *reinterpret_cast<uint4*>(y + idx * 8) = *reinterpret_cast<uint4*>(mx);
}

// grid (N, C / 32), 256 threads: 32 channels x 8 pixel lanes, fp32 sums; y fp16 [N, C] (the pooled rows of a GEMM)
__global__ void __launch_bounds__(256) ip_channel_mean_kernel(const __half* __restrict__ x, int HW, int C, __half* __restrict__ y) {
    __shared__ float part[8][33];
    const int n = blockIdx.x, c = blockIdx.y * 32 + (threadIdx.x & 31), pl = threadIdx.x >> 5;
    float s = 0.f;
    for (int p = pl; p < HW; p += 8) s += __half2float(x[((size_t)n * HW + p) * C + c]);
    part[pl][threadIdx.x & 31] = s;
    __syncthreads();
    if (pl == 0) {
        float t = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) t += part[k][threadIdx.x & 31];
        y[(size_t)n * C + c] = __float2half_rn(t / (float)HW);
    }
}

// y[n, p, yc0 + c] = v[n, c] for every pixel p; one thread per (pixel, 2 channels)
__global__ void ip_broadcast_kernel(const __half* __restrict__ v, int N, int HW, int C, __half* __restrict__ y, int ys, int yc0) {
    const int c2 = C / 2;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * HW * c2) return;
    const int c = (int)(idx % c2) * 2;
    const long long pix = idx / c2;
    const int n = (int)(pix / HW);
    *reinterpret_cast<__half2*>(y + pix * ys + yc0 + c) = *reinterpret_cast<const __half2*>(v + (size_t)n * C + c);
}

// tokens x (+ t) fp32 [N, h*w, 4C] -> y fp16 [N, 2h, 2w] pixels of ys halves at channels [yc0, yc0 + C):
// y[n, 2a + i, 2b + j, c] = x[n, a*w + b, 4c + 2i + j].  One thread per (output pixel, 2 channels).
__global__ void ip_pixel_shuffle_kernel(const float* __restrict__ x, const float* __restrict__ t, int N, int h, int w, int C,
                                        __half* __restrict__ y, int ys, int yc0) {
    const int c2 = C / 2, H = 2 * h, W = 2 * w;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * H * W * c2) return;
    const int c = (int)(idx % c2) * 2;
    const long long pix = idx / c2;
    const int X = (int)(pix % W), Y = (int)((pix / W) % H), n = (int)(pix / ((long long)W * H));
    const size_t src = ((size_t)n * h * w + (Y >> 1) * w + (X >> 1)) * (4 * C) + 2 * (Y & 1) + (X & 1);
    float v0 = x[src + 4 * c], v1 = x[src + 4 * c + 4];
    if (t) { v0 += t[src + 4 * c]; v1 += t[src + 4 * c + 4]; }
    *reinterpret_cast<__half2*>(y + pix * ys + yc0 + c) = __floats2half2_rn(v0, v1);
}

// nn.UpsamplingBilinear2d(x2) (align_corners=True) of x fp16 NHWC [N,h,w,C] -> y [N,2h,2w,C]; one thread per (output pixel, 8 channels)
__global__ void ip_upsample2_kernel(const __half* __restrict__ x, int N, int h, int w, int C, __half* __restrict__ y) {
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
    *reinterpret_cast<uint4*>(y + pix * C + cc * 8) = res;
}

// conv output x fp32 [N,H,W,96] -> out fp32 [N,H,W,3,32] (hwpc): out[n, Y, X, p, c] = x[n, H-1-Y, p < 2 ? X : W-1-X, 32p + c].
// One thread per (output pixel, plane, 4 channels).
__global__ void ip_flip_hwpc_kernel(const float* __restrict__ x, int N, int H, int W, float* __restrict__ out) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * H * W * 24) return;
    const int q = (int)(idx % 24), p = q / 8;
    const long long pix = idx / 24;
    const int X = (int)(pix % W), Y = (int)((pix / W) % H), n = (int)(pix / ((long long)W * H));
    const int sx = p < 2 ? X : W - 1 - X;
    const float4 v = *reinterpret_cast<const float4*>(x + (((size_t)n * H + (H - 1 - Y)) * W + sx) * 96 + 4 * q);
    *reinterpret_cast<float4*>(out + pix * 96 + 4 * q) = v;
}

inline unsigned blocks(long long n, int t) { return (unsigned)((n + t - 1) / t); }

// ---- host side: tensor maps ----------------------------------------------------------------------------------------------------------
// fp16 rows [N][T][stride] read in 64-channel x 64-row boxes (128-byte swizzle), zero fill past T
static int token_map(CUtensorMap* m, const void* ptr, int N, int T, int stride) {
    EncodeTiledFn fn = encode_fn();
    R3DP_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled is not available from the driver");
    const cuuint64_t dims[4] = {(cuuint64_t)stride, (cuuint64_t)T, (cuuint64_t)N, 1};
    const cuuint64_t strides[3] = {(cuuint64_t)stride * 2, (cuuint64_t)T * stride * 2, (cuuint64_t)N * T * stride * 2};
    const cuuint32_t box[4] = {64, 64, 1, 1};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    R3DP_REQUIRE(r == CUDA_SUCCESS, "ip_attention: cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
    return 0;
}

}  // namespace ip
}  // namespace r3dp

using namespace r3dp;
using namespace r3dp::ip;

extern "C" int r3dp_ip_attention(const void* q_f16, int qs, const void* kv_f16, int kvs, int N, int Tq, int Tk, int heads, float scale, void* o_f16,
                                 int os, r3dp_stream_t stream) {
    R3DP_REQUIRE(q_f16 && kv_f16 && o_f16, "ip_attention: null pointer");
    const int C = heads * kHd;
    R3DP_REQUIRE(N > 0 && Tq > 0 && Tk > 0 && heads > 0 && qs >= C && kvs >= 2 * C && os >= C && qs % 8 == 0 && kvs % 8 == 0 && os % 2 == 0,
                 "ip_attention: bad shape (head_dim 256; row strides multiples of 8 halves)");
    R3DP_REQUIRE((reinterpret_cast<uintptr_t>(q_f16) & 15) == 0 && (reinterpret_cast<uintptr_t>(kv_f16) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(o_f16) & 3) == 0, "ip_attention: q / kv must be 16-byte aligned");
    CUtensorMap tq, tkv;
    if (token_map(&tq, q_f16, N, Tq, qs) || token_map(&tkv, kv_f16, N, Tk, kvs)) return 1;
    R3DP_CUDA(cudaFuncSetAttribute(ip_flash_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kFaSmem));
    const dim3 grid(blocks(Tq, 2 * kBQ), heads, N);
    ip_flash_attention_kernel<<<grid, kFaThreads, kFaSmem, as_stream(stream)>>>(tq, tkv, Tq, Tk, C, scale * 1.4426950408889634f,
                                                                               reinterpret_cast<__half*>(o_f16), os);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_ip_input(const float* x, int N, int H, int W, void* y_f16, r3dp_stream_t stream) {
    R3DP_REQUIRE(x && y_f16, "ip_input: null pointer");
    R3DP_REQUIRE(N > 0 && H > 0 && W > 0, "ip_input: bad shape");
    const long long n = (long long)N * H * W;
    ip_input_kernel<<<blocks(n, 256), 256, 0, as_stream(stream)>>>(x, N, H, W, reinterpret_cast<__half*>(y_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_ip_maxpool(const void* x_f16, int N, int H, int W, int C, void* y_f16, r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && y_f16, "ip_maxpool: null pointer");
    R3DP_REQUIRE(N > 0 && H > 0 && W > 0 && C % 8 == 0 && C > 0, "ip_maxpool: bad shape");
    const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
    const long long n = (long long)N * Ho * Wo * (C / 8);
    ip_maxpool_kernel<<<blocks(n, 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<const __half*>(x_f16), N, H, W, C, Ho, Wo,
                                                                     reinterpret_cast<__half*>(y_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_ip_channel_mean(const void* x_f16, int N, int HW, int C, void* y_f16, r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && y_f16, "ip_channel_mean: null pointer");
    R3DP_REQUIRE(N > 0 && HW > 0 && C % 32 == 0 && C > 0, "ip_channel_mean: bad shape");
    ip_channel_mean_kernel<<<dim3(N, C / 32), 256, 0, as_stream(stream)>>>(reinterpret_cast<const __half*>(x_f16), HW, C,
                                                                           reinterpret_cast<__half*>(y_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_ip_broadcast(const void* v_f16, int N, int HW, int C, void* y_f16, int ys, int yc0, r3dp_stream_t stream) {
    R3DP_REQUIRE(v_f16 && y_f16, "ip_broadcast: null pointer");
    R3DP_REQUIRE(N > 0 && HW > 0 && C > 0 && C % 2 == 0 && yc0 % 2 == 0 && ys % 2 == 0 && yc0 >= 0 && ys >= yc0 + C, "ip_broadcast: bad shape");
    const long long n = (long long)N * HW * (C / 2);
    ip_broadcast_kernel<<<blocks(n, 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<const __half*>(v_f16), N, HW, C,
                                                                       reinterpret_cast<__half*>(y_f16), ys, yc0);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_ip_pixel_shuffle(const float* x, const float* t, int N, int h, int w, int C, void* y_f16, int ys, int yc0, r3dp_stream_t stream) {
    R3DP_REQUIRE(x && y_f16, "ip_pixel_shuffle: null pointer");
    R3DP_REQUIRE(N > 0 && h > 0 && w > 0 && C > 0 && C % 2 == 0 && yc0 % 2 == 0 && ys % 2 == 0 && yc0 >= 0 && ys >= yc0 + C,
                 "ip_pixel_shuffle: bad shape");
    const long long n = (long long)N * 4 * h * w * (C / 2);
    ip_pixel_shuffle_kernel<<<blocks(n, 256), 256, 0, as_stream(stream)>>>(x, t, N, h, w, C, reinterpret_cast<__half*>(y_f16), ys, yc0);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_ip_upsample2(const void* x_f16, int N, int h, int w, int C, void* y_f16, r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && y_f16, "ip_upsample2: null pointer");
    R3DP_REQUIRE(N > 0 && h > 0 && w > 0 && C % 8 == 0 && C > 0, "ip_upsample2: bad shape");
    const long long n = (long long)N * 4 * h * w * (C / 8);
    ip_upsample2_kernel<<<blocks(n, 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<const __half*>(x_f16), N, h, w, C,
                                                                       reinterpret_cast<__half*>(y_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_ip_flip_hwpc(const float* x, int N, int H, int W, float* out, r3dp_stream_t stream) {
    R3DP_REQUIRE(x && out, "ip_flip_hwpc: null pointer");
    R3DP_REQUIRE(N > 0 && H > 0 && W > 0, "ip_flip_hwpc: bad shape");
    const long long n = (long long)N * H * W * 24;
    ip_flip_hwpc_kernel<<<blocks(n, 256), 256, 0, as_stream(stream)>>>(x, N, H, W, out);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}
