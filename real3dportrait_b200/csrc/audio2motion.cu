// The audio2secc VAE (modules/audio2motion/vae.py, PitchContourVAEModel / VAEModel at inference) on sm_90a.
//   a2m_wn_kernel      one WaveNet layer (flow_base.py:70-96) fused: the k-tap in_layer conv over a 64-frame tile plus halo, the layer's
//                      slice of the precomputed cond_layer output, tanh(a) * sigmoid(b), the 1x1 res_skip GEMM on the gated tile in shared
//                      memory, and the residual / skip updates in the epilogue.  wgmma, split-fp16 operands ([hi | lo], weights of w * 2^10).
//   a2m_input_kernel   the x0.5 downsample of the audio features, f0 -> coarse bin -> pitch_embed row, and the one-hot blink / amplitude block
//   a2m_split_kernel   fp32 rows -> split fp16 per frame and / or per group of four frames (g_pre_net's input view)
//   a2m_latent_kernel  the prior draw [B,16,T/4] x temperature -> the flow's channels-last split state
//   a2m_store_kernel   the expression rows x y_mask -> the caller's (row-strided) destination
// The convolutions and GEMMs around the WaveNets run on r3dp_mf_conv3d (1-D as D = H = 1, W = T).
#include "common.cuh"
#include "tc_prims.cuh"
#include <cuda_fp16.h>

namespace r3dp {
namespace a2m {
using namespace r3dp::tc;

constexpr int kBM = 64;                  // frames per CTA (one consumer warpgroup)
constexpr int kThreads = 128;
constexpr int kStages = 4;               // weight ring; loads run 2 steps ahead, one MMA group stays in flight
constexpr int kStepHalves = 2 * 64 * 32; // one streamed weight step: [hi | lo] x 64 rows x 32 channels
constexpr int kStepBytes = 2 * kStepHalves;
constexpr float kInvScale = 1.0f / 1024.0f;

__device__ __forceinline__ uint32_t sw64(int r, int j) { return (uint32_t)(r * 64 + ((j ^ ((r >> 1) & 3)) << 4)); }
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// shared-memory plan of one WN layer shape
template <int H, int K>
struct WnCfg {
    static constexpr int NC = H / 32;                       // 32-channel chunks of the hidden state
    static constexpr int HALO = K / 2;
    static constexpr int XR = (kBM + K - 1 + 7) / 8 * 8;   // rows of the input tile (frames t0 - HALO ...), whole 8-row atoms
    static constexpr int XBLK = XR * 64;                    // one (chunk, half) block of the input tile, a multiple of 512
    static constexpr int GBLK = kBM * 64;                   // one (chunk, half) block of the gated tile
    static constexpr int X_OFF = 0, G_OFF = 2 * NC * XBLK, R_OFF = G_OFF + 2 * NC * GBLK;
    static constexpr int SMEM = R_OFF + kStages * kStepBytes + 1024;
    static constexpr int S1 = NC * K * NC;                  // in_layer steps: (gate chunk, tap, input chunk)
};

struct WnArgs {
    const float* x;          // residual stream in [B][T][H] fp32
    float* x_out;            // residual stream out (not written by the last layer); never aliases x (neighbours read x through the halo)
    const float* cond;       // [B][T] rows of cs floats: this layer's 2H cond_layer outputs, (tanh, sigmoid) interleaved, in_layer bias added
    int cs;
    const __half* w;         // packed steps: S1 in_layer steps, then (NO / 64) * NC res_skip steps, each [hi | lo][64][32]
    const float* bias;       // res_skip bias [NO]
    float* skip;             // skip sum [B][T][H] fp32, updated in place (not read when first)
    __half* out;             // last layer: the WaveNet output (skip sum) as split fp16 [B][T][hi H | lo H]
    int T, first, last;
};

// CTA = 64 consecutive frames of one batch item.  The input tile (frames t0 - K/2 .. t0 + 64 + K/2, zero outside [0, T)) is split to
// [hi | lo] fp16 in shared memory once; every in_layer tap is the same tile read from a row-shifted descriptor.  The in_layer runs as
// H/32 gate chunks of 64 packed rows (row 2m = tanh row of channel m, 2m + 1 its sigmoid row, so each thread's accumulator column pair
// is one channel's (a, b)); each chunk's gated values go to the gated tile in shared memory, which is the A operand of the res_skip GEMM.
template <int H, int K>
__global__ void __launch_bounds__(kThreads) a2m_wn_kernel(const WnArgs a) {
    using C = WnCfg<H, K>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = align_smem_1024(smem_raw);
    const int tid = threadIdx.x;
    const int b = blockIdx.y, t0 = blockIdx.x * kBM, T = a.T;
    const int NO = a.last ? H : 2 * H;
    const int S = C::S1 + (NO / 64) * C::NC;
    const size_t row0 = (size_t)b * T;

    auto load_step = [&](int s, int slot) {
        const __half* src = a.w + (size_t)s * kStepHalves;
        const uint32_t base = smem_u32(smem + C::R_OFF + slot * kStepBytes);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int e = tid + q * kThreads;                 // 512 16-byte pieces
            const int hh = e >> 8, r = (e >> 2) & 63, j = e & 3;
            cp_async16(base + hh * (64 * 64) + sw64(r, j), src + hh * 2048 + r * 32 + j * 8);
        }
    };
#pragma unroll
    for (int s = 0; s < kStages - 2; ++s) {
        if (s < S) load_step(s, s);
        cp_async_commit();
    }

    // the input tile, split to [hi | lo] (zero outside the sequence: the conv's per-item zero padding)
    for (int e = tid; e < C::XR * (H / 4); e += kThreads) {
        const int r = e / (H / 4), ch = (e - r * (H / 4)) * 4;
        const int t = t0 - C::HALO + r;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (t >= 0 && t < T && r < kBM + K - 1) v = *reinterpret_cast<const float4*>(a.x + (row0 + t) * H + ch);
        const __half h0 = __float2half_rn(v.x), h1 = __float2half_rn(v.y), h2 = __float2half_rn(v.z), h3 = __float2half_rn(v.w);
        const __half l0 = __float2half_rn(v.x - __half2float(h0)), l1 = __float2half_rn(v.y - __half2float(h1));
        const __half l2 = __float2half_rn(v.z - __half2float(h2)), l3 = __float2half_rn(v.w - __half2float(h3));
        const int c = ch >> 5, k = ch & 31;
        const uint32_t off = sw64(r, k >> 3) + (k & 7) * 2;
        uint8_t* hi = smem + C::X_OFF + (2 * c) * C::XBLK + off;
        uint8_t* lo = hi + C::XBLK;
        *reinterpret_cast<__half2*>(hi) = __halves2half2(h0, h1);
        *reinterpret_cast<__half2*>(hi + 4) = __halves2half2(h2, h3);
        *reinterpret_cast<__half2*>(lo) = __halves2half2(l0, l1);
        *reinterpret_cast<__half2*>(lo + 4) = __halves2half2(l2, l3);
    }

    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    const uint32_t xs_base = smem_u32(smem + C::X_OFF), gs_base = smem_u32(smem + C::G_OFF);
    for (int s = 0; s < S; ++s) {
        cp_async_wait<kStages - 3>();
        fence_proxy_async();                                  // this thread's cp.async and generic smem writes -> the async proxy
        __syncthreads();
        if (s + kStages - 2 < S) load_step(s + kStages - 2, (s + kStages - 2) % kStages);
        cp_async_commit();
        const uint32_t sb = smem_u32(smem + C::R_OFF + (s % kStages) * kStepBytes);
        uint32_t sa;
        bool first_k;
        if (s < C::S1) {
            const int c = s % C::NC, tap = (s / C::NC) % K;
            sa = xs_base + (2 * c) * C::XBLK + tap * 64;       // row shift = tap
            first_k = (s % (K * C::NC)) == 0;
        } else {
            const int c = (s - C::S1) % C::NC;
            sa = gs_base + (2 * c) * C::GBLK;
            first_k = c == 0;
        }
        const uint32_t sa_lo = sa + (s < C::S1 ? C::XBLK : C::GBLK);
        wg_fence_acc<32>(acc);
        wg_fence();
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const uint64_t dah = gmma_desc_sw64(sa + 32 * k), dbh = gmma_desc_sw64(sb + 32 * k);
            wgmma_m64n64k16(acc, dah, dbh, (first_k && k == 0) ? 0u : 1u);
            wgmma_m64n64k16(acc, gmma_desc_sw64(sa_lo + 32 * k), dbh, 1u);
            wgmma_m64n64k16(acc, dah, gmma_desc_sw64(sb + 64 * 64 + 32 * k), 1u);
        }
        wg_commit();
        wg_wait<1>();
        wg_fence_acc<32>(acc);

        const bool group_end = s < C::S1 ? ((s + 1) % (K * C::NC)) == 0 : ((s - C::S1 + 1) % C::NC) == 0;
        if (!group_end) continue;
        wg_wait<0>();
        wg_fence_acc<32>(acc);
        if (s < C::S1) {
            // gate epilogue: channel 32 j + m of every frame -> the gated tile (chunk j)
            const int j = s / (K * C::NC);
            uint8_t* g_hi = smem + C::G_OFF + (2 * j) * C::GBLK;
#pragma unroll
            for (int i = 0; i < 32; i += 2) {
                const int row = acc_row(i), m = acc_col(i) >> 1;
                const int t = t0 + row;
                float2 cv = make_float2(0.f, 0.f);
                if (t < T) cv = *reinterpret_cast<const float2*>(a.cond + (row0 + t) * a.cs + 2 * (32 * j + m));
                const float za = __fmaf_rn(acc[i], kInvScale, cv.x), zb = __fmaf_rn(acc[i + 1], kInvScale, cv.y);
                const float gv = tanhf(za) * (1.f / (1.f + expf(-zb)));
                const __half gh = __float2half_rn(gv), gl = __float2half_rn(gv - __half2float(gh));
                const uint32_t off = sw64(row, m >> 3) + (m & 7) * 2;
                *reinterpret_cast<__half*>(g_hi + off) = gh;
                *reinterpret_cast<__half*>(g_hi + C::GBLK + off) = gl;
            }
        } else {
            // res_skip epilogue: output columns [64 n, 64 n + 64)
            const int n = (s - C::S1) / C::NC;
#pragma unroll
            for (int i = 0; i < 32; i += 2) {
                const int row = acc_row(i), col = 64 * n + acc_col(i);
                const int t = t0 + row;
                if (t >= T) continue;
                const size_t r = row0 + t;
                const float v0 = __fmaf_rn(acc[i], kInvScale, a.bias[col]), v1 = __fmaf_rn(acc[i + 1], kInvScale, a.bias[col + 1]);
                if (!a.last && col < H) {
                    const float2 xv = *reinterpret_cast<const float2*>(a.x + r * H + col);
                    *reinterpret_cast<float2*>(a.x_out + r * H + col) = make_float2(xv.x + v0, xv.y + v1);
                } else {
                    const int c = a.last ? col : col - H;
                    float2 sv = make_float2(v0, v1);
                    if (!a.first) {
                        const float2 p = *reinterpret_cast<const float2*>(a.skip + r * H + c);
                        sv = make_float2(p.x + v0, p.y + v1);
                    }
                    if (a.last) {
                        const __half h0 = __float2half_rn(sv.x), h1 = __float2half_rn(sv.y);
                        __half* o = a.out + r * (2 * H) + c;
                        *reinterpret_cast<__half2*>(o) = __halves2half2(h0, h1);
                        *reinterpret_cast<__half2*>(o + H) =
                            __halves2half2(__float2half_rn(sv.x - __half2float(h0)), __float2half_rn(sv.y - __half2float(h1)));
                    } else {
                        *reinterpret_cast<float2*>(a.skip + r * H + c) = sv;
                    }
                }
            }
        }
    }
    cp_async_wait<0>();
}

template <int H, int K>
static int launch_wn(const WnArgs& a, int B, cudaStream_t st) {
    using C = WnCfg<H, K>;
    R3DP_CUDA(cudaFuncSetAttribute(a2m_wn_kernel<H, K>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM));
    const dim3 grid((unsigned)((a.T + kBM - 1) / kBM), (unsigned)B);
    a2m_wn_kernel<H, K><<<grid, kThreads, C::SMEM, st>>>(a);
    return 0;
}

// ---- the small kernels around the WaveNets --------------------------------------------------------------------------------------
__device__ __forceinline__ void put_split(__half* y, int lo, float v) {
    const __half h = __float2half_rn(v);
    y[0] = h;
    y[lo] = __float2half_rn(v - __half2float(h));
}

// f0_to_coarse (utils/commons/pitch_utils.py:17-26) in the reference's fp32 order: mel = 1127 log(1 + f0 / 700); mel > 0 -> (mel - mel_min)
// * 254 / (mel_max - mel_min) + 1; clamp to [1, 255]; bin = (long)(mel + 0.5).  Every step is rounded on its own (no contraction).
__device__ __forceinline__ int coarse_bin(float f0, float mel_min, float mel_span) {
    float mel = __fmul_rn(1127.f, logf(__fadd_rn(1.f, __fdiv_rn(f0, 700.f))));
    if (mel > 0.f) mel = __fadd_rn(__fdiv_rn(__fmul_rn(__fsub_rn(mel, mel_min), 254.f), mel_span), 1.f);
    if (mel <= 1.f) mel = 1.f;
    if (mel > 255.f) mel = 255.f;
    return (int)__fadd_rn(mel, 0.5f);
}

// one thread per (output frame, 4-channel group).  Output frame i of item b reads input frame 2i (nearest) or the mean of 2i, 2i + 1.
// Channels of y (split, lo at ylo): [0, A) the audio features, [A, Ap) zero; with `table`: [Ap, Ap + 128) pitch_embed[coarse(f0[2i])],
// and the 32 channels of yb (frame stride ybs, lo at yblo): blink == 0, blink == 1, mouth_amp[b], eye_amp[b], zeros.
__global__ void a2m_input_kernel(const float* __restrict__ audio, int B, int Tx, int A, int Ap, int mean, const float* __restrict__ f0,
                                 const long long* __restrict__ blink, const float* __restrict__ mouth, const float* __restrict__ eye,
                                 const float* __restrict__ table, float mel_min, float mel_span, __half* __restrict__ y, int ys, int ylo,
                                 __half* __restrict__ yb, int ybs, int yblo) {
    const int T = Tx / 2;
    const int G = (Ap + (table ? 160 : 0)) / 4;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)B * T * G) return;
    const int g = (int)(idx % G);
    const long long fr = idx / G;
    const int i = (int)(fr % T), b = (int)(fr / T);
    __half* out = y + (size_t)fr * ys;
    const size_t src = (size_t)b * Tx + 2 * i;
    for (int e = 0; e < 4; ++e) {
        const int c = 4 * g + e;
        float v = 0.f;
        if (c < A) {
            const float x0 = audio[src * A + c];
            v = mean ? 0.5f * (x0 + audio[(src + 1) * A + c]) : x0;
        } else if (c >= Ap && c < Ap + 128) {
            v = table[coarse_bin(f0[src], mel_min, mel_span) * 128 + (c - Ap)];
        } else if (c >= Ap + 128) {
            const int k = c - Ap - 128;
            const long long bl = blink ? blink[src] : 0;
            v = k == 0 ? (float)(bl == 0) : k == 1 ? (float)(bl == 1) : k == 2 ? (mouth ? mouth[b] : 0.f) : k == 3 ? (eye ? eye[b] : 0.f) : 0.f;
            put_split(yb + (size_t)fr * ybs + k, yblo, v);
            continue;
        }
        put_split(out + c, ylo, v);
    }
}

// x fp32 [R][C] -> y1: split per frame [R][hi C | lo C]; y4: split per group of four frames [R/4][hi 4C | lo 4C] (frame 4u + r, channel
// r C + c).  Either may be null.
__global__ void a2m_split_kernel(const float* __restrict__ x, long long R, int C, __half* __restrict__ y1, __half* __restrict__ y4) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= R * C) return;
    const int c = (int)(idx % C);
    const long long r = idx / C;
    const float v = x[idx];
    if (y1) put_split(y1 + r * 2 * C + c, C, v);
    if (y4) put_split(y4 + (r >> 2) * 8 * C + (r & 3) * C + c, 4 * C, v);
}

// z [B][16][T4] fp32 (the prior draw) x temperature -> y [B*T4][hi 32 | lo 32], channels 16..31 zero
__global__ void a2m_latent_kernel(const float* __restrict__ z, int B, int T4, float temperature, __half* __restrict__ y) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)B * T4 * 32) return;
    const int c = (int)(idx & 31);
    const long long fr = idx >> 5;
    const int t = (int)(fr % T4), b = (int)(fr / T4);
    const float v = c < 16 ? z[((size_t)b * 16 + c) * T4 + t] * temperature : 0.f;
    put_split(y + fr * 64 + c, 32, v);
}

// x [N][C] fp32 -> out[n * ld + c] = x * mask[n] (mask may be null: ones)
__global__ void a2m_store_kernel(const float* __restrict__ x, const float* __restrict__ mask, long long N, int C, float* __restrict__ out, long long ld) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= N * C) return;
    const long long n = idx / C;
    const int c = (int)(idx % C);
    out[n * ld + c] = mask ? x[idx] * mask[n] : x[idx];
}

inline unsigned blocks(long long n, int t) { return (unsigned)((n + t - 1) / t); }

}  // namespace a2m
}  // namespace r3dp

using namespace r3dp;
using namespace r3dp::a2m;

extern "C" int r3dp_a2m_wn_layer(const float* x, float* x_out, const float* cond, int cs, const void* w_f16, const float* bias, float* skip, void* out_f16,
                                 int B, int T, int hidden, int k, int first, int last, r3dp_stream_t stream) {
    R3DP_REQUIRE(x && cond && w_f16 && bias && skip, "a2m_wn_layer: null pointer");
    R3DP_REQUIRE(B > 0 && T > 0 && ((hidden == 64 && k == 3) || (hidden == 256 && k == 5)), "a2m_wn_layer: shapes (hidden, k) = (64, 3) | (256, 5)");
    R3DP_REQUIRE(last ? (out_f16 != nullptr && !first) : (x_out != nullptr && x_out != x), "a2m_wn_layer: x_out (a separate buffer) / out");
    R3DP_REQUIRE(cs >= 2 * hidden && cs % 2 == 0 && (reinterpret_cast<uintptr_t>(cond) & 7) == 0, "a2m_wn_layer: cond row stride / alignment");
    R3DP_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(x_out) & 7) == 0 && (reinterpret_cast<uintptr_t>(skip) & 7) == 0 &&
                 (reinterpret_cast<uintptr_t>(out_f16) & 3) == 0, "a2m_wn_layer: buffer alignment");
    WnArgs a;
    a.x = x; a.x_out = x_out; a.cond = cond; a.cs = cs; a.w = reinterpret_cast<const __half*>(w_f16); a.bias = bias; a.skip = skip;
    a.out = reinterpret_cast<__half*>(out_f16); a.T = T; a.first = first; a.last = last;
    cudaStream_t st = as_stream(stream);
    if ((hidden == 64 ? launch_wn<64, 3>(a, B, st) : launch_wn<256, 5>(a, B, st)) != 0) return 1;
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_a2m_input(const float* audio, int B, int Tx, int A, int Ap, int mean, const float* f0, const long long* blink, const float* mouth_amp,
                              const float* eye_amp, const float* pitch_table, float mel_min, float mel_span, void* y_f16, int ys, int ylo,
                              void* yb_f16, int ybs, int yblo, r3dp_stream_t stream) {
    R3DP_REQUIRE(audio && y_f16, "a2m_input: null pointer");
    R3DP_REQUIRE(B > 0 && Tx > 0 && Tx % 2 == 0 && A > 0 && Ap >= A && Ap % 32 == 0, "a2m_input: bad shape");
    R3DP_REQUIRE(!pitch_table || (f0 && yb_f16 && yblo >= 32 && ybs >= yblo + 32), "a2m_input: the pitch blocks need f0 and yb");
    const int C = Ap + (pitch_table ? 128 : 0);
    R3DP_REQUIRE(ylo >= C && ys >= ylo + C, "a2m_input: frame stride / lo offset");
    const long long total = (long long)B * (Tx / 2) * ((C + (pitch_table ? 32 : 0)) / 4);
    a2m_input_kernel<<<blocks(total, 256), 256, 0, as_stream(stream)>>>(audio, B, Tx, A, Ap, mean, f0, blink, mouth_amp, eye_amp, pitch_table, mel_min,
                                                                        mel_span, reinterpret_cast<__half*>(y_f16), ys, ylo,
                                                                        reinterpret_cast<__half*>(yb_f16), ybs, yblo);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_a2m_split(const float* x, long long R, int C, void* y1_f16, void* y4_f16, r3dp_stream_t stream) {
    R3DP_REQUIRE(x && (y1_f16 || y4_f16), "a2m_split: null pointer");
    R3DP_REQUIRE(R > 0 && C > 0 && (!y4_f16 || R % 4 == 0), "a2m_split: bad shape");
    a2m_split_kernel<<<blocks(R * C, 256), 256, 0, as_stream(stream)>>>(x, R, C, reinterpret_cast<__half*>(y1_f16), reinterpret_cast<__half*>(y4_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_a2m_latent(const float* z, int B, int T4, float temperature, void* y_f16, r3dp_stream_t stream) {
    R3DP_REQUIRE(z && y_f16, "a2m_latent: null pointer");
    R3DP_REQUIRE(B > 0 && T4 > 0, "a2m_latent: bad shape");
    a2m_latent_kernel<<<blocks((long long)B * T4 * 32, 256), 256, 0, as_stream(stream)>>>(z, B, T4, temperature, reinterpret_cast<__half*>(y_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_a2m_store(const float* x, const float* mask, long long N, int C, float* out, long long ld, r3dp_stream_t stream) {
    R3DP_REQUIRE(x && out, "a2m_store: null pointer");
    R3DP_REQUIRE(N > 0 && C > 0 && ld >= C, "a2m_store: bad shape");
    a2m_store_kernel<<<blocks(N * C, 256), 256, 0, as_stream(stream)>>>(x, mask, N, C, out, ld);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}
