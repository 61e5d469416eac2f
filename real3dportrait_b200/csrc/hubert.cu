// HuBERT (transformers' HubertModel, the hubert-large-ls960-ft architecture: layer-norm conv feature extractor, stable-layer-norm encoder)
// on sm_90a, in split fp16 ([hi | lo] operands, three MMAs per product, fp32 accumulation; weights [hi | lo] of w * 2^10).
//   hb_gemm_kernel       the token GEMM: one TMA producer warp feeds a ring of 64-channel K steps (A hi, A lo, B hi, B lo) to two consumer
//                        warpgroups (setmaxnreg) of 64 rows each; n128 (n64 for the positional conv) wgmma tiles; epilogues: bias -> split
//                        fp16, bias + GELU -> split fp16, bias added into the fp32 residual stream, bias -> fp32, bias + GELU added into
//                        the residual stream (positional conv).  The strided convs read their windows in place: A row t is the k frames
//                        starting at frame s t, a tensor map whose row stride is s frames.  The positional conv is a grouped GEMM whose
//                        K step j is the 128-frame window shifted by tap j, read through a 4-D map (channel, frame, group, segment) whose
//                        out-of-range frames are the per-segment zero padding.
//   hb_attention_kernel  head_dim-64 flash attention over a batch of consecutive segments (no key crosses a segment): TMA producer, two
//                        consumer warpgroups of 64 queries, QK^T and P.V each as three MMAs, fp32 online softmax, P x 2^10 split after it.
//   hb_stats_kernel      the clip's mean and 1 / sqrt(var + 1e-7) (Wav2Vec2FeatureExtractor's do_normalize) in fp64, one CTA, fixed order
//   hb_conv0_kernel      normalise, conv 1 -> C (k10, s5) on CUDA cores, LayerNorm, GELU, split rows
// LayerNorm runs on layernorm.cuh's row kernel (shared with r3dp_sp_layernorm).
#include "common.cuh"
#include "layernorm.cuh"
#include "tc_prims.cuh"
#include <cuda_fp16.h>
#include <math.h>

namespace r3dp {
namespace hb {
using namespace r3dp::tc;

constexpr int kThreads = 384;              // producer warpgroup + 2 consumer warpgroups
constexpr int kProducerRegs = 40, kConsumerRegs = 232;
constexpr int kBM = 128;                   // rows per CTA (64 per consumer warpgroup)
constexpr int kATile = kBM * 128;          // 128 rows x 64 channels fp16 (SWIZZLE_128B rows of 128 B)
constexpr float kInvScale = 1.0f / 1024.0f;

enum Epi { kSplit = 0, kGeluSplit = 1, kResidual = 2, kF32 = 3, kGeluResidual = 4 };

template <int BN>
struct GemmCfg {
    static constexpr int kBTile = BN * 128;
    static constexpr int kStage = 2 * kATile + 2 * kBTile;
    static constexpr int kStages = BN == 128 ? 3 : 4;
    static constexpr int kSmem = kStages * kStage + 1024 + 128;
};

struct GemmArgs {
    int M, N, nk;       // output rows, output columns, K steps of 64 channels
    int seg;            // A columns: K channel kk sits at (kk / seg) * 2 seg + kk % seg (hi), + seg (lo); 0: the positional conv's map
    int blo;            // B: lo columns at blo + kk
    int Lseg, tps, G;   // positional conv: frames per segment, m tiles per segment, groups
    int epi;
    const float* bias;  // [N] or null
    float* yf;
    __half* yh;
    int ldy, ylo;
};

__device__ __forceinline__ float gelu(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }

template <int BN>
__device__ __forceinline__ void mma_step(float* acc, uint64_t a, uint64_t b, uint32_t accumulate) {
    if constexpr (BN == 128) wgmma_m64n128k16(acc, a, b, accumulate);
    else wgmma_m64n64k16(acc, a, b, accumulate);
}

// grid (m tiles, N / BN).  tmA / tmB: 4-D fp16 maps, boxes of 64 channels x 128 (A) / BN (B) rows, zero fill out of range.
template <int BN>
__global__ void __launch_bounds__(kThreads, 1) hb_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                                                             const GemmArgs a) {
    using Cf = GemmCfg<BN>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = align_smem_1024(smem_raw);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + Cf::kStages * Cf::kStage);
    uint64_t* empty = full + Cf::kStages;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int bx = blockIdx.x, n0 = blockIdx.y * BN;
    const bool pos = a.seg == 0;
    const int pseg = pos ? bx / a.tps : 0, pt0 = pos ? (bx % a.tps) * kBM : 0;
    if (threadIdx.x == 0) {
        for (int i = 0; i < Cf::kStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 256); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    }
    __syncthreads();

    if (warp < 4) {
        setmaxnreg_dec<kProducerRegs>();
        if (warp == 0 && lane == 0) {
            for (int ks = 0; ks < a.nk; ++ks) {
                const int s = ks % Cf::kStages;
                mbar_wait(&empty[s], ((ks / Cf::kStages) & 1) ^ 1);
                mbar_expect_tx(&full[s], Cf::kStage);
                uint8_t* st = smem + s * Cf::kStage;
                if (pos) {
                    const int f = pt0 - 64 + ks;                        // tap ks of the centred window (pad 64, the k128 conv's last frame dropped)
                    tma_load_4d(st, &tmA, &full[s], 0, f, blockIdx.y, pseg);
                    tma_load_4d(st + kATile, &tmA, &full[s], 0, f, a.G + blockIdx.y, pseg);
                } else {
                    const int kk = ks * 64;
                    const int col = (kk / a.seg) * 2 * a.seg + kk % a.seg;
                    tma_load_4d(st, &tmA, &full[s], col, bx * kBM, 0, 0);
                    tma_load_4d(st + kATile, &tmA, &full[s], col + a.seg, bx * kBM, 0, 0);
                }
                tma_load_4d(st + 2 * kATile, &tmB, &full[s], ks * 64, n0, 0, 0);
                tma_load_4d(st + 2 * kATile + Cf::kBTile, &tmB, &full[s], a.blo + ks * 64, n0, 0, 0);
            }
        }
        return;
    }
    setmaxnreg_inc<kConsumerRegs>();
    const int g = (warp >> 2) - 1;
    constexpr int NR = BN / 2;
    float acc[NR];
#pragma unroll
    for (int i = 0; i < NR; ++i) acc[i] = 0.f;
    for (int ks = 0; ks < a.nk; ++ks) {
        const int s = ks % Cf::kStages;
        mbar_wait(&full[s], (ks / Cf::kStages) & 1);
        const uint32_t ah = smem_u32(smem + s * Cf::kStage) + g * 64 * 128, al = ah + kATile;
        const uint32_t bh = smem_u32(smem + s * Cf::kStage + 2 * kATile), bl = bh + Cf::kBTile;
        wg_fence_acc<NR>(acc);
        wg_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint64_t dah = gmma_desc_sw128(ah + 32 * k), dbh = gmma_desc_sw128(bh + 32 * k);
            mma_step<BN>(acc, dah, dbh, (ks | k) ? 1u : 0u);
            mma_step<BN>(acc, gmma_desc_sw128(al + 32 * k), dbh, 1u);
            mma_step<BN>(acc, dah, gmma_desc_sw128(bl + 32 * k), 1u);
        }
        wg_commit();
        wg_wait<1>();
        wg_fence_acc<NR>(acc);
        if (ks > 0) mbar_arrive(&empty[(ks - 1) % Cf::kStages]);
    }
    wg_wait<0>();
    wg_fence_acc<NR>(acc);

#pragma unroll
    for (int i = 0; i < NR; i += 2) {
        const int r = g * 64 + acc_row(i);
        long long row;
        if (pos) {
            const int t = pt0 + r;
            row = (long long)pseg * a.Lseg + t;
            if (t >= a.Lseg) continue;
        } else {
            row = (long long)bx * kBM + r;
        }
        const int n = n0 + acc_col(i);
        if (row >= a.M || n >= a.N) continue;
        float v0 = acc[i] * kInvScale, v1 = acc[i + 1] * kInvScale;
        if (a.bias) { v0 += a.bias[n]; v1 += a.bias[n + 1]; }
        if (a.epi == kGeluSplit || a.epi == kGeluResidual) { v0 = gelu(v0); v1 = gelu(v1); }
        const size_t o = (size_t)row * a.ldy + n;
        if (a.epi == kSplit || a.epi == kGeluSplit) {
            const __half2 h = __floats2half2_rn(v0, v1);
            const float2 hf = __half22float2(h);
            *reinterpret_cast<__half2*>(a.yh + o) = h;
            *reinterpret_cast<__half2*>(a.yh + o + a.ylo) = __floats2half2_rn(v0 - hf.x, v1 - hf.y);
        } else if (a.epi == kF32) {
            *reinterpret_cast<float2*>(a.yf + o) = make_float2(v0, v1);
        } else {
            float2* p = reinterpret_cast<float2*>(a.yf + o);
            const float2 y = *p;
            *p = make_float2(y.x + v0, y.y + v1);
        }
    }
}

// ---- flash attention, head_dim 64, split operands -------------------------------------------------------------------------------------
constexpr int kMaxSeg = 64;
constexpr int kHTile = 64 * 128;           // 64 rows x 64 dims fp16
constexpr int kSlots = 3;
constexpr int kFaSmem = 4 * kHTile + kSlots * 4 * kHTile + 1024 + 128;

struct Segs {
    int n;
    int start[kMaxSeg + 1];                // row offsets of the segments (consecutive), start[n] = total rows
    int tile[kMaxSeg + 1];                 // prefix sums of ceil(len / 128)
};

// grid (tile[n], heads).  tm: fp16 rows [rows][ld], boxes of 64 channels x 64 rows.  q / k / v of head h at columns qc / kc / vc + 64 h (hi),
// lo + those (lo).  o: split rows, hi at oc + 64 h, lo at olo + oc + 64 h.
__global__ void __launch_bounds__(kThreads, 1) hb_attention_kernel(const __grid_constant__ CUtensorMap tm, const Segs sg, int qc, int kc, int vc, int lo,
                                                                   __half* __restrict__ o, int os, int olo) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = align_smem_1024(smem_raw);
    uint8_t* sQ = smem;                                  // [warpgroup][hi, lo][64 rows x 128 B]
    uint8_t* sKV = smem + 4 * kHTile;                    // [slot][K hi, K lo, V hi, V lo]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + kSlots * 4 * kHTile);
    uint64_t* q_full = bars;
    uint64_t* kv_full = bars + 1;
    uint64_t* kv_empty = bars + 1 + kSlots;
    const int h = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int s = 0;
    while (s + 1 < sg.n && (int)blockIdx.x >= sg.tile[s + 1]) ++s;
    const int r0 = sg.start[s], len = sg.start[s + 1] - r0;
    const int q0 = r0 + ((int)blockIdx.x - sg.tile[s]) * 128;
    const int nkv = (len + 63) / 64;
    if (threadIdx.x == 0) {
        mbar_init(q_full, 1);
        for (int i = 0; i < kSlots; ++i) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], 256); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tm) : "memory");
    }
    __syncthreads();

    if (warp < 4) {
        setmaxnreg_dec<kProducerRegs>();
        if (warp == 0 && lane == 0) {
            mbar_expect_tx(q_full, 4 * kHTile);
            for (int w = 0; w < 2; ++w) {
                tma_load_4d(sQ + (2 * w) * kHTile, &tm, q_full, qc + 64 * h, q0 + 64 * w, 0, 0);
                tma_load_4d(sQ + (2 * w + 1) * kHTile, &tm, q_full, lo + qc + 64 * h, q0 + 64 * w, 0, 0);
            }
            for (int it = 0; it < nkv; ++it) {
                const int sl = it % kSlots;
                mbar_wait(&kv_empty[sl], ((it / kSlots) & 1) ^ 1);
                mbar_expect_tx(&kv_full[sl], 4 * kHTile);
                uint8_t* b = sKV + sl * 4 * kHTile;
                const int kr = r0 + it * 64;
                tma_load_4d(b, &tm, &kv_full[sl], kc + 64 * h, kr, 0, 0);
                tma_load_4d(b + kHTile, &tm, &kv_full[sl], lo + kc + 64 * h, kr, 0, 0);
                tma_load_4d(b + 2 * kHTile, &tm, &kv_full[sl], vc + 64 * h, kr, 0, 0);
                tma_load_4d(b + 3 * kHTile, &tm, &kv_full[sl], lo + vc + 64 * h, kr, 0, 0);
            }
        }
        return;
    }
    setmaxnreg_inc<kConsumerRegs>();
    const int g = (warp >> 2) - 1;
    float oacc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) oacc[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    const uint32_t qh = smem_u32(sQ + 2 * g * kHTile), ql = qh + kHTile;
    mbar_wait(q_full, 0);
    for (int it = 0; it < nkv; ++it) {
        const int sl = it % kSlots;
        mbar_wait(&kv_full[sl], (it / kSlots) & 1);
        const uint32_t kh = smem_u32(sKV + sl * 4 * kHTile), kl = kh + kHTile, vh = kh + 2 * kHTile, vl = kh + 3 * kHTile;
        float sc[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) sc[i] = 0.f;
        wg_fence_acc<32>(sc);
        wg_fence();
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint64_t dqh = desc_sw128(qh + 32 * j), dkh = desc_sw128(kh + 32 * j);
            wgmma_m64n64k16(sc, dqh, dkh, j ? 1u : 0u);
            wgmma_m64n64k16(sc, desc_sw128(ql + 32 * j), dkh, 1u);
            wgmma_m64n64k16(sc, dqh, desc_sw128(kl + 32 * j), 1u);
        }
        wg_commit();
        wg_wait<0>();
        wg_fence_acc<32>(sc);
        // keys past the segment (the next segment's rows, or zero fill) are masked; online softmax in the log2 domain (the 1/8 scale is in q)
        const int kbase = it * 64;
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            const float v = kbase + acc_col(i) < len ? sc[i] * 1.4426950408889634f : -INFINITY;
            sc[i] = v;
            mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], v);
        }
        float corr[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            const float mn = fmaxf(m[r], mx[r]);            // finite: every tile holds at least one key of the segment
            corr[r] = exp2f(m[r] - mn);
            m[r] = mn;
            l[r] *= corr[r];
        }
        // P x 2^10 split to [hi | lo] fp16 (the scale keeps the lo half of small probabilities out of fp16's subnormals)
        uint32_t ph[4][4], pl[4][4];
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
            const int r = (i >> 1) & 1;
            const float p0 = exp2f(sc[i] - m[r]), p1 = exp2f(sc[i + 1] - m[r]);
            l[r] += p0 + p1;
            const float a0 = 1024.f * p0, a1 = 1024.f * p1;
            const __half2 hh = __floats2half2_rn(a0, a1);
            const float2 hf = __half22float2(hh);
            ph[i >> 3][(i >> 1) & 3] = *reinterpret_cast<const uint32_t*>(&hh);
            pl[i >> 3][(i >> 1) & 3] = pack_h2(a0 - hf.x, a1 - hf.y);
        }
#pragma unroll
        for (int i = 0; i < 32; ++i) oacc[i] *= corr[(i >> 1) & 1];
        wg_fence_acc<32>(oacc);
        wg_fence();
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const uint64_t dvh = desc_sw128(vh + t * 2048);
            wgmma_rs_m64n64k16_tb(oacc, ph[t], dvh);
            wgmma_rs_m64n64k16_tb(oacc, pl[t], dvh);
            wgmma_rs_m64n64k16_tb(oacc, ph[t], desc_sw128(vl + t * 2048));
        }
        wg_commit();
        wg_wait<0>();
        wg_fence_acc<32>(oacc);
        mbar_arrive(&kv_empty[sl]);
    }
    float inv[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
        l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
        inv[r] = 1.f / (1024.f * l[r]);
    }
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
        const int row = q0 + g * 64 + acc_row(i);
        if (row >= r0 + len) continue;
        const float iv = inv[(i >> 1) & 1];
        const float v0 = oacc[i] * iv, v1 = oacc[i + 1] * iv;
        __half* orow = o + (size_t)row * os + 64 * h + acc_col(i);
        const __half2 hh = __floats2half2_rn(v0, v1);
        const float2 hf = __half22float2(hh);
        *reinterpret_cast<__half2*>(orow) = hh;
        *reinterpret_cast<__half2*>(orow + olo) = __floats2half2_rn(v0 - hf.x, v1 - hf.y);
    }
}

// ---- front end ------------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double block_sum_1024(double v, double* red) {
#pragma unroll
    for (int m = 16; m; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    for (int i = 0; i < 32; ++i) t += red[i];
    __syncthreads();
    return t;
}

// one CTA of 1024 threads: stats = (mean, 1 / sqrt(var + 1e-7)) of x[0, L), fp64, two passes, a fixed summation order
__global__ void __launch_bounds__(1024) hb_stats_kernel(const float* __restrict__ x, long long L, double* __restrict__ stats) {
    __shared__ double red[32];
    double s = 0.0;
    for (long long i = threadIdx.x; i < L; i += 1024) s += (double)x[i];
    const double mean = block_sum_1024(s, red) / (double)L;
    double q = 0.0;
    for (long long i = threadIdx.x; i < L; i += 1024) { const double d = (double)x[i] - mean; q += d * d; }
    const double var = block_sum_1024(q, red) / (double)L;
    if (threadIdx.x == 0) { stats[0] = mean; stats[1] = 1.0 / sqrt(var + 1e-7); }
}

// one warp per output frame f (reads samples [5f, 5f + 10)); lane holds channels lane + 32 i.  y: split rows (ys halves, lo at ylo).
__global__ void __launch_bounds__(256) hb_conv0_kernel(const float* __restrict__ x, const double* __restrict__ stats, int F, int C,
                                                       const float* __restrict__ w, const float* __restrict__ bias, const float* __restrict__ gam,
                                                       const float* __restrict__ bet, float eps, __half* __restrict__ y, int ys, int ylo) {
    const int f = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (f >= F) return;
    const double mean = stats[0], rstd = stats[1];
    float xn[10];
#pragma unroll
    for (int j = 0; j < 10; ++j) xn[j] = (float)(((double)x[(size_t)5 * f + j] - mean) * rstd);
    const int nv = C / 32;
    float v[16];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        if (i < nv) {
            const int c = lane + 32 * i;
            float a = bias ? bias[c] : 0.f;
#pragma unroll
            for (int j = 0; j < 10; ++j) a = fmaf(w[c * 10 + j], xn[j], a);
            v[i] = a;
            s += a;
        }
    }
#pragma unroll
    for (int m = 16; m; m >>= 1) s += __shfl_xor_sync(0xffffffffu, s, m);
    const float mu = s / C;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i)
        if (i < nv) { const float d = v[i] - mu; q = fmaf(d, d, q); }
#pragma unroll
    for (int m = 16; m; m >>= 1) q += __shfl_xor_sync(0xffffffffu, q, m);
    const float rs = rsqrtf(q / C + eps);
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        if (i >= nv) break;
        const int c = lane + 32 * i;
        const float u = gelu(fmaf((v[i] - mu) * rs, gam[c], bet[c]));
        const __half hh = __float2half_rn(u);
        y[(size_t)f * ys + c] = hh;
        y[(size_t)f * ys + ylo + c] = __float2half_rn(u - __half2float(hh));
    }
}

inline unsigned blocks(long long n, int t) { return (unsigned)((n + t - 1) / t); }

// fp16 tensor map: dims d[4] (d[0] innermost, halves), byte strides of dims 1..3, box {64, box1, 1, 1}, 128-byte swizzle, zero fill
static int map4(CUtensorMap* m, const void* ptr, const cuuint64_t* dims, const cuuint64_t* strides, int box1, const char* who) {
    EncodeTiledFn fn = encode_fn();
    R3DP_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled is not available from the driver");
    const cuuint32_t box[4] = {64, (cuuint32_t)box1, 1, 1};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    R3DP_REQUIRE(r == CUDA_SUCCESS, "%s: cuTensorMapEncodeTiled failed with CUresult %d", who, (int)r);
    return 0;
}

template <int BN>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const GemmArgs& a, int mtiles, cudaStream_t st) {
    R3DP_CUDA(cudaFuncSetAttribute(hb_gemm_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, GemmCfg<BN>::kSmem));
    hb_gemm_kernel<BN><<<dim3((unsigned)mtiles, (unsigned)((a.N + BN - 1) / BN)), kThreads, GemmCfg<BN>::kSmem, st>>>(ta, tb, a);
    return 0;
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace hb
}  // namespace r3dp

using namespace r3dp;
using namespace r3dp::hb;

extern "C" int r3dp_hb_gemm(const void* a_f16, int M, int a_width, int a_stride, int seg, const void* w_f16, int N, int Kp, const float* bias, int epi,
                            void* y, int ldy, int ylo, r3dp_stream_t stream) {
    R3DP_REQUIRE(a_f16 && w_f16 && y, "hb_gemm: null pointer");
    R3DP_REQUIRE(M > 0 && N > 0 && N % 2 == 0 && Kp > 0 && Kp % 64 == 0 && seg > 0 && seg % 64 == 0 && Kp % seg == 0 &&
                 a_width >= Kp / seg * 2 * seg && a_width % 8 == 0 && a_stride % 8 == 0 && a_stride > 0,
                 "hb_gemm: bad shape (Kp, seg multiples of 64, seg | Kp, A rows of >= 2 Kp halves with strides of 8 halves)");
    R3DP_REQUIRE(epi >= kSplit && epi <= kF32, "hb_gemm: epilogue must be 0 (split), 1 (GELU split), 2 (residual) or 3 (fp32)");
    R3DP_REQUIRE(ldy >= N && (epi > kGeluSplit || (ylo >= N && ldy >= ylo + N)) && ldy % 2 == 0 && ylo % 2 == 0,
                 "hb_gemm: output row stride / lo offset (split rows need ylo >= N and ldy >= ylo + N)");
    R3DP_REQUIRE(aligned16(a_f16) && aligned16(w_f16) && (reinterpret_cast<uintptr_t>(y) & 7) == 0, "hb_gemm: buffer alignment");
    CUtensorMap ta, tb;
    const cuuint64_t ad[4] = {(cuuint64_t)a_width, (cuuint64_t)M, 1, 1};
    const cuuint64_t as[3] = {(cuuint64_t)a_stride * 2, (cuuint64_t)a_stride * 2 * M, (cuuint64_t)a_stride * 2 * M};
    const cuuint64_t bd[4] = {(cuuint64_t)2 * Kp, (cuuint64_t)N, 1, 1};
    const cuuint64_t bs[3] = {(cuuint64_t)4 * Kp, (cuuint64_t)4 * Kp * N, (cuuint64_t)4 * Kp * N};
    if (map4(&ta, a_f16, ad, as, kBM, "hb_gemm A")) return 1;
    const bool wide = N > 64;
    if (map4(&tb, w_f16, bd, bs, wide ? 128 : 64, "hb_gemm B")) return 1;
    GemmArgs g{};
    g.M = M; g.N = N; g.nk = Kp / 64; g.seg = seg; g.blo = Kp; g.epi = epi; g.bias = bias;
    g.yf = reinterpret_cast<float*>(y); g.yh = reinterpret_cast<__half*>(y); g.ldy = ldy; g.ylo = ylo;
    const int mt = (M + kBM - 1) / kBM;
    cudaStream_t st = as_stream(stream);
    if ((wide ? launch_gemm<128>(ta, tb, g, mt, st) : launch_gemm<64>(ta, tb, g, mt, st)) != 0) return 1;
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_hb_pos_conv(const void* x_f16, int nseg, int Lseg, int M, int H, const void* w_f16, const float* bias, float* y,
                                r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && w_f16 && bias && y, "hb_pos_conv: null pointer");
    R3DP_REQUIRE(nseg > 0 && Lseg > 0 && M > (long long)(nseg - 1) * Lseg && M <= (long long)nseg * Lseg && H > 0 && H % 64 == 0,
                 "hb_pos_conv: bad shape (M rows in nseg segments of Lseg; H a multiple of 64)");
    R3DP_REQUIRE(aligned16(x_f16) && aligned16(w_f16) && (reinterpret_cast<uintptr_t>(y) & 7) == 0, "hb_pos_conv: buffer alignment");
    const int G = H / 64;
    CUtensorMap ta, tb;
    const cuuint64_t ad[4] = {64, (cuuint64_t)Lseg, (cuuint64_t)2 * G, (cuuint64_t)nseg};
    const cuuint64_t as[3] = {(cuuint64_t)H * 4, 128, (cuuint64_t)Lseg * H * 4};
    const int Kp = 128 * 64;
    const cuuint64_t bd[4] = {(cuuint64_t)2 * Kp, (cuuint64_t)H, 1, 1};
    const cuuint64_t bs[3] = {(cuuint64_t)4 * Kp, (cuuint64_t)4 * Kp * H, (cuuint64_t)4 * Kp * H};
    if (map4(&ta, x_f16, ad, as, kBM, "hb_pos_conv x") || map4(&tb, w_f16, bd, bs, 64, "hb_pos_conv w")) return 1;
    GemmArgs g{};
    g.M = M; g.N = H; g.nk = 128; g.seg = 0; g.blo = Kp; g.Lseg = Lseg; g.tps = (Lseg + kBM - 1) / kBM; g.G = G; g.epi = kGeluResidual;
    g.bias = bias; g.yf = y; g.ldy = H;
    if (launch_gemm<64>(ta, tb, g, nseg * g.tps, as_stream(stream)) != 0) return 1;
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_hb_attention(const void* qkv_f16, int rows, int ld, int lo, int heads, const int* seg_len, int nseg, void* o_f16, int os, int olo,
                                 r3dp_stream_t stream) {
    R3DP_REQUIRE(qkv_f16 && seg_len && o_f16, "hb_attention: null pointer");
    const int H = 64 * heads;
    R3DP_REQUIRE(heads > 0 && nseg > 0 && nseg <= kMaxSeg && lo >= 3 * H && ld >= lo + 3 * H && ld % 8 == 0 && lo % 8 == 0 && os >= H &&
                 olo >= H && os >= olo + H && os % 2 == 0 && olo % 2 == 0, "hb_attention: bad shape (at most 64 segments)");
    R3DP_REQUIRE(aligned16(qkv_f16) && (reinterpret_cast<uintptr_t>(o_f16) & 3) == 0, "hb_attention: buffer alignment");
    Segs sg{};
    sg.n = nseg;
    long long r = 0, t = 0;
    for (int i = 0; i < nseg; ++i) {
        R3DP_REQUIRE(seg_len[i] > 0, "hb_attention: segment lengths must be positive");
        sg.start[i] = (int)r; sg.tile[i] = (int)t;
        r += seg_len[i]; t += (seg_len[i] + 127) / 128;
    }
    R3DP_REQUIRE(r == rows, "hb_attention: the segment lengths must add up to rows");
    sg.start[nseg] = (int)r; sg.tile[nseg] = (int)t;
    CUtensorMap tm;
    const cuuint64_t d[4] = {(cuuint64_t)ld, (cuuint64_t)rows, 1, 1};
    const cuuint64_t s[3] = {(cuuint64_t)ld * 2, (cuuint64_t)ld * 2 * rows, (cuuint64_t)ld * 2 * rows};
    if (map4(&tm, qkv_f16, d, s, 64, "hb_attention")) return 1;
    R3DP_CUDA(cudaFuncSetAttribute(hb_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kFaSmem));
    hb_attention_kernel<<<dim3((unsigned)t, (unsigned)heads), kThreads, kFaSmem, as_stream(stream)>>>(tm, sg, 0, H, 2 * H, lo,
                                                                                                     reinterpret_cast<__half*>(o_f16), os, olo);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_hb_stats(const float* x, long long L, double* stats, r3dp_stream_t stream) {
    R3DP_REQUIRE(x && stats, "hb_stats: null pointer");
    R3DP_REQUIRE(L > 0, "hb_stats: empty input");
    hb_stats_kernel<<<1, 1024, 0, as_stream(stream)>>>(x, L, stats);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_hb_conv0(const float* x, const double* stats, int F, int C, const float* w, const float* bias, const float* g, const float* b,
                             float eps, void* y_f16, int ys, int ylo, r3dp_stream_t stream) {
    R3DP_REQUIRE(x && stats && w && g && b && y_f16, "hb_conv0: null pointer");
    R3DP_REQUIRE(F > 0 && C % 32 == 0 && C >= 32 && C <= 512 && ylo >= C && ys >= ylo + C, "hb_conv0: bad shape (C a multiple of 32, at most 512)");
    hb_conv0_kernel<<<blocks(F, 8), 256, 0, as_stream(stream)>>>(x, stats, F, C, w, bias, g, b, eps, reinterpret_cast<__half*>(y_f16), ys, ylo);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_hb_layernorm(const float* x, int R, int C, const float* g, const float* b, float eps, int gelu, float* yf, int yfs, void* yh_f16,
                                 int yhs, int yhlo, r3dp_stream_t stream) {
    R3DP_REQUIRE(x && (yf || yh_f16) && (!g == !b), "hb_layernorm: null pointer (g and b go together)");
    R3DP_REQUIRE(R > 0 && C % 32 == 0 && C >= 32 && C <= 1024 && (!yf || yfs >= C) && (!yh_f16 || (yhlo >= C && yhs >= yhlo + C)),
                 "hb_layernorm: bad shape (C a multiple of 32, at most 1024; split rows [hi | lo])");
    __half* yh = reinterpret_cast<__half*>(yh_f16);
    if (C <= 256)
        layernorm_rows_kernel<8><<<blocks(R, 8), 256, 0, as_stream(stream)>>>(x, nullptr, R, C, g, b, eps, nullptr, yf, yfs, yh, yhs, yhlo, gelu);
    else
        layernorm_rows_kernel<32><<<blocks(R, 8), 256, 0, as_stream(stream)>>>(x, nullptr, R, C, g, b, eps, nullptr, yf, yfs, yh, yhs, yhlo, gelu);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}
