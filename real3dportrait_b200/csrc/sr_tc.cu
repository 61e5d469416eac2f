// Tensor-core super-resolution path for sm_90a: the modulated 3x3 convolutions of SuperresolutionHybrid8XDC (197.6 GFLOP/frame,
// SURVEY.md §8d) and the plain convolutions of the torso head as TMA-fed wgmma implicit GEMMs.
//
//   activations  NHWC fp16, channels padded to a multiple of 64 (one 128-byte swizzle row = 64 channels)
//   weights      per-sample folded (modulated+demodulated) fp16, packed [n][tap][Cout][Cin_pad]  (K-major B operand)
//   accumulate   fp32 in registers; epilogue in fp32 (bias, lrelu*sqrt2, ToRGB + skip) then fp16 / fp32 stores
//
// The conv kernel (conv_tc3_kernel): persistent CTAs, M64 x N128 x K16 warpgroup MMAs (two consumer warpgroups = 128 pixels), A row strips
// reused by the horizontal taps through row-shifted descriptors and by the R output rows of a tile.
// The im2col is done by TMA itself: every (tap, 64-channel chunk) of the K loop is a box load at the tap's shifted
// coordinates, zero-filled outside the image (= the conv's zero padding).
//
// The stride-2 transposed convolution of the up layers (conv2d_resample.py:116-133) keeps the reference's operation order for large Cin:
// four output-parity phases (4/2/2/1 taps) as units of ONE launch -> (2H+1)x(2W+1) fp16 result -> fir_tma_kernel (TMA-staged 4x4 FIR +
// bias + lrelu) + upconv_edge_kernel (last column).  For small Cin (block0.conv0) the FIR is composed into the weights instead.
#include "common.cuh"
#include "tc_prims.cuh"
#include <mutex>
#include <vector>
#include <type_traits>
#include <stdlib.h>

#ifndef R3DP_TC_DEBUG_TIMING
#define R3DP_TC_DEBUG_TIMING 0
#endif
namespace r3dp {
namespace tc {

constexpr int BM = 128, BN = 128, BK = 64;
constexpr float kSplitWeightScale = 1024.0f;       // split-fp16 weights are stored x 2^10: their lo halves (|w| 2^-11) stay normal fp16 numbers

// =====================================================================================================================
// Persistent implicit-GEMM conv design (conv_tc3_kernel): R = kConvRows output rows (R x 128 pixels) x 128 couts per tile.
//
// The design cuts the operand fill traffic and the per-tile overheads:
//   * an input ROW STRIP {64 ch, 130 px} is loaded once per 64-channel chunk and serves all horizontal taps (the wgmma smem
//     descriptor starts 128 B x shift later; the 128-byte swizzle is a function of the ABSOLUTE smem address, so the descriptor's
//     base_offset stays 0) and the R output rows that touch it vertically; launches with at most 32 real input channels use {32 ch, 130 px}
//     strips and {32 ch, 128 couts} taps in the 64-byte swizzle instead (Cfg3<32>), so no MMA runs on the zero-padded channels;
//   * every weight tile {64 ch, 128 couts} of a tap is used by R MMA groups before it is released;
//   * persistent CTAs;
//   * the four output-parity phases of a transposed conv are units of ONE launch;
//   * a unit = (image, phase, row group, x block); the CTA loops over the cout blocks of its unit so that ToRGB partial sums of a
//     256-channel layer stay in registers (block0's ToRGB is fused like the last layer's).
// Two mbarrier rings (A strips, B taps) are filled by one TMA lane in exactly the order the consumer warpgroups use them.
// =====================================================================================================================
constexpr int A2_ROWS = 130, A2_SLOT = 17408;                                // 17 x 1024: every slot keeps the swizzle alignment
struct Taps {
    int n, ngroups;                 // taps sorted by (dy, dx); group = taps sharing dy
    int dyi[9], shift[9], widx[9];  // group index, horizontal shift (dx + 1, in pixels: strips start at x0 - 1), weight tap index
    int gstart[4];                  // first tap of each group (+ sentinel)
    int dy_min;
};
struct Phase {
    Taps taps;
    int rows, oy_off, ox_off;       // valid grid rows of this phase; output pixel = (row*oy_mul + oy_off, col*ox_mul + ox_off)
};
enum Mode {
    kStoreAct = 0,                  // bias + activation -> fp16 NHWC
    kStoreRaw = 1,                  // the raw sums -> fp16 NHWC (the transposed conv's grid, filtered afterwards)
    kToRgbFinal = 2,                // only the image: img_out = skip(img_prev) + ToRGB(activated sums) + brgb
    kActRgb = 3                     // kStoreAct + ToRGB/skip accumulated over the cout blocks
};
struct ConvArgs {
    Phase ph[4];
    int n_phases, k_chunks, tiles_x, row_groups, n_blocks, n_images, total_units;
    int w_shared, mode;             // w_shared: all samples use weight set 0; mode: a Mode
    __half* out; int out_H, out_W, out_C, oy_mul, ox_mul;
    // bias [n_blocks * 128]; ToRGB: wrgb [Nw][3][n_blocks * 128], brgb [3], img_out [N][3][img_H][img_W], img_prev at half or (skip_same_res) full size
    const float* bias; const float* wrgb; const float* brgb; const float* img_prev; float* img_out; int img_H, img_W;
    float act_slope, act_gain;      // epilogue activation: v < 0 ? v*slope : v, then * gain  (0.2, sqrt2 = bias_act lrelu; 0.01, 1 = nn.LeakyReLU; 1, 1 = linear)
    int skip_same_res;              // ToRGB skip image has the output resolution (SynthesisBlockNoUp) instead of half (FIR-upsampled)
    const __half* residual;         // non-null: added to the activated output before the store (ResBlock2d of large_sr)
    int out_clamp;                  // final image clamped to [-1, 1] (the caller-side imgs.clamp(-1,1), inference/real3d_infer.py:515)
    uint8_t* img_out_u8;            // non-null: final image as uint8 HWC frames [N][H][W][3] = int((clamp(x)+1)/2*255) (real3d_infer.py:519) instead of fp32 NCHW
    int split;                      // fp32-grade operands: activations [hi | lo] (2 x Cin_pad channels), weights [hi | lo]; K loop = hi*hi + lo*hi + hi*lo
    int lo_off;                     // split: channel offset of the lo half in the OUTPUT tensor (= logical output channels); out_C is the physical pixel stride
    float acc_scale;                // accumulator scale applied before the bias (split weights are stored x 2^10 so their lo halves stay normal fp16)
    unsigned long long* debug;      // R3DP_TC_DEBUG_TIMING builds: [acc wait, strip wait, tap wait, issue, total, #CTAs] clock sums of the MMA warp
};


// FIR-upsampled skip image (upsample2d, upfirdn2d.py:317-354) at output pixel (Y,X): zero-insert x2, pad (2,1,2,1), [1,3,3,1]^2/64 * 4
__device__ __forceinline__ float upsampled_skip(const float* __restrict__ ip, int h, int w, int Y, int X) {
    const float k4[4] = {0.25f, 0.75f, 0.75f, 0.25f};
    float acc = 0.f;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int zy = Y + u - 2;
        if (zy < 0 || (zy & 1) || (zy >> 1) >= h) continue;
        float rowv = 0.f;
#pragma unroll
        for (int v = 0; v < 4; ++v) {
            const int zx = X + v - 2;
            if (zx < 0 || (zx & 1) || (zx >> 1) >= w) continue;
            rowv = fmaf(k4[v], __ldg(ip + (size_t)(zy >> 1) * w + (zx >> 1)), rowv);
        }
        acc = fmaf(k4[u], rowv, acc);
    }
    return acc;
}

// the same sum as upsampled_skip without branches: the two rows / columns of the half-resolution image that reach (Y, X) are (Y-1)>>1
// and its successor with weights (.25,.75) for even Y and (.75,.25) for odd Y; out-of-range taps get weight 0 and a clamped address, so
// the four loads are independent (one L2 round trip) and the fma order - hence the bits - are those of the loop above.
__device__ __forceinline__ float upsampled_skip_bf(const float* __restrict__ ip, int h, int w, int Y, int X) {
    const int y0 = (Y - 1) >> 1, x0 = (X - 1) >> 1;
    const float ky0 = (y0 >= 0 && y0 < h) ? ((Y & 1) ? 0.75f : 0.25f) : 0.f, ky1 = (y0 + 1 < h) ? ((Y & 1) ? 0.25f : 0.75f) : 0.f;
    const float kx0 = (x0 >= 0 && x0 < w) ? ((X & 1) ? 0.75f : 0.25f) : 0.f, kx1 = (x0 + 1 < w) ? ((X & 1) ? 0.25f : 0.75f) : 0.f;
    const int ya = min(max(y0, 0), h - 1), yb = min(y0 + 1, h - 1), xa = min(max(x0, 0), w - 1), xb = min(x0 + 1, w - 1);
    const float v00 = __ldg(ip + (size_t)ya * w + xa), v01 = __ldg(ip + (size_t)ya * w + xb);
    const float v10 = __ldg(ip + (size_t)yb * w + xa), v11 = __ldg(ip + (size_t)yb * w + xb);
    const float r0 = fmaf(kx1, v01, fmaf(kx0, v00, 0.f)), r1 = fmaf(kx1, v11, fmaf(kx0, v10, 0.f));
    return fmaf(ky1, r1, fmaf(ky0, r0, 0.f));
}

__device__ __forceinline__ void store_half32(__half* dst, const float* f) {
    uint4* d4 = reinterpret_cast<uint4*>(dst);
#pragma unroll
    for (int v = 0; v < 4; ++v) {
        __half2 h0 = __floats2half2_rn(f[8 * v + 0], f[8 * v + 1]), h1 = __floats2half2_rn(f[8 * v + 2], f[8 * v + 3]);
        __half2 h2 = __floats2half2_rn(f[8 * v + 4], f[8 * v + 5]), h3 = __floats2half2_rn(f[8 * v + 6], f[8 * v + 7]);
        uint4 pk;
        pk.x = *reinterpret_cast<uint32_t*>(&h0); pk.y = *reinterpret_cast<uint32_t*>(&h1);
        pk.z = *reinterpret_cast<uint32_t*>(&h2); pk.w = *reinterpret_cast<uint32_t*>(&h3);
        d4[v] = pk;
    }
}

// =====================================================================================================================
// conv_tc3_kernel: one CTA per unit stream, three warpgroups.  Warpgroup 0 hands most of its registers to the consumers (setmaxnreg 40) and
// one lane of it issues the TMA loads; warpgroups 1 and 2 (setmaxnreg 232) are the consumers: warpgroup c computes pixels
// [64 (c-1), 64 (c-1) + 64) of both output rows of the tile x all 128 couts (wgmma M64 N128 K16, fp32 accumulators in registers:
// kConvRows x 64 per thread).  The epilogue works on the accumulator fragments: bias and activation per column in registers, ToRGB as
// per-thread partial dot products summed over the quad, fp16 stores through a per-warp swizzled tile.  Ring slots are released one MMA
// group late (wgmma.wait_group 1), so the tensor core always has the next tap queued.
// =====================================================================================================================
constexpr int kConvRows = 2;                                                 // output rows per tile
constexpr int kThreads3 = 384;                                               // TMA warpgroup + 2 consumer warpgroups
constexpr int kProducerRegs = 40, kConsumerRegs = 232;                       // 128 x 40 + 256 x 232 <= 64 K registers
// KC = channels per K chunk: 64 (128-byte rows, SWIZZLE_128B), or 32 for launches with at most 32 real input channels (64-byte rows,
// SWIZZLE_64B: the boxes read the first 32 channels of each 64-channel pixel, so no MMA runs on the zero padding).
template <int KC>
struct Cfg3 {
    // ring depths: what the 227 KB of shared memory leave.  A 3x3 chunk needs kConvRows + 2 = 4 strips and 3 x 3 taps, so 6-deep rings let
    // the producer fill the next chunk while the current one drains; the half-size slots of KC = 32 allow 8 strips and 16 taps.
    static constexpr int ROW = KC * 2;                                       // bytes per pixel row of a strip / per cout row of a tap
    static constexpr int A_BYTES = A2_ROWS * ROW, A_SLOT = KC == BK ? A2_SLOT : (A_BYTES + 1023) / 1024 * 1024;
    static constexpr int B_BYTES = BN * ROW;
    static constexpr int NA = KC == BK ? 6 : 8, NB = KC == BK ? 6 : 16;
    static constexpr int TAIL = 8192;                                        // barriers, bias, ToRGB weights
    static constexpr int STAGE = 8 * 8 * BN * 2;                             // fp16 store staging: 8 consumer warps x 8 px x 128 couts
    static constexpr int SMEM = NA * A_SLOT + NB * B_BYTES + 1024 + TAIL + STAGE;
    static_assert(KC == BK || KC == 32, "conv_tc3: 64- or 32-channel chunks");
    static_assert(SMEM <= 227 * 1024, "conv_tc3: shared memory over the sm_90 per-block limit");
    static_assert(2 * (NA + NB) * 8 <= 512, "conv_tc3: ring barriers overlap the bias");
};
template <int KC>
__device__ __forceinline__ uint64_t conv_desc(uint32_t saddr) { return KC == BK ? gmma_desc_sw128(saddr) : gmma_desc_sw64(saddr); }

template <bool SPLIT, int KC>
__global__ void __launch_bounds__(kThreads3, 1) conv_tc3_kernel(const __grid_constant__ CUtensorMap tmA,
                                                               const __grid_constant__ CUtensorMap tmB, const ConvArgs a) {
    using C = Cfg3<KC>;
    constexpr int R = kConvRows;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = align_smem_1024(smem_raw);
    uint8_t* a_ring = smem;
    uint8_t* b_ring = smem + C::NA * C::A_SLOT;
    uint8_t* tail = b_ring + C::NB * C::B_BYTES;
    uint64_t* a_full = reinterpret_cast<uint64_t*>(tail);
    uint64_t* a_empty = a_full + C::NA;
    uint64_t* b_full = a_empty + C::NA;
    uint64_t* b_empty = b_full + C::NB;
    float* s_bias = reinterpret_cast<float*>(tail + 512);                    // [256]
    float* s_wrgb = s_bias + 256;                                            // [3][n_blocks*128]
    uint4* s_stage = reinterpret_cast<uint4*>(tail + C::TAIL);               // [8 warps][8 px][16 x 16 B] fp16 store staging (XOR-swizzled)

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int units_per_image = a.n_phases * a.row_groups * a.tiles_x;

    if (threadIdx.x == 0) {
        for (int i = 0; i < C::NA; ++i) { mbar_init(&a_full[i], 1); mbar_init(&a_empty[i], 256); }
        for (int i = 0; i < C::NB; ++i) { mbar_init(&b_full[i], 1); mbar_init(&b_empty[i], 256); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    }
    if (warp >= 4) {
        const int t = threadIdx.x - 128;
        for (int e = t; e < a.n_blocks * BN && e < 256; e += 256) s_bias[e] = a.bias ? a.bias[e] : 0.f;
    }
    __syncthreads();

    // unit index -> (image n, phase, row group, x block); x fastest so neighbouring CTAs share strips in L2
    // Multi-phase launches with an even number of x blocks (the 4/2/2/1-tap phases of a transposed conv at W = 256): phases are interleaved,
    // slot = rg * n_phases + p' with ph = (p' + rg) mod n_phases, so that at any moment the CTAs are spread over all phases (the 1- and
    // 2-tap phases need more operand bandwidth per MMA than the 4-tap phase) and every CTA sees every phase.
    const bool mix = a.n_phases > 1 && (a.tiles_x & 1) == 0;
    auto decode = [&](int unit, int& n, int& ph, int& row0, int& col0) {
        n = unit / units_per_image; int r = unit - n * units_per_image;
        const int xb = r % a.tiles_x; r /= a.tiles_x;
        int rg;
        if (mix) { rg = r / a.n_phases; ph = (r - rg * a.n_phases + rg) % a.n_phases; }
        else { rg = r % a.row_groups; ph = r / a.row_groups; }
        row0 = rg * R; col0 = xb * BM;
    };

    if (warp < 4) {
        setmaxnreg_dec<kProducerRegs>();
        // ===== TMA producer (one lane): strips and taps in consumption order; the other three warps are done =====
        if (warp == 0 && lane == 0) {
            uint32_t aq = 0, bq = 0;                                         // running strip / tap sequence numbers
            for (int unit = blockIdx.x; unit < a.total_units; unit += gridDim.x) {
                int n, ph, row0, col0; decode(unit, n, ph, row0, col0);
                const Taps& tp = a.ph[ph].taps;
                const int DY = tp.ngroups;
                const int wn = a.w_shared ? 0 : n;
                const int K3 = SPLIT ? 3 * a.k_chunks : a.k_chunks;               // split: [x_hi w_hi | x_lo w_hi | x_hi w_lo] over the channel chunks
                for (int nblk = 0; nblk < a.n_blocks; ++nblk)
                    for (int kq = 0; kq < K3; ++kq) {
                        const int kc = kq < 2 * a.k_chunks ? kq : kq - 2 * a.k_chunks;    // activation chunk: hi, lo (at k_chunks + c), hi again
                        const int kb = kq < a.k_chunks ? kq : kq - a.k_chunks;            // weight chunk: hi, hi, lo (at k_chunks + c)
                        // chunk c starts at channel 64 c for both widths: KC = 32 has one chunk per half (channels [0, 32) of hi, and of lo at 64)
                        for (int d = 0; d < DY; ++d) {
                            const int s_lo = d == 0 ? 0 : R - 1 + d, s_hi = R - 1 + d;
                            for (int s = s_lo; s <= s_hi; ++s, ++aq) {
                                const int slot = aq % C::NA;
                                mbar_wait(&a_empty[slot], ((aq / C::NA) & 1) ^ 1);
                                mbar_expect_tx(&a_full[slot], C::A_BYTES);
                                tma_load_4d(a_ring + slot * C::A_SLOT, &tmA, &a_full[slot], kc * BK, col0 - 1, row0 + tp.dy_min + s, n);
                            }
                            for (int t = tp.gstart[d]; t < tp.gstart[d + 1]; ++t, ++bq) {
                                const int slot = bq % C::NB;
                                mbar_wait(&b_empty[slot], ((bq / C::NB) & 1) ^ 1);
                                mbar_expect_tx(&b_full[slot], C::B_BYTES);
                                tma_load_4d(b_ring + slot * C::B_BYTES, &tmB, &b_full[slot], kb * BK, nblk * BN, tp.widx[t], wn);
                            }
                        }
                    }
            }
        }
    } else {
        setmaxnreg_inc<kConsumerRegs>();
        // ===== consumers: warpgroup wg = 0, 1 multiplies pixels [64 wg, 64 wg + 64) of each row; then the epilogue =====
        // The thread holds fragment rows (tile pixels) pix + 8 h, h = 0, 1, and columns (couts) 8 i + 2 quad + e of the cout block.
        const int wg = (warp >> 2) - 1;
        const int quad = lane & 3, pix = 64 * wg + 16 * (warp & 3) + (lane >> 2);
        const bool want_rgb = (a.mode == kToRgbFinal) || (a.mode == kActRgb);
        const int CW = a.n_blocks * BN;                                      // channels ToRGB sums over
        float brgb[3] = {0.f, 0.f, 0.f};
        if (want_rgb) { brgb[0] = a.brgb[0]; brgb[1] = a.brgb[1]; brgb[2] = a.brgb[2]; }
        int n_loaded = -1;
        uint32_t aq = 0, bq = 0;
        // slots read by the most recently committed MMA group, released once the NEXT group has been committed and this one has retired
        int pend_b = -1; uint32_t pend_a0 = 0, pend_an = 0;
        auto release_pending = [&]() {
            if (pend_b >= 0) mbar_arrive(&b_empty[pend_b]);
            for (uint32_t s = 0; s < pend_an; ++s) mbar_arrive(&a_empty[(pend_a0 + s) % C::NA]);
            pend_b = -1; pend_an = 0;
        };
        float acc[R][64];
        for (int unit = blockIdx.x; unit < a.total_units; unit += gridDim.x) {
            int n, ph, row0, col0; decode(unit, n, ph, row0, col0);
            const Phase& P = a.ph[ph];
            const Taps& tp = P.taps;
            const int DY = tp.ngroups, NS = R + DY - 1;
            const int wn = a.w_shared ? 0 : n;
            if (want_rgb && wn != n_loaded) {
                asm volatile("bar.sync 1, 256;" ::: "memory");               // all eight consumer warps are done with the old weights
                for (int e = threadIdx.x - 128; e < 3 * CW; e += 256) s_wrgb[e] = a.wrgb[(size_t)wn * 3 * CW + e];
                asm volatile("bar.sync 1, 256;" ::: "memory");
                n_loaded = wn;
            }
            // ToRGB: after the quad sum, lane quad = h (h = 0, 1) finishes pixel pix + 8 h of every row
            const bool rgb_lane = want_rgb && quad < 2;
            const int X = (col0 + pix + 8 * quad) * a.ox_mul + P.ox_off;
            float rgb[R][2][3];
#pragma unroll
            for (int j = 0; j < R; ++j)
#pragma unroll
                for (int h = 0; h < 2; ++h) { rgb[j][h][0] = 0.f; rgb[j][h][1] = 0.f; rgb[j][h][2] = 0.f; }
            // skip-image taps of the finishing lanes' pixels, fetched before the K loop (clamped addresses, zero weights outside the image:
            // the loads are independent)
            float skipv[R][3];
#pragma unroll
            for (int j = 0; j < R; ++j) { skipv[j][0] = 0.f; skipv[j][1] = 0.f; skipv[j][2] = 0.f; }
            if (rgb_lane && a.img_prev) {
                if (a.skip_same_res) {
                    const int Xc = min(X, a.img_W - 1);
#pragma unroll
                    for (int j = 0; j < R; ++j) {
                        const int Yc = min((row0 + j) * a.oy_mul + P.oy_off, a.img_H - 1);
#pragma unroll
                        for (int c = 0; c < 3; ++c) skipv[j][c] = __ldg(a.img_prev + (((size_t)n * 3 + c) * a.img_H + Yc) * a.img_W + Xc);
                    }
                } else {
                    const int h = a.img_H / 2, w = a.img_W / 2;
                    const int x0 = (X - 1) >> 1;
                    const float kx0 = (x0 >= 0 && x0 < w) ? ((X & 1) ? 0.75f : 0.25f) : 0.f, kx1 = (x0 + 1 < w) ? ((X & 1) ? 0.25f : 0.75f) : 0.f;
                    const int xa = min(max(x0, 0), w - 1), xb = min(max(x0 + 1, 0), w - 1);
#pragma unroll
                    for (int j = 0; j < R; ++j) {
                        const int Y = (row0 + j) * a.oy_mul + P.oy_off, y0 = (Y - 1) >> 1;
                        const float ky0 = (y0 >= 0 && y0 < h) ? ((Y & 1) ? 0.75f : 0.25f) : 0.f;
                        const float ky1 = (y0 + 1 < h) ? ((Y & 1) ? 0.25f : 0.75f) : 0.f;
                        const int ya = min(max(y0, 0), h - 1), yb = min(max(y0 + 1, 0), h - 1);
#pragma unroll
                        for (int c = 0; c < 3; ++c) {                        // the fma order of upsampled_skip
                            const float* ip = a.img_prev + ((size_t)n * 3 + c) * h * w;
                            const float v0 = __ldg(ip + ya * w + xa), v1 = __ldg(ip + ya * w + xb), v2 = __ldg(ip + yb * w + xa), v3 = __ldg(ip + yb * w + xb);
                            const float r0 = fmaf(kx1, v1, fmaf(kx0, v0, 0.f)), r1 = fmaf(kx1, v3, fmaf(kx0, v2, 0.f));
                            skipv[j][c] = fmaf(ky1, r1, fmaf(ky0, r0, 0.f));
                        }
                    }
                }
            }
            for (int nblk = 0; nblk < a.n_blocks; ++nblk) {
                // ---- K loop: (channel chunk) x (dy group) x (tap), R rows per tap, 4 k-steps of 16 channels ----
                const int K3 = SPLIT ? 3 * a.k_chunks : a.k_chunks;
                for (int kc = 0; kc < K3; ++kc) {
                    const uint32_t a_base = aq;                               // sequence number of strip 0 of this chunk
                    for (int d = 0; d < DY; ++d) {
                        const int s_lo = d == 0 ? 0 : R - 1 + d, s_hi = R - 1 + d;
                        for (int s = s_lo; s <= s_hi; ++s, ++aq) mbar_wait(&a_full[aq % C::NA], (aq / C::NA) & 1);
                        for (int t = tp.gstart[d]; t < tp.gstart[d + 1]; ++t, ++bq) {
                            const int bslot = bq % C::NB;
                            mbar_wait(&b_full[bslot], (bq / C::NB) & 1);
                            const uint64_t db = conv_desc<KC>(smem_u32(b_ring + bslot * C::B_BYTES));
                            const int sh = tp.shift[t];
                            const uint32_t first = (uint32_t)(kc | t);
                            uint64_t da[R];
#pragma unroll
                            for (int j = 0; j < R; ++j) da[j] = conv_desc<KC>(smem_u32(a_ring + ((a_base + j + d) % C::NA) * C::A_SLOT) + C::ROW * (64 * wg + sh));
                            wg_fence();
#pragma unroll
                            for (int k = 0; k < KC / 16; ++k) {
#pragma unroll
                                for (int j = 0; j < R; ++j) wgmma_m64n128k16(acc[j], da[j] + (uint64_t)(2 * k), db + (uint64_t)(2 * k), first | (uint32_t)k);
                            }
                            wg_commit();
                            wg_wait<1>();                                     // the previous group has retired: its slots can be refilled
                            release_pending();
                            pend_b = bslot;
                        }
                        // strips no later group needs: strip d after group d; everything left after the last group
                        if (d < DY - 1) { pend_a0 = a_base + d; pend_an = 1; }
                        else { pend_a0 = a_base + DY - 1; pend_an = (uint32_t)(NS - (DY - 1)); }
                    }
                }
                wg_wait<0>();
#pragma unroll
                for (int j = 0; j < R; ++j) wg_fence_acc<64>(acc[j]);
                release_pending();
                // ---- epilogue on the fragments: d[4 i + 2 h + e] of row j is pixel pix + 8 h, cout nblk * 128 + 8 i + 2 quad + e ----
                if (a.mode == kStoreRaw) {
                    if (SPLIT) {
#pragma unroll
                        for (int j = 0; j < R; ++j)
#pragma unroll
                            for (int i = 0; i < 64; ++i) acc[j][i] = __fmul_rn(acc[j][i], a.acc_scale);
                    }
                } else {
                    // bias, leaky relu as max(v, v*slope) (slope <= 1), gain: bias_act lrelu*sqrt2 | nn.LeakyReLU | linear
#pragma unroll
                    for (int i = 0; i < 16; ++i) {
                        const float2 b2 = *reinterpret_cast<const float2*>(s_bias + nblk * BN + 8 * i + 2 * quad);
#pragma unroll
                        for (int j = 0; j < R; ++j)
#pragma unroll
                            for (int h = 0; h < 2; ++h)
#pragma unroll
                                for (int e = 0; e < 2; ++e) {
                                    float& x = acc[j][4 * i + 2 * h + e];
                                    const float b = e ? b2.y : b2.x;
                                    const float v = SPLIT ? __fmaf_rn(x, a.acc_scale, b) : __fadd_rn(x, b);
                                    x = __fmul_rn(fmaxf(v, __fmul_rn(v, a.act_slope)), a.act_gain);
                                }
                    }
                }
                if (SPLIT && a.residual) {
                    // ResBlock2d with split operands: the residual [hi | lo] (the output's layout) is summed to fp32 and added to the activated
                    // value BEFORE the hi/lo split, so the stored pair is the split of the full fp32 sum
#pragma unroll
                    for (int j = 0; j < R; ++j) {
                        const int row = row0 + j, Y = row * a.oy_mul + P.oy_off;
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const int Xr = (col0 + pix + 8 * h) * a.ox_mul + P.ox_off;
                            if (row >= P.rows || Y >= a.out_H || Xr >= a.out_W) continue;
                            const __half* rp = a.residual + (((size_t)n * a.out_H + Y) * a.out_W + Xr) * a.out_C + nblk * BN + 2 * quad;
#pragma unroll
                            for (int i = 0; i < 16; ++i) {
                                const float2 rh = __half22float2(__ldg(reinterpret_cast<const __half2*>(rp + 8 * i)));
                                const float2 rl = __half22float2(__ldg(reinterpret_cast<const __half2*>(rp + a.lo_off + 8 * i)));
                                acc[j][4 * i + 2 * h] += rh.x + rl.x;
                                acc[j][4 * i + 2 * h + 1] += rh.y + rl.y;
                            }
                        }
                    }
                }
                if (a.mode != kToRgbFinal) {
                    // NHWC fp16 store through smem, 8 pixels of the warp at a time: the fragment's 4-byte pairs go to pixel row lane / 4,
                    // 16-byte chunk i ^ (lane / 4) (conflict-free), then each half-warp writes one pixel's 256 contiguous bytes.
                    // Split mode: a second pass stores the fp16 remainders (v - fp16(v)) lo_off channels further.
                    uint4* st = s_stage + (warp - 4) * 128;
                    uint32_t* st32 = reinterpret_cast<uint32_t*>(st);
                    const int sr = lane >> 2;
                    constexpr int passes = SPLIT ? 2 : 1;
#pragma unroll
                    for (int j = 0; j < R; ++j) {
                        const int row = row0 + j, Y = row * a.oy_mul + P.oy_off;
                        const bool row_ok = (row < P.rows) && (Y < a.out_H);
#pragma unroll
                        for (int pass = 0; pass < passes; ++pass)
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
#pragma unroll
                                for (int i = 0; i < 16; ++i) {
                                    float x0 = acc[j][4 * i + 2 * h], x1 = acc[j][4 * i + 2 * h + 1];
                                    if (pass) { x0 = x0 - __half2float(__float2half_rn(x0)); x1 = x1 - __half2float(__float2half_rn(x1)); }
                                    const __half2 hv = __floats2half2_rn(x0, x1);
                                    st32[sr * 64 + (i ^ sr) * 4 + quad] = *reinterpret_cast<const uint32_t*>(&hv);
                                }
                                __syncwarp();
#pragma unroll
                                for (int it = 0; it < 4; ++it) {
                                    const int p = 2 * it + (lane >> 4), cch = lane & 15;
                                    uint4 pk = st[p * 16 + (cch ^ p)];
                                    const int Xp = (col0 + pix - sr + p + 8 * h) * a.ox_mul + P.ox_off;
                                    if (row_ok && Xp < a.out_W) {
                                        const size_t eo = ((size_t)n * a.out_H + Y) * a.out_W * a.out_C + nblk * BN + (size_t)Xp * a.out_C + cch * 8 + pass * a.lo_off;
                                        if (!SPLIT && a.residual) {          // ResBlock2d: out = act(conv) + x (superresolution.py:283-288), same NHWC fp16 layout as the output
                                            const uint4 rv = __ldg(reinterpret_cast<const uint4*>(a.residual + eo));
                                            __half2* ph2 = reinterpret_cast<__half2*>(&pk); const __half2* rh = reinterpret_cast<const __half2*>(&rv);
#pragma unroll
                                            for (int e = 0; e < 4; ++e) { const float2 x = __half22float2(ph2[e]), r = __half22float2(rh[e]); ph2[e] = __floats2half2_rn(x.x + r.x, x.y + r.y); }
                                        }
                                        *reinterpret_cast<uint4*>(a.out + eo) = pk;
                                    }
                                }
                                __syncwarp();
                            }
                    }
                }
                if (want_rgb) {
                    // per-thread partial dot products over the thread's 32 couts of this block, carried across the cout blocks
#pragma unroll
                    for (int c = 0; c < 3; ++c)
#pragma unroll
                        for (int i = 0; i < 16; ++i) {
                            const float2 w2 = *reinterpret_cast<const float2*>(s_wrgb + c * CW + nblk * BN + 8 * i + 2 * quad);
#pragma unroll
                            for (int j = 0; j < R; ++j)
#pragma unroll
                                for (int h = 0; h < 2; ++h)
                                    rgb[j][h][c] = fmaf(acc[j][4 * i + 2 * h + 1], w2.y, fmaf(acc[j][4 * i + 2 * h], w2.x, rgb[j][h][c]));
                        }
                }
            }
            if (want_rgb) {
                // the four lanes of a quad hold the partial sums of the same two pixels
#pragma unroll
                for (int j = 0; j < R; ++j)
#pragma unroll
                    for (int h = 0; h < 2; ++h)
#pragma unroll
                        for (int c = 0; c < 3; ++c) {
                            rgb[j][h][c] += __shfl_xor_sync(0xffffffffu, rgb[j][h][c], 1);
                            rgb[j][h][c] += __shfl_xor_sync(0xffffffffu, rgb[j][h][c], 2);
                        }
                if (rgb_lane) {
#pragma unroll
                    for (int j = 0; j < R; ++j) {
                        const int row = row0 + j, Y = row * a.oy_mul + P.oy_off;
                        if (row >= P.rows || Y >= a.out_H || X >= a.out_W) continue;
#pragma unroll
                        for (int c = 0; c < 3; ++c) {
                            float v = ((quad ? rgb[j][1][c] : rgb[j][0][c]) + skipv[j][c]) + brgb[c];
                            if (a.out_clamp) v = fminf(fmaxf(v, -1.0f), 1.0f);
                            if (a.img_out_u8)          // torch: ((x + 1) / 2 * 255.).int() -> uint8, every step rounded in fp32, truncation
                                a.img_out_u8[(((size_t)n * a.img_H + Y) * a.img_W + X) * 3 + c] =
                                    (uint8_t)(int)__fmul_rn(__fmul_rn(__fadd_rn(v, 1.0f), 0.5f), 255.0f);
                            else
                                a.img_out[(((size_t)n * 3 + c) * a.img_H + Y) * a.img_W + X] = v;
                        }
                    }
                }
            }
        }
    }
}

// ---- helpers around the GEMMs ---------------------------------------------------------------------------------------
// fp16 pair of a fp32 value: hi = fp16(v), lo = fp16(v - hi)  (v = hi + lo to ~2^-22 |v| while lo is a normal fp16 number)
__device__ __forceinline__ void split_half(float v, __half& hi, __half& lo) {
    hi = __float2half_rn(v);
    lo = __float2half_rn(v - __half2float(hi));
}

// wf fp32 [Nw][O][I][3][3] -> packed fp16 [Nw][9][O][Ip]  (zero for i >= I); split: [Nw][9][O][2*Ip] = [hi | lo] of wf * 2^10
__global__ void pack_weights_kernel(const float* __restrict__ wf, int Nw, int O, int I, int Ip, int split, __half* __restrict__ out) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)Nw * 9 * O * Ip;
    if (idx >= total) return;
    const int i = (int)(idx % Ip); const int o = (int)((idx / Ip) % O); const int t = (int)((idx / ((long long)Ip * O)) % 9);
    const int nw = (int)(idx / ((long long)Ip * O * 9));
    const float v = i < I ? wf[(((size_t)nw * O + o) * I + i) * 9 + t] : 0.f;
    if (!split) { out[idx] = __float2half_rn(v); return; }
    __half hi, lo;
    split_half(v * kSplitWeightScale, hi, lo);
    const size_t row = (idx / Ip) * (size_t)(2 * Ip);
    out[row + i] = hi; out[row + Ip + i] = lo;
}

// bilinear up-resize (or copy when size == h) of NCHW fp32 -> NHWC fp16 with channel padding to Cp
__global__ void resize_to_nhwc_f16_kernel(const float* __restrict__ x, int N, int C, int h, int w, int size, int Cp, int split, __half* __restrict__ y) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * size * size * Cp) return;
    const int c = (int)(idx % Cp); const int ox = (int)((idx / Cp) % size); const int oy = (int)((idx / ((long long)Cp * size)) % size);
    const int n = (int)(idx / ((long long)Cp * size * size));
    float v = 0.f;
    if (c < C) {
        int y0, y1, x0, x1;
        float ty, tx;
        bilinear_coord(oy, h, size, y0, y1, ty);
        bilinear_coord(ox, w, size, x0, x1, tx);
        const float* p = x + ((size_t)n * C + c) * h * w;
        v = bilinear_mix(p[y0 * w + x0], p[y1 * w + x0], p[y0 * w + x1], p[y1 * w + x1], ty, tx);
    }
    if (!split) { y[idx] = __float2half_rn(v); return; }
    __half hi, lo;
    split_half(v, hi, lo);
    const size_t pix = (idx / Cp) * (size_t)(2 * Cp);
    y[pix + c] = hi; y[pix + Cp + c] = lo;
}

// last column X = 2W of the transposed-conv result (the only part of the (2H+1)x(2W+1) grid the 128-wide GEMM tiles do not
// cover): yb[n][Y][2W][co] = sum_{ci, ky == Y (mod 2)} x[(Y-ky)/2][W-1][ci] * w[ky*3+2][co][ci].
// CTA = 32 couts x 16 rows of one image.  The kx = 2 column of the kernel for these couts ([3][32][Cp] fp16) and the <= 10 input
// pixels are staged in smem; thread (co, row pair) then runs plain dot products - no cross-lane reductions.  Cp <= 256.
constexpr int kEdgeRows = 16, kEdgeRowsSplit = 16, kEdgeCo = 32;      // (64 rows per CTA - the weight column staged 9 instead of 33 times per image - measured slower: 28.3 vs 25.3 us, 144 CTAs are too few)
__global__ void __launch_bounds__(256) upconv_edge_kernel(const __half* __restrict__ x, const __half* __restrict__ wp, int H, int W, int Cp, int O,
                                                          int w_shared, __half* __restrict__ yb) {
    extern __shared__ __align__(16) uint8_t edge_smem[];
    __half* s_x = reinterpret_cast<__half*>(edge_smem);                      // [10][Cp]
    __half* s_w = s_x + (kEdgeRows / 2 + 2) * Cp;                            // [3][32][Cp + 8]   (+8 halfs: rows land in different banks)
    const int WS = Cp + 8;
    const int n = blockIdx.z, Y0 = blockIdx.x * kEdgeRows, co0 = blockIdx.y * kEdgeCo;
    const int BH = 2 * H + 1, BW = 2 * W + 1;
    const int wn = w_shared ? 0 : n;
    const int iy0 = Y0 / 2 - 1;                                              // first input row any of these Y can touch
    const int vec = Cp / 8;
    for (int e = threadIdx.x; e < (kEdgeRows / 2 + 2) * vec; e += 256) {
        const int r = e / vec, c8 = e - r * vec, iy = iy0 + r;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (iy >= 0 && iy < H) v = __ldg(reinterpret_cast<const uint4*>(x + (((size_t)n * H + iy) * W + (W - 1)) * Cp) + c8);
        *reinterpret_cast<uint4*>(s_x + r * Cp + c8 * 8) = v;
    }
    for (int e = threadIdx.x; e < 3 * kEdgeCo * vec; e += 256) {
        const int c8 = e % vec, co = (e / vec) % kEdgeCo, ky = e / (vec * kEdgeCo);
        uint4 v = make_uint4(0, 0, 0, 0);
        if (co0 + co < O) v = __ldg(reinterpret_cast<const uint4*>(wp + (((size_t)wn * 9 + ky * 3 + 2) * O + co0 + co) * Cp) + c8);
        *reinterpret_cast<uint4*>(s_w + (ky * kEdgeCo + co) * WS + c8 * 8) = v;
    }
    __syncthreads();
    const int co = threadIdx.x & 31, yp = threadIdx.x >> 5;                  // 8 warps x 2 rows each; lanes = couts
    if (co0 + co >= O) return;
    constexpr int RPW = kEdgeRows / 8;                                        // rows per warp
#pragma unroll 2
    for (int hh = 0; hh < RPW; ++hh) {
        const int yy = yp * RPW + hh, Y = Y0 + yy;
        if (Y >= BH) continue;
        float acc = 0.f;
        for (int ky = (yy & 1); ky < 3; ky += 2) {                           // Y0 is even: parity of Y == parity of yy
            const int r = ((yy - ky) >> 1) + 1;                              // == (Y-ky)/2 - iy0 ; rows outside the image hold zeros
            const uint4* xr = reinterpret_cast<const uint4*>(s_x + r * Cp);
            const uint4* wr = reinterpret_cast<const uint4*>(s_w + (ky * kEdgeCo + co) * WS);
            for (int c8 = 0; c8 < vec; ++c8) {
                const uint4 xv = xr[c8], wv = wr[c8];
                const __half2* xh = reinterpret_cast<const __half2*>(&xv);
                const __half2* wh = reinterpret_cast<const __half2*>(&wv);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 a = __half22float2(xh[j]), b = __half22float2(wh[j]);
                    acc = fmaf(a.x, b.x, acc); acc = fmaf(a.y, b.y, acc);
                }
            }
        }
        yb[(((size_t)n * BH + Y) * BW + 2 * W) * O + co0 + co] = __float2half_rn(acc);
    }
}

// FIR 4x4 (pad 1, gain 4) + bias + lrelu*sqrt2 on the transposed-conv result: yb [N][2H+1][2W+1][C] fp16 -> y [N][2H][2W][C] fp16.
// HBM-bound stencil (read 1x + write 1x), done the Blackwell way: a persistent CTA streams {64 ch, 35 px, 11 rows} boxes of yb
// into shared memory with ONE TMA instruction each (double-buffered on mbarriers; the box is zero-filled outside the image,
// which IS the FIR's zero padding), then 256 threads (32 px x 8 channel-vectors) march down the tile: 4 swizzled LDS.128 per
// input row -> horizontal taps -> 4-row register window -> vertical taps, bias, lrelu -> one 16-byte store per output row.
constexpr int FIR_TW = 32, FIR_TH = 8, FIR_SEG = 32, FIR_BW = FIR_TW + 3, FIR_BH = FIR_TH + 3;
constexpr int FIR_BOX8_BYTES = FIR_BW * FIR_TH * 128;
constexpr int FIR_BOX_BYTES = FIR_BW * FIR_BH * 128, FIR_SLOT = (FIR_BOX_BYTES + 1023) / 1024 * 1024;
constexpr int FIR_SMEM = 2 * FIR_SLOT + 1024 + 64;
// (d0,d1) += (a0,a1) * (b0,b1)
__device__ __forceinline__ void ffma2(float& d0, float& d1, float a0, float a1, float b0, float b1) {
    d0 = __fmaf_rn(a0, b0, d0); d1 = __fmaf_rn(a1, b1, d1);
}
// Work item = a strip of FIR_TW px x FIR_SEG output rows of one 64-channel group, streamed as FIR_SEG / FIR_TH chunks: the first box has the
// 3 halo rows (35 px x 11 rows), the following boxes only new rows (35 x 8) - the 4-row register window simply keeps rolling across the
// chunks, so only 35 input rows are loaded and converted per 32 output rows (ncu on the one-box-per-tile form: 386 MB read for 270 MB of
// input, the vertical halo rows came from DRAM twice).  A two-output-pixels-per-thread variant (2.5 LDS.128 and 20 converts per output vector
// instead of 4 and 32) was measured at 122-124 us against 124.5-126 us and dropped: the pass is not bound by instruction issue alone.
template <bool SPLIT>
__global__ void __launch_bounds__(256) fir_tma_kernel(const __grid_constant__ CUtensorMap tmY, const __grid_constant__ CUtensorMap tmY8,
                                                      const float* __restrict__ bias, int N, int OH, int OW, int C, __half* __restrict__ y) {
    // SPLIT: yb and y hold [hi | lo] fp16 halves of C channels each (fp32-grade path): both halves of a tile are loaded, summed in fp32,
    // filtered, and the result is split again
    constexpr int NSL = SPLIT ? 2 : 1;
    constexpr int NCH = FIR_SEG / FIR_TH;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = align_smem_1024(smem_raw);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + 2 * NSL * FIR_SLOT);
    const int tid = threadIdx.x, px = tid >> 3, c8 = tid & 7;
    const int tiles_x = OW / FIR_TW, segs = (OH + FIR_SEG - 1) / FIR_SEG, cgs = C / 64;
    const int total = N * cgs * segs * tiles_x;
    const int my_items = (int)blockIdx.x < total ? (total - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    const int nseq = my_items * NCH;
    const int CS = SPLIT ? 2 * C : C;                                      // physical channels per pixel
    if (tid == 0) {
        mbar_init(&full[0], 1); mbar_init(&full[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmY) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmY8) : "memory");
    }
    __syncthreads();
    auto item_of = [&](int s, int& tx, int& sg, int& cg, int& n) {
        int r = blockIdx.x + (s / NCH) * gridDim.x;
        tx = r % tiles_x; r /= tiles_x;
        sg = r % segs; r /= segs;
        cg = r % cgs; n = r / cgs;
    };
    auto issue = [&](int s, int buf) {
        int tx, sg, cg, n; item_of(s, tx, sg, cg, n);
        const int c = s % NCH;
        const int y0 = sg * FIR_SEG - 1 + (c == 0 ? 0 : FIR_BH + FIR_TH * (c - 1));
        const CUtensorMap* map = c == 0 ? &tmY : &tmY8;
        mbar_expect_tx(&full[buf], NSL * (c == 0 ? FIR_BOX_BYTES : FIR_BOX8_BYTES));
        tma_load_4d(smem + buf * NSL * FIR_SLOT, map, &full[buf], cg * 64, tx * FIR_TW - 1, y0, n);
        if (SPLIT) tma_load_4d(smem + (buf * NSL + 1) * FIR_SLOT, map, &full[buf], C + cg * 64, tx * FIR_TW - 1, y0, n);
    };
    if (tid == 0) {
        if (nseq > 0) issue(0, 0);
        if (nseq > 1) issue(1, 1);
    }
    const float k4[4] = {0.25f, 0.75f, 0.75f, 0.25f};
    float win[4][8];
    float b[8];
    for (int s = 0; s < nseq; ++s) {
        const int buf = s & 1, c = s % NCH;
        int tx, sg, cg, n; item_of(s, tx, sg, cg, n);
        if (c == 0) {
#pragma unroll
            for (int j = 0; j < 8; ++j) b[j] = bias[cg * 64 + c8 * 8 + j];
#pragma unroll
            for (int rr = 0; rr < 4; ++rr)
#pragma unroll
                for (int j = 0; j < 8; ++j) win[rr][j] = 0.f;
        }
        mbar_wait(&full[buf], (s >> 1) & 1);
        const uint8_t* sb = smem + buf * NSL * FIR_SLOT;
        const int ox = tx * FIR_TW + px;
        const int gy0 = c == 0 ? 0 : FIR_BH + FIR_TH * (c - 1);            // index of this box's first row inside the item's 35 input rows
        auto rows = [&](auto nrows_tag) {
            constexpr int NROWS = decltype(nrows_tag)::value;
#pragma unroll
            for (int ry = 0; ry < NROWS; ++ry) {
#pragma unroll
                for (int j = 0; j < 8; ++j) { win[0][j] = win[1][j]; win[1][j] = win[2][j]; win[2][j] = win[3][j]; win[3][j] = 0.f; }
#pragma unroll
                for (int v = 0; v < 4; ++v) {
                    const int row = ry * FIR_BW + px + v;                        // 128-byte row of the box; swizzle = chunk ^ (row & 7)
                    const uint4 raw = *reinterpret_cast<const uint4*>(sb + row * 128 + ((c8 ^ (row & 7)) << 4));
                    const __half2* h = reinterpret_cast<const __half2*>(&raw);
                    uint4 rawl = make_uint4(0, 0, 0, 0);
                    if (SPLIT) rawl = *reinterpret_cast<const uint4*>(sb + FIR_SLOT + row * 128 + ((c8 ^ (row & 7)) << 4));
                    const __half2* hl = reinterpret_cast<const __half2*>(&rawl);
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        float2 f = __half22float2(h[j]);
                        if (SPLIT) { const float2 g = __half22float2(hl[j]); f.x += g.x; f.y += g.y; }
                        ffma2(win[3][2 * j], win[3][2 * j + 1], k4[v], k4[v], f.x, f.y);
                    }
                }
                const int gy = gy0 + ry;
                if (gy >= 3) {
                    const int oy = sg * FIR_SEG + gy - 3;
                    if (oy < OH) {
                        uint4 pk; __half2* ph = reinterpret_cast<__half2*>(&pk);
                        uint4 pl; __half2* pq = reinterpret_cast<__half2*>(&pl);
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            float a0 = b[2 * j], a1 = b[2 * j + 1];
#pragma unroll
                            for (int u = 0; u < 4; ++u) ffma2(a0, a1, k4[u], k4[u], win[u][2 * j], win[u][2 * j + 1]);
                            a0 = (a0 < 0.f ? a0 * 0.2f : a0) * 1.4142135623730951f; a1 = (a1 < 0.f ? a1 * 0.2f : a1) * 1.4142135623730951f;
                            ph[j] = __floats2half2_rn(a0, a1);
                            if (SPLIT) { const float2 hf = __half22float2(ph[j]); pq[j] = __floats2half2_rn(a0 - hf.x, a1 - hf.y); }
                        }
                        __half* dst = y + (((size_t)n * OH + oy) * OW + ox) * CS + cg * 64 + c8 * 8;
                        *reinterpret_cast<uint4*>(dst) = pk;
                        if (SPLIT) *reinterpret_cast<uint4*>(dst + C) = pl;
                    }
                }
            }
        };
        if (c == 0) rows(std::integral_constant<int, FIR_BH>{}); else rows(std::integral_constant<int, FIR_TH>{});
        __syncthreads();                                                      // everyone is done reading this buffer
        if (tid == 0 && s + 2 < nseq) issue(s + 2, buf);
    }
}

// split-operand version of upconv_edge_kernel (fp32-grade path): x [N][H][W][2*Cp] and the packed weights [..][2*Cp] hold [hi | lo] halves, the
// weights x 2^10; both are summed to fp32 while they are staged, the dot products run in fp32, the result is written as [hi | lo] of O channels.
__global__ void __launch_bounds__(256) upconv_edge_split_kernel(const __half* __restrict__ x, const __half* __restrict__ wp, int H, int W, int Cp, int O,
                                                                int w_shared, __half* __restrict__ yb) {
    extern __shared__ __align__(16) uint8_t edge_smem[];
    float* s_x = reinterpret_cast<float*>(edge_smem);                        // [10][Cp]
    float* s_w = s_x + (kEdgeRowsSplit / 2 + 2) * Cp;                             // [3][32][Cp + 4]
    const int WS = Cp + 4;
    const int n = blockIdx.z, Y0 = blockIdx.x * kEdgeRowsSplit, co0 = blockIdx.y * kEdgeCo;
    const int BH = 2 * H + 1, BW = 2 * W + 1;
    const int wn = w_shared ? 0 : n;
    const int iy0 = Y0 / 2 - 1;
    for (int e = threadIdx.x; e < (kEdgeRowsSplit / 2 + 2) * Cp; e += 256) {
        const int r = e / Cp, c = e - r * Cp, iy = iy0 + r;
        float v = 0.f;
        if (iy >= 0 && iy < H) { const __half* px = x + (((size_t)n * H + iy) * W + (W - 1)) * 2 * Cp; v = __half2float(px[c]) + __half2float(px[Cp + c]); }
        s_x[r * Cp + c] = v;
    }
    for (int e = threadIdx.x; e < 3 * kEdgeCo * Cp; e += 256) {
        const int c = e % Cp, co = (e / Cp) % kEdgeCo, ky = e / (Cp * kEdgeCo);
        float v = 0.f;
        if (co0 + co < O) { const __half* pw = wp + (((size_t)wn * 9 + ky * 3 + 2) * O + co0 + co) * 2 * Cp; v = __half2float(pw[c]) + __half2float(pw[Cp + c]); }
        s_w[(ky * kEdgeCo + co) * WS + c] = v;
    }
    __syncthreads();
    const int co = threadIdx.x & 31, yp = threadIdx.x >> 5;
    if (co0 + co >= O) return;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        const int yy = yp * 2 + half, Y = Y0 + yy;
        if (Y >= BH) continue;
        float acc = 0.f;
        for (int ky = (yy & 1); ky < 3; ky += 2) {
            const int r = ((yy - ky) >> 1) + 1;
            const float4* xr = reinterpret_cast<const float4*>(s_x + r * Cp);
            const float4* wr = reinterpret_cast<const float4*>(s_w + (ky * kEdgeCo + co) * WS);
            for (int c4 = 0; c4 < Cp / 4; ++c4) {
                const float4 a = xr[c4], b = wr[c4];
                acc = fmaf(a.x, b.x, acc); acc = fmaf(a.y, b.y, acc); acc = fmaf(a.z, b.z, acc); acc = fmaf(a.w, b.w, acc);
            }
        }
        acc *= 1.0f / kSplitWeightScale;
        __half hi, lo;
        split_half(acc, hi, lo);
        __half* dst = yb + (((size_t)n * BH + Y) * BW + 2 * W) * 2 * O + co0 + co;
        dst[0] = hi; dst[O] = lo;
    }
}

// ToRGB for the first block: x NHWC fp16 [N][H][W][C] -> img_out NCHW fp32 = upsample2d(img_prev) + conv1x1 + bias.  One warp per
// 32 consecutive pixels is wasteful on loads, so: one thread per pixel, 16-byte channel vectors, weights in smem.
// SPLIT: x is [N][H][W][2C] = [hi | lo]; the dot product runs over hi + lo in fp32.
template <bool SPLIT>
__global__ void __launch_bounds__(256) torgb_f16_kernel(const __half* __restrict__ x, const float* __restrict__ wrgb, const float* __restrict__ brgb,
                                                        const float* __restrict__ img_prev, int H, int W, int C, int w_shared, int same_res,
                                                        float* __restrict__ img_out) {
    extern __shared__ float s_w[];                               // [3][C]
    const int n = blockIdx.y;
    const int wn = w_shared ? 0 : n;
    for (int e = threadIdx.x; e < 3 * C; e += blockDim.x) s_w[e] = wrgb[(size_t)wn * 3 * C + e];
    __syncthreads();
    const int pix = blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= H * W) return;
    const int Y = pix / W, X = pix - Y * W;
    const uint4* xp = reinterpret_cast<const uint4*>(x + ((size_t)n * H * W + pix) * (SPLIT ? 2 * C : C));
    float r = 0.f, g = 0.f, b = 0.f;
    for (int c8 = 0; c8 < C / 8; ++c8) {
        const uint4 raw = __ldg(xp + c8);
        const __half2* h = reinterpret_cast<const __half2*>(&raw);
        uint4 rawl = make_uint4(0, 0, 0, 0);
        if (SPLIT) rawl = __ldg(xp + C / 8 + c8);
        const __half2* hl = reinterpret_cast<const __half2*>(&rawl);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float2 f = __half22float2(h[j]);
            if (SPLIT) { const float2 fl = __half22float2(hl[j]); f.x += fl.x; f.y += fl.y; }
            const int c = c8 * 8 + 2 * j;
            r = fmaf(f.x, s_w[c], r); r = fmaf(f.y, s_w[c + 1], r);
            g = fmaf(f.x, s_w[C + c], g); g = fmaf(f.y, s_w[C + c + 1], g);
            b = fmaf(f.x, s_w[2 * C + c], b); b = fmaf(f.y, s_w[2 * C + c + 1], b);
        }
    }
    float out[3] = {r + brgb[0], g + brgb[1], b + brgb[2]};
    if (img_prev && same_res) {                                  // rgb = rgb + to_rgb(x) (LargeSynthesisBlock, superresolution.py:311,328)
#pragma unroll
        for (int c = 0; c < 3; ++c) out[c] += img_prev[((size_t)n * 3 + c) * H * W + pix];
    } else if (img_prev) {
        const int h = H / 2, w = W / 2;
#pragma unroll
        for (int c = 0; c < 3; ++c) out[c] += upsampled_skip(img_prev + ((size_t)n * 3 + c) * h * w, h, w, Y, X);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) img_out[((size_t)n * 3 + c) * H * W + pix] = out[c];
}

// ---- host side: tensor maps -----------------------------------------------------------------------------------------
// fp16 tensor [d3][d2][d1][d0] (d0 innermost, dense) read in boxes of box[0..3] elements, zero fill outside
static int make_map(CUtensorMap* m, const void* ptr, const cuuint64_t (&dims)[4], const cuuint32_t (&box)[4], CUtensorMapSwizzle swizzle,
                    CUtensorMapL2promotion l2) {
    EncodeTiledFn fn = encode_fn();
    R3DP_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled is not available from the driver");
    const cuuint64_t strides[3] = {dims[0] * 2, dims[0] * dims[1] * 2, dims[0] * dims[1] * dims[2] * 2};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    swizzle, l2, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    R3DP_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with CUresult %d (dims %llu x %llu x %llu x %llu)", (int)r,
                 (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2], (unsigned long long)dims[3]);
    return 0;
}

// ---- optional in-library timing of the conv launches (bench.py's roofline): CUDA events on the launching stream around each launch --------
struct ConvProf { bool on = false; std::vector<cudaEvent_t> ev; size_t used = 0; };
static ConvProf g_prof;
static void prof_mark(cudaStream_t st) {
    if (!g_prof.on) return;
    if (g_prof.used == g_prof.ev.size()) { cudaEvent_t e; if (cudaEventCreate(&e) != cudaSuccess) return; g_prof.ev.push_back(e); }
    cudaEventRecord(g_prof.ev[g_prof.used++], st);
}

static unsigned long long* g_debug_buf = nullptr;
static int g_debug_launch = 0;
template <bool SPLIT, int KC>
static int launch_conv3_s(const CUtensorMap& tmA, const CUtensorMap& tmB, ConvArgs a, cudaStream_t st) {
    R3DP_CUDA(cudaFuncSetAttribute(conv_tc3_kernel<SPLIT, KC>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg3<KC>::SMEM));
    a.debug = g_debug_buf ? g_debug_buf + 24 * (g_debug_launch++ % 32) : nullptr;
    a.total_units = a.n_images * a.n_phases * a.row_groups * a.tiles_x;
    const int grid = a.total_units < sm_count() ? a.total_units : sm_count();
    prof_mark(st);
    conv_tc3_kernel<SPLIT, KC><<<grid, kThreads3, Cfg3<KC>::SMEM, st>>>(tmA, tmB, a);
    R3DP_LAUNCH_CHECK();
    prof_mark(st);
    count_launches(1);
    return 0;
}

// ---- host side: conv_tc3 launch descriptions -------------------------------------------------------------------------
// Taps are added in (dy, dx) order, so the taps sharing a dy are contiguous and form one group.  The order within a group is the order of
// the fp32 accumulation: it decides the output bits.
static void add_tap(Taps& t, int dy, int dx, int widx) {
    if (t.n == 0) t.dy_min = dy;
    if (t.n == 0 || dy - t.dy_min != t.dyi[t.n - 1]) t.gstart[t.ngroups++] = t.n;
    t.dyi[t.n] = dy - t.dy_min; t.shift[t.n] = dx + 1; t.widx[t.n] = widx;         // strip box starts at x0 - 1
    t.gstart[t.ngroups] = ++t.n;
}
// 3x3 box on weight taps base + (dy + 1) * 3 + (dx + 1)  (base = 9 * phase for the composed up weights)
static Taps taps_3x3(int base) {
    Taps t = {};
    for (int i = 0; i < 9; ++i) add_tap(t, i / 3 - 1, i % 3 - 1, base + i);
    return t;
}
// 1x1 conv: the centre tap of the packed 3x3 weights
static Taps taps_1x1() {
    Taps t = {};
    add_tap(t, 0, 0, 4);
    return t;
}
// output parity (p, q) of the stride-2 transposed conv: the kernel rows ky == p (mod 2), read at dy = -(ky >> 1); the same for columns (4/2/2/1 taps)
static Taps taps_transposed(int p, int q) {
    Taps t = {};
    for (int dy = -1; dy <= 0; ++dy)
        for (int dx = -1; dx <= 0; ++dx) {
            const int ky = p - 2 * dy, kx = q - 2 * dx;
            if (ky < 3 && kx < 3) add_tap(t, dy, dx, ky * 3 + kx);
        }
    return t;
}
// output parity (p, q) of nearest-up x2 + 3x3: taps dy in {p - 1, p}, dx in {q - 1, q} of the composed weight set p * 2 + q
static Taps taps_up_nearest(int p, int q) {
    Taps t = {};
    for (int dy = p - 1; dy <= p; ++dy)
        for (int dx = q - 1; dx <= q; ++dx) add_tap(t, dy, dx, (p * 2 + q) * 9 + (dy + 1) * 3 + (dx + 1));
    return t;
}

// the output y [N][out_H][out_W][O] fp16 NHWC and what the epilogue writes to it; grid pixel (row, col) of a phase lands at
// (row * mul + oy_off, col * mul + ox_off)
static void set_output(ConvArgs& a, Mode mode, void* y, int out_H, int out_W, int O, int mul) {
    a.mode = mode; a.out = reinterpret_cast<__half*>(y); a.out_H = out_H; a.out_W = out_W; a.out_C = O; a.oy_mul = a.ox_mul = mul;
}

constexpr float kLreluSlope = 0.2f, kLreluGain = 1.4142135623730951f;          // bias_act lrelu: max(v, 0.2 v) * sqrt2

// Runs the launch a describes (phases, output, epilogue).  x [N][H][W][Cp] is the input grid; wp [Nw][w_taps][O][Cp] the packed weights
// (w_taps = 9, or 36 for four composed phase sets).  I = the real input channels; x and wp hold them padded to Cp = I rounded up to 64.
// I <= 32 runs the 32-channel K chunks (KC = 32).
static int run_conv(const void* x, int N, int H, int W, int I, const void* wp, int Nw, int w_taps, int O, ConvArgs a, cudaStream_t st) {
    CUtensorMap tmA, tmB;
    const int Cp = (I + 63) / 64 * 64;
    const bool kc32 = I <= 32;
    const cuuint64_t Cphys = (cuuint64_t)Cp * (a.split ? 2 : 1);                  // split: [hi | lo] halves of Cp channels each
    const cuuint32_t kc = kc32 ? 32 : BK;
    const CUtensorMapSwizzle swizzle = kc32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B;
    if (make_map(&tmA, x, {Cphys, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N}, {kc, A2_ROWS, 1, 1}, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B))
        return 1;
    if (make_map(&tmB, wp, {Cphys, (cuuint64_t)O, (cuuint64_t)w_taps, (cuuint64_t)Nw}, {kc, BN, 1, 1}, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B))
        return 1;
    if (a.split) { a.acc_scale = 1.0f / kSplitWeightScale; a.lo_off = a.out_C; a.out_C *= 2; }
    else { a.acc_scale = 1.0f; a.lo_off = 0; }
    // W = 64 (the torso warper's 64^2 maps): one tile per row whose right half reads TMA zero fill and stores nothing (the stores check out_W)
    a.k_chunks = Cp / BK; a.tiles_x = (W + BM - 1) / BM; a.n_blocks = O / BN; a.n_images = N; a.w_shared = (Nw == 1);
    int max_rows = 0;
    for (int p = 0; p < a.n_phases; ++p) max_rows = a.ph[p].rows > max_rows ? a.ph[p].rows : max_rows;
    a.row_groups = (max_rows + kConvRows - 1) / kConvRows;
    R3DP_REQUIRE(a.n_blocks >= 1 && a.n_blocks <= 2, "conv_tc3: 128 or 256 output channels");
    if (kc32) return a.split ? launch_conv3_s<true, 32>(tmA, tmB, a, st) : launch_conv3_s<false, 32>(tmA, tmB, a, st);
    return a.split ? launch_conv3_s<true, BK>(tmA, tmB, a, st) : launch_conv3_s<false, BK>(tmA, tmB, a, st);
}

// Plain nn.Conv2d (k = 1 or 3, stride 1, "same" padding) at the input's resolution, y [N][H][W][O] fp16: act = max(v, v * slope) * gain,
// residual (if any) added after it.  The launch behind the up == 1 SynthesisLayer, r3dp_sr_tc_conv(_res) / r3dp_sr_tcx_conv(_res) and
// r3dp_tw_conv (shapes checked by the callers).
static int conv_plain_launch(const void* x_f16, const void* wp_f16, const float* bias, int N, int Nw, int I, int O, int H, int W, int ksize,
                             float slope, float gain, const void* residual_f16, void* y_f16, int split, r3dp_stream_t stream) {
    ConvArgs a = {};
    a.n_phases = 1; a.ph[0] = {ksize == 3 ? taps_3x3(0) : taps_1x1(), H, 0, 0};
    set_output(a, kStoreAct, y_f16, H, W, O, 1);
    a.bias = bias; a.act_slope = slope; a.act_gain = gain; a.residual = reinterpret_cast<const __half*>(residual_f16); a.split = split;
    return run_conv(x_f16, N, H, W, I, wp_f16, Nw, 9, O, a, as_stream(stream));
}

}  // namespace tc
}  // namespace r3dp

using namespace r3dp;
using namespace r3dp::tc;

static int pack_weights_impl(const float* wf, int Nw, int O, int I, void* packed_f16, int split, r3dp_stream_t stream) {
    R3DP_REQUIRE(wf && packed_f16, "sr_tc_pack_weights: null pointer");
    R3DP_REQUIRE(Nw > 0 && O > 0 && I > 0, "sr_tc_pack_weights: bad shape");
    const int Ip = (I + 63) / 64 * 64;
    const long long total = (long long)Nw * 9 * O * Ip;
    pack_weights_kernel<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(wf, Nw, O, I, Ip, split, reinterpret_cast<__half*>(packed_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}
extern "C" int r3dp_sr_tc_pack_weights(const float* wf, int Nw, int O, int I, void* packed_f16, r3dp_stream_t stream) { return pack_weights_impl(wf, Nw, O, I, packed_f16, 0, stream); }
extern "C" int r3dp_sr_tcx_pack_weights(const float* wf, int Nw, int O, int I, void* packed_f16, r3dp_stream_t stream) { return pack_weights_impl(wf, Nw, O, I, packed_f16, 1, stream); }

static int input_impl(const float* x, int N, int C, int h, int w, int size, void* y_f16, int split, r3dp_stream_t stream) {
    R3DP_REQUIRE(x && y_f16, "sr_tc_input: null pointer");
    R3DP_REQUIRE(N > 0 && C > 0 && h > 0 && w > 0 && size >= h && size >= w, "sr_tc_input: up-scaling (or copy) only");
    const int Cp = (C + 63) / 64 * 64;
    const long long total = (long long)N * size * size * Cp;
    resize_to_nhwc_f16_kernel<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(x, N, C, h, w, size, Cp, split, reinterpret_cast<__half*>(y_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}
extern "C" int r3dp_sr_tc_input(const float* x, int N, int C, int h, int w, int size, void* y_f16, r3dp_stream_t stream) { return input_impl(x, N, C, h, w, size, y_f16, 0, stream); }
extern "C" int r3dp_sr_tcx_input(const float* x, int N, int C, int h, int w, int size, void* y_f16, r3dp_stream_t stream) { return input_impl(x, N, C, h, w, size, y_f16, 1, stream); }

extern "C" size_t r3dp_sr_tc_scratch_bytes(int N, int O, int H, int W) { return (size_t)N * (2 * H + 1) * (2 * W + 1) * O * sizeof(__half); }
extern "C" size_t r3dp_sr_tcx_scratch_bytes(int N, int O, int H, int W) { return 2 * r3dp_sr_tc_scratch_bytes(N, O, H, W); }

// SynthesisLayer on tensor cores.  x [N][H][W][Ip] fp16 NHWC (Ip = I rounded up to 64), wp packed weights [Nw][9][O][Ip] fp16
// (Nw == N per-sample, or 1 shared), bias [O] fp32.  up == 1: y [N][H][W][O]; up == 2: y [N][2H][2W][O], scratch >= r3dp_sr_tc_scratch_bytes.
static int layer_impl(const void* x_f16, const void* wp_f16, const float* bias, int N, int Nw, int I, int O, int H, int W, int up,
                      void* y_f16, void* scratch, int split, r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && wp_f16 && bias && y_f16, "sr_tc_layer: null pointer");
    R3DP_REQUIRE(N > 0 && (Nw == N || Nw == 1) && I > 0 && H > 0, "sr_tc_layer: bad shape");
    R3DP_REQUIRE(W % BM == 0 && O % BN == 0, "sr_tc_layer: needs W %% 128 == 0 and Cout %% 128 == 0 (got W=%d, Cout=%d)", W, O);
    R3DP_REQUIRE(up == 1 || up == 2, "sr_tc_layer: up must be 1 or 2");
    if (up == 1) return conv_plain_launch(x_f16, wp_f16, bias, N, Nw, I, O, H, W, 3, kLreluSlope, kLreluGain, nullptr, y_f16, split, stream);
    R3DP_REQUIRE(scratch, "sr_tc_layer: up=2 needs scratch");
    const int Ip = (I + 63) / 64 * 64;
    cudaStream_t st = as_stream(stream);
    __half* yb = reinterpret_cast<__half*>(scratch);
    // all four output-parity phases of the stride-2 transposed conv in ONE persistent launch: raw sums on the (2H+1)x(2W+1) grid, whose
    // bias and activation the FIR pass applies
    ConvArgs a = {};
    a.n_phases = 4;
    for (int p = 0; p < 4; ++p) a.ph[p] = {taps_transposed(p >> 1, p & 1), p < 2 ? H + 1 : H, p >> 1, p & 1};
    set_output(a, kStoreRaw, yb, 2 * H + 1, 2 * W + 1, O, 2);
    a.split = split;
    if (run_conv(x_f16, N, H, W, I, wp_f16, Nw, 9, O, a, st)) return 1;
    // the grid's last column; the split form stages fp32 operands
    R3DP_REQUIRE(Ip <= 256, "sr_tc_layer: up=2 supports at most 256 input channels");
    const int erows = split ? kEdgeRowsSplit : kEdgeRows;
    const dim3 egrid((2 * H + 1 + erows - 1) / erows, (O + kEdgeCo - 1) / kEdgeCo, N);
    const size_t esmem = split ? ((size_t)(kEdgeRowsSplit / 2 + 2) * Ip + 3 * (size_t)kEdgeCo * (Ip + 4)) * sizeof(float)
                               : ((size_t)(kEdgeRows / 2 + 2) * Ip + 3 * (size_t)kEdgeCo * (Ip + 8)) * sizeof(__half);
    const auto edge = split ? upconv_edge_split_kernel : upconv_edge_kernel;
    R3DP_CUDA(cudaFuncSetAttribute(edge, cudaFuncAttributeMaxDynamicSharedMemorySize, split ? 128 * 1024 : 80 * 1024));
    edge<<<egrid, 256, esmem, st>>>(reinterpret_cast<const __half*>(x_f16), reinterpret_cast<const __half*>(wp_f16), H, W, Ip, O, Nw == 1, yb);
    // the FIR pass.  128-byte L2 promotion: a box row is 128 B (one 64-channel group) of a pixel that is 2 or 4 such groups wide, and the other
    // groups are read by work items far away in the schedule; 256-byte promotion fetched the neighbouring group from DRAM too, and it was
    // evicted before its use.
    R3DP_REQUIRE((2 * W) % FIR_TW == 0 && O % 64 == 0, "sr_tc_layer: FIR needs 2W %% 32 == 0 and Cout %% 64 == 0");
    CUtensorMap tmY, tmY8;
    const cuuint64_t ydims[4] = {(cuuint64_t)O * (split ? 2 : 1), (cuuint64_t)(2 * W + 1), (cuuint64_t)(2 * H + 1), (cuuint64_t)N};
    if (make_map(&tmY, yb, ydims, {64, FIR_BW, FIR_BH, 1}, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B)) return 1;
    if (make_map(&tmY8, yb, ydims, {64, FIR_BW, FIR_TH, 1}, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B)) return 1;
    const int total = N * (O / 64) * ((2 * H + FIR_SEG - 1) / FIR_SEG) * (2 * W / FIR_TW);
    // persistent CTAs, as many as are resident at once: two per SM, one with the split form's twice as large buffers
    const auto fir = split ? fir_tma_kernel<true> : fir_tma_kernel<false>;
    const int fsmem = split ? 4 * FIR_SLOT + 1024 + 64 : FIR_SMEM;
    const int fcap = split ? sm_count() : 2 * sm_count();
    R3DP_CUDA(cudaFuncSetAttribute(fir, cudaFuncAttributeMaxDynamicSharedMemorySize, fsmem));
    fir<<<total < fcap ? total : fcap, 256, fsmem, st>>>(tmY, tmY8, bias, N, 2 * H, 2 * W, O, reinterpret_cast<__half*>(y_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(2);
    return 0;
}
extern "C" int r3dp_sr_tc_layer(const void* x_f16, const void* wp_f16, const float* bias, int N, int Nw, int I, int O, int H, int W, int up,
                                void* y_f16, void* scratch, r3dp_stream_t stream) {
    return layer_impl(x_f16, wp_f16, bias, N, Nw, I, O, H, W, up, y_f16, scratch, 0, stream);
}
extern "C" int r3dp_sr_tcx_layer(const void* x_f16, const void* wp_f16, const float* bias, int N, int Nw, int I, int O, int H, int W, int up,
                                 void* y_f16, void* scratch, r3dp_stream_t stream) {
    return layer_impl(x_f16, wp_f16, bias, N, Nw, I, O, H, W, up, y_f16, scratch, 1, stream);
}

// Last layer fused with ToRGB: conv3x3 (I -> 128) + bias + lrelu, then img_out = upsample2d(img_prev) + torgb + brgb; the 128-channel
// activation itself is never written (SynthesisBlock is_last: only the image leaves the block).
static int last_layer_impl(const void* x_f16, const void* wp_f16, const float* bias, const float* wrgb, const float* brgb,
                           const float* img_prev, int N, int Nw, int I, int H, int W, float* img_out, uint8_t* img_out_u8, int clamp, int split,
                           r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && wp_f16 && bias && wrgb && brgb && (img_out || img_out_u8), "sr_tc_last_layer: null pointer");
    R3DP_REQUIRE(N > 0 && (Nw == N || Nw == 1) && W % BM == 0 && H % 2 == 0, "sr_tc_last_layer: bad shape");
    ConvArgs a = {};
    a.n_phases = 1; a.ph[0] = {taps_3x3(0), H, 0, 0};
    set_output(a, kToRgbFinal, nullptr, H, W, BN, 1);
    a.bias = bias; a.act_slope = kLreluSlope; a.act_gain = kLreluGain;
    a.wrgb = wrgb; a.brgb = brgb; a.img_prev = img_prev; a.img_out = img_out; a.img_H = H; a.img_W = W;
    a.img_out_u8 = img_out_u8; a.out_clamp = clamp || img_out_u8; a.split = split;
    return run_conv(x_f16, N, H, W, I, wp_f16, Nw, 9, BN, a, as_stream(stream));
}
extern "C" int r3dp_sr_tc_last_layer_ex(const void* x_f16, const void* wp_f16, const float* bias, const float* wrgb, const float* brgb,
                                        const float* img_prev, int N, int Nw, int I, int H, int W, float* img_out, uint8_t* img_out_u8, int clamp,
                                        r3dp_stream_t stream) {
    return last_layer_impl(x_f16, wp_f16, bias, wrgb, brgb, img_prev, N, Nw, I, H, W, img_out, img_out_u8, clamp, 0, stream);
}
extern "C" int r3dp_sr_tcx_last_layer(const void* x_f16, const void* wp_f16, const float* bias, const float* wrgb, const float* brgb,
                                      const float* img_prev, int N, int Nw, int I, int H, int W, float* img_out, uint8_t* img_out_u8, int clamp,
                                      r3dp_stream_t stream) {
    return last_layer_impl(x_f16, wp_f16, bias, wrgb, brgb, img_prev, N, Nw, I, H, W, img_out, img_out_u8, clamp, 1, stream);
}
extern "C" int r3dp_sr_tc_last_layer(const void* x_f16, const void* wp_f16, const float* bias, const float* wrgb, const float* brgb,
                                     const float* img_prev, int N, int Nw, int I, int H, int W, float* img_out, r3dp_stream_t stream) {
    return r3dp_sr_tc_last_layer_ex(x_f16, wp_f16, bias, wrgb, brgb, img_prev, N, Nw, I, H, W, img_out, nullptr, 0, stream);
}

// ToRGB of a non-final block: x NHWC fp16 [N][H][W][C] -> img_out NCHW fp32 [N][3][H][W] (+ upsample2d(img_prev) + bias).
static int torgb_impl(const void* x_f16, const float* wrgb, const float* brgb, const float* img_prev, int same_res, int N, int Nw, int C,
                      int H, int W, float* img_out, int split, r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && wrgb && brgb && img_out, "sr_tc_torgb: null pointer");
    R3DP_REQUIRE(N > 0 && (Nw == N || Nw == 1) && C % 8 == 0 && H % 2 == 0 && W % 2 == 0, "sr_tc_torgb: bad shape");
    dim3 grid((H * W + 255) / 256, N);
    auto kern = split ? torgb_f16_kernel<true> : torgb_f16_kernel<false>;
    kern<<<grid, 256, 3 * C * sizeof(float), as_stream(stream)>>>(reinterpret_cast<const __half*>(x_f16), wrgb, brgb, img_prev, H, W, C,
                                                                  Nw == 1, same_res, img_out);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}
extern "C" int r3dp_sr_tc_torgb_ex(const void* x_f16, const float* wrgb, const float* brgb, const float* img_prev, int same_res, int N, int Nw, int C,
                                   int H, int W, float* img_out, r3dp_stream_t stream) {
    return torgb_impl(x_f16, wrgb, brgb, img_prev, same_res, N, Nw, C, H, W, img_out, 0, stream);
}
extern "C" int r3dp_sr_tcx_torgb_ex(const void* x_f16, const float* wrgb, const float* brgb, const float* img_prev, int same_res, int N, int Nw, int C,
                                    int H, int W, float* img_out, r3dp_stream_t stream) {
    return torgb_impl(x_f16, wrgb, brgb, img_prev, same_res, N, Nw, C, H, W, img_out, 1, stream);
}
extern "C" int r3dp_sr_tc_torgb(const void* x_f16, const float* wrgb, const float* brgb, const float* img_prev, int N, int Nw, int C, int H,
                                int W, float* img_out, r3dp_stream_t stream) {
    return r3dp_sr_tc_torgb_ex(x_f16, wrgb, brgb, img_prev, 0, N, Nw, C, H, W, img_out, stream);
}

// SynthesisLayer (up == 1) fused with the block's ToRGB + skip (networks_stylegan2.py:463-469): y [N,H,W,O] fp16 AND
// img_out [N,3,H,W] fp32 = upsample2d(img_prev [N,3,H/2,W/2]) + conv1x1(y, wrgb [Nw,3,O]) + brgb.  O = 128 or 256.
static int layer_torgb_impl(const void* x_f16, const void* wp_f16, const float* bias, const float* wrgb, const float* brgb,
                            const float* img_prev, int N, int Nw, int I, int O, int H, int W, void* y_f16, float* img_out, int split,
                            r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && wp_f16 && bias && wrgb && brgb && y_f16 && img_out, "sr_tc_layer_torgb: null pointer");
    R3DP_REQUIRE(N > 0 && (Nw == N || Nw == 1) && W % BM == 0 && O % BN == 0 && O <= 256 && H % 2 == 0, "sr_tc_layer_torgb: bad shape");
    ConvArgs a = {};
    a.n_phases = 1; a.ph[0] = {taps_3x3(0), H, 0, 0};
    set_output(a, kActRgb, y_f16, H, W, O, 1);
    a.bias = bias; a.act_slope = kLreluSlope; a.act_gain = kLreluGain;
    a.wrgb = wrgb; a.brgb = brgb; a.img_prev = img_prev; a.img_out = img_out; a.img_H = H; a.img_W = W; a.split = split;
    return run_conv(x_f16, N, H, W, I, wp_f16, Nw, 9, O, a, as_stream(stream));
}
extern "C" int r3dp_sr_tc_layer_torgb(const void* x_f16, const void* wp_f16, const float* bias, const float* wrgb, const float* brgb,
                                      const float* img_prev, int N, int Nw, int I, int O, int H, int W, void* y_f16, float* img_out,
                                      r3dp_stream_t stream) {
    return layer_torgb_impl(x_f16, wp_f16, bias, wrgb, brgb, img_prev, N, Nw, I, O, H, W, y_f16, img_out, 0, stream);
}
extern "C" int r3dp_sr_tcx_layer_torgb(const void* x_f16, const void* wp_f16, const float* bias, const float* wrgb, const float* brgb,
                                       const float* img_prev, int N, int Nw, int I, int O, int H, int W, void* y_f16, float* img_out,
                                       r3dp_stream_t stream) {
    return layer_torgb_impl(x_f16, wp_f16, bias, wrgb, brgb, img_prev, N, Nw, I, O, H, W, y_f16, img_out, 1, stream);
}

// bilinear up-resize of a CHANNELS-LAST fp32 image [N,h,w,C] (e.g. the renderer's [N,M,32] output viewed as an image) to
// NHWC fp16 [N,size,size,Cpad]: one thread = one output pixel x 8 channels.  idx < N * size * size * Cp / 8.
__device__ __forceinline__ void resize_nhwc_to_f16_item(long long idx, const float* __restrict__ x, int C, int h, int w, int size, int Cp, int split,
                                                        __half* __restrict__ y, float* __restrict__ rgb_out) {
    const int cv = Cp / 8;
    const int c8 = (int)(idx % cv); const int ox = (int)((idx / cv) % size); const int oy = (int)((idx / ((long long)cv * size)) % size);
    const int n = (int)(idx / ((long long)cv * size * size));
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (c8 * 8 < C) {
        int y0, y1, x0, x1;
        float ty, tx;
        bilinear_coord(oy, h, size, y0, y1, ty);
        bilinear_coord(ox, w, size, x0, x1, tx);
        const float* b = x + (size_t)n * h * w * C + c8 * 8;
        const float4* p00 = reinterpret_cast<const float4*>(b + ((size_t)y0 * w + x0) * C);
        const float4* p10 = reinterpret_cast<const float4*>(b + ((size_t)y1 * w + x0) * C);
        const float4* p01 = reinterpret_cast<const float4*>(b + ((size_t)y0 * w + x1) * C);
        const float4* p11 = reinterpret_cast<const float4*>(b + ((size_t)y1 * w + x1) * C);
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            const float4 a00 = __ldg(p00 + q), a10 = __ldg(p10 + q), a01 = __ldg(p01 + q), a11 = __ldg(p11 + q);
            const float e00[4] = {a00.x, a00.y, a00.z, a00.w}, e10[4] = {a10.x, a10.y, a10.z, a10.w};
            const float e01[4] = {a01.x, a01.y, a01.z, a01.w}, e11[4] = {a11.x, a11.y, a11.z, a11.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) v[q * 4 + j] = bilinear_mix(e00[j], e10[j], e01[j], e11[j], ty, tx);
        }
    }
    if (rgb_out != nullptr && c8 == 0) {                       // channels 0..2 = the raw RGB image the SR takes beside the features (secc_img2plane.py:126), fp32 NCHW
#pragma unroll
        for (int c = 0; c < 3; ++c) rgb_out[(((size_t)n * 3 + c) * size + oy) * size + ox] = v[c];
    }
    uint4 pk; __half2* ph = reinterpret_cast<__half2*>(&pk);
#pragma unroll
    for (int j = 0; j < 4; ++j) ph[j] = __floats2half2_rn(v[2 * j], v[2 * j + 1]);
    if (!split) { *reinterpret_cast<uint4*>(y + idx * 8) = pk; return; }
    uint4 pl; __half2* pq = reinterpret_cast<__half2*>(&pl);
#pragma unroll
    for (int j = 0; j < 4; ++j) { const float2 hf = __half22float2(ph[j]); pq[j] = __floats2half2_rn(v[2 * j] - hf.x, v[2 * j + 1] - hf.y); }
    const size_t pix = (size_t)(idx / cv) * (size_t)(2 * Cp);
    *reinterpret_cast<uint4*>(y + pix + c8 * 8) = pk;
    *reinterpret_cast<uint4*>(y + pix + Cp + c8 * 8) = pl;
}

__global__ void resize_nhwc_to_f16_kernel(const float* __restrict__ x, int N, int C, int h, int w, int size, int Cp, int split, __half* __restrict__ y,
                                          float* __restrict__ rgb_out) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * size * size * (Cp / 8)) return;
    resize_nhwc_to_f16_item(idx, x, C, h, w, size, Cp, split, y, rgb_out);
}

// The torso head's inputs from the renderer's output in one launch (sr_with_ref.py:70-78).  Threads [0, n_feat) write x0 and rgb0 exactly as
// resize_nhwc_to_f16_kernel does; thread n_feat + p writes pixel p of rgb_256 = resize(rgb0, 256) and of w_256 = resize(wsum as [N,1,h,w], 256).
// rgb0 is written by other threads of the same launch, so its four source values are recomputed from x with the same helpers: same bits.
constexpr int kWarpRes = 256;
__global__ void warp_input_kernel(const float* __restrict__ x, const float* __restrict__ wsum, int N, int C, int h, int w, int size, int Cp, int split,
                                  __half* __restrict__ y, float* __restrict__ rgb0, float* __restrict__ rgb_256, float* __restrict__ w_256) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long n_feat = (long long)N * size * size * (Cp / 8);
    if (idx < n_feat) { resize_nhwc_to_f16_item(idx, x, C, h, w, size, Cp, split, y, rgb0); return; }
    const long long p = idx - n_feat;
    if (p >= (long long)N * kWarpRes * kWarpRes) return;
    const int ox = (int)(p % kWarpRes), oy = (int)((p / kWarpRes) % kWarpRes), n = (int)(p / ((long long)kWarpRes * kWarpRes));
    int y0, y1, x0, x1;
    float ty, tx;
    bilinear_coord(oy, size, kWarpRes, y0, y1, ty);
    bilinear_coord(ox, size, kWarpRes, x0, x1, tx);
    const int ry[2] = {y0, y1}, rx[2] = {x0, x1};
    float a[3][2][2];                                          // rgb0[c][ry[i]][rx[j]]
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            int sy0, sy1, sx0, sx1;
            float sty, stx;
            bilinear_coord(ry[i], h, size, sy0, sy1, sty);
            bilinear_coord(rx[j], w, size, sx0, sx1, stx);
            const float* b = x + (size_t)n * h * w * C;
#pragma unroll
            for (int c = 0; c < 3; ++c)
                a[c][i][j] = bilinear_mix(__ldg(b + ((size_t)sy0 * w + sx0) * C + c), __ldg(b + ((size_t)sy1 * w + sx0) * C + c),
                                          __ldg(b + ((size_t)sy0 * w + sx1) * C + c), __ldg(b + ((size_t)sy1 * w + sx1) * C + c), sty, stx);
        }
#pragma unroll
    for (int c = 0; c < 3; ++c)
        rgb_256[(((size_t)n * 3 + c) * kWarpRes + oy) * kWarpRes + ox] = bilinear_mix(a[c][0][0], a[c][1][0], a[c][0][1], a[c][1][1], ty, tx);
    bilinear_coord(oy, h, kWarpRes, y0, y1, ty);
    bilinear_coord(ox, w, kWarpRes, x0, x1, tx);
    const float* q = wsum + (size_t)n * h * w;
    w_256[((size_t)n * kWarpRes + oy) * kWarpRes + ox] = bilinear_mix(__ldg(q + y0 * w + x0), __ldg(q + y1 * w + x0), __ldg(q + y0 * w + x1),
                                                                      __ldg(q + y1 * w + x1), ty, tx);
}

static int input_nhwc_impl(const float* x_nhwc, int N, int C, int h, int w, int size, void* y_f16, float* rgb_out, int split, r3dp_stream_t stream) {
    R3DP_REQUIRE(x_nhwc && y_f16, "sr_tc_input_nhwc: null pointer");
    R3DP_REQUIRE(N > 0 && C > 0 && C % 8 == 0 && h > 0 && w > 0 && size >= h && size >= w, "sr_tc_input_nhwc: bad shape (C %% 8 == 0, up-scaling only)");
    const int Cp = (C + 63) / 64 * 64;
    const long long total = (long long)N * size * size * (Cp / 8);
    resize_nhwc_to_f16_kernel<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(x_nhwc, N, C, h, w, size, Cp, split, reinterpret_cast<__half*>(y_f16), rgb_out);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}
extern "C" int r3dp_sr_tc_input_nhwc(const float* x_nhwc, int N, int C, int h, int w, int size, void* y_f16, r3dp_stream_t stream) { return input_nhwc_impl(x_nhwc, N, C, h, w, size, y_f16, nullptr, 0, stream); }
extern "C" int r3dp_sr_tcx_input_nhwc(const float* x_nhwc, int N, int C, int h, int w, int size, void* y_f16, r3dp_stream_t stream) { return input_nhwc_impl(x_nhwc, N, C, h, w, size, y_f16, nullptr, 1, stream); }
// the same, plus rgb_out [N,3,size,size] fp32 = the bilinear resize of channels 0..2 (the raw RGB image of the render head, secc_img2plane.py:126)
extern "C" int r3dp_sr_tc_input_nhwc_rgb(const float* x_nhwc, int N, int C, int h, int w, int size, void* y_f16, float* rgb_out, int split, r3dp_stream_t stream) {
    R3DP_REQUIRE(rgb_out != nullptr && C >= 3, "sr_tc_input_nhwc_rgb: needs rgb_out and at least 3 channels");
    return input_nhwc_impl(x_nhwc, N, C, h, w, size, y_f16, rgb_out, split != 0, stream);
}
extern "C" int r3dp_sr_warp_input(const float* x_nhwc, const float* wsum, int N, int C, int h, int w, int size, void* y_f16, float* rgb0,
                                  float* rgb_256, float* w_256, int split, r3dp_stream_t stream) {
    R3DP_REQUIRE(x_nhwc && wsum && y_f16 && rgb0 && rgb_256 && w_256, "sr_warp_input: null pointer");
    R3DP_REQUIRE(N > 0 && C >= 3 && C % 8 == 0 && h > 0 && w > 0 && size >= h && size >= w && size <= kWarpRes,
                 "sr_warp_input: bad shape (C >= 3, C %% 8 == 0, h, w <= size <= %d)", kWarpRes);
    const int Cp = (C + 63) / 64 * 64;
    const long long total = (long long)N * size * size * (Cp / 8) + (long long)N * kWarpRes * kWarpRes;
    warp_input_kernel<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(x_nhwc, wsum, N, C, h, w, size, Cp, split != 0,
                                                                                     reinterpret_cast<__half*>(y_f16), rgb0, rgb_256, w_256);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

// ---- composed up-convolution for small Cin -------------------------------------------------------------------------------
// FIR(conv_transpose(x, w)) == four 3x3 correlations on the low-resolution input, one per output parity (p,q), with weights
//   G[p][q][dy][dx] = sum_{ky,kx} A[p][dy][ky] * A[q][dx][kx] * w[ky][kx],   A[p][dy][ky] = sum_u g[u] * [p + u - 1 - ky == 2 dy],
// g = [1,3,3,1]/4 (FIR * gain 4), dy,dx in {-1,0,1}  (derivation in DESIGN.md).  This costs 4x the MACs of the two-step form but
// needs no (2H+1)x(2W+1) intermediate, no FIR pass and no edge column: a win when Cin is small (block0.conv0: 32 -> 256).
// wf fp32 [Nw][O][I][3][3] -> packed fp16 [Nw][36][O][Ip], tap index = (p*2+q)*9 + (dy+1)*3 + (dx+1).
__global__ void compose_up_weights_kernel(const float* __restrict__ wf, int Nw, int O, int I, int Ip, int split, __half* __restrict__ out) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)Nw * 36 * O * Ip;
    if (idx >= total) return;
    const int i = (int)(idx % Ip); const int o = (int)((idx / Ip) % O); const int t = (int)((idx / ((long long)Ip * O)) % 36);
    const int nw = (int)(idx / ((long long)Ip * O * 36));
    float acc = 0.f;
    if (i < I) {
        const int ph = t / 9, tap = t % 9, p = ph >> 1, q = ph & 1, dy = tap / 3 - 1, dx = tap % 3 - 1;
        const float g[4] = {0.25f, 0.75f, 0.75f, 0.25f};
        const float* w = wf + (((size_t)nw * O + o) * I + i) * 9;
        for (int ky = 0; ky < 3; ++ky) {
            const int u = 2 * dy + 1 + ky - p;                      // p + u - 1 - ky == 2 dy
            if (u < 0 || u > 3) continue;
            for (int kx = 0; kx < 3; ++kx) {
                const int v = 2 * dx + 1 + kx - q;
                if (v < 0 || v > 3) continue;
                acc = fmaf(g[u] * g[v], w[ky * 3 + kx], acc);
            }
        }
    }
    if (!split) { out[idx] = __float2half_rn(acc); return; }
    __half hi, lo;
    split_half(acc * kSplitWeightScale, hi, lo);
    const size_t row = (idx / Ip) * (size_t)(2 * Ip);
    out[row + i] = hi; out[row + Ip + i] = lo;
}

static int pack_up_composed_impl(const float* wf, int Nw, int O, int I, void* packed_f16, int split, r3dp_stream_t stream) {
    R3DP_REQUIRE(wf && packed_f16, "sr_tc_pack_weights_up_composed: null pointer");
    R3DP_REQUIRE(Nw > 0 && O > 0 && I > 0, "sr_tc_pack_weights_up_composed: bad shape");
    const int Ip = (I + 63) / 64 * 64;
    const long long total = (long long)Nw * 36 * O * Ip;
    compose_up_weights_kernel<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(wf, Nw, O, I, Ip, split, reinterpret_cast<__half*>(packed_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}
extern "C" int r3dp_sr_tc_pack_weights_up_composed(const float* wf, int Nw, int O, int I, void* packed_f16, r3dp_stream_t stream) { return pack_up_composed_impl(wf, Nw, O, I, packed_f16, 0, stream); }
extern "C" int r3dp_sr_tcx_pack_weights_up_composed(const float* wf, int Nw, int O, int I, void* packed_f16, r3dp_stream_t stream) { return pack_up_composed_impl(wf, Nw, O, I, packed_f16, 1, stream); }

// SynthesisLayer with up == 2 through the composed weights: x [N][H][W][Ip] fp16 -> y [N][2H][2W][O] fp16 (bias + lrelu fused).
static int layer_up_composed_impl(const void* x_f16, const void* wpc_f16, const float* bias, int N, int Nw, int I, int O, int H,
                                  int W, void* y_f16, int split, r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && wpc_f16 && bias && y_f16, "sr_tc_layer_up_composed: null pointer");
    R3DP_REQUIRE(N > 0 && (Nw == N || Nw == 1) && W % BM == 0 && O % BN == 0 && O <= 256, "sr_tc_layer_up_composed: bad shape");
    ConvArgs a = {};
    a.n_phases = 4;
    for (int p = 0; p < 4; ++p) a.ph[p] = {taps_3x3(9 * p), H, p >> 1, p & 1};
    set_output(a, kStoreAct, y_f16, 2 * H, 2 * W, O, 2);
    a.bias = bias; a.act_slope = kLreluSlope; a.act_gain = kLreluGain; a.split = split;
    return run_conv(x_f16, N, H, W, I, wpc_f16, Nw, 36, O, a, as_stream(stream));
}
extern "C" int r3dp_sr_tc_layer_up_composed(const void* x_f16, const void* wpc_f16, const float* bias, int N, int Nw, int I, int O, int H,
                                            int W, void* y_f16, r3dp_stream_t stream) {
    return layer_up_composed_impl(x_f16, wpc_f16, bias, N, Nw, I, O, H, W, y_f16, 0, stream);
}
extern "C" int r3dp_sr_tcx_layer_up_composed(const void* x_f16, const void* wpc_f16, const float* bias, int N, int Nw, int I, int O, int H,
                                             int W, void* y_f16, r3dp_stream_t stream) {
    return layer_up_composed_impl(x_f16, wpc_f16, bias, N, Nw, I, O, H, W, y_f16, 1, stream);
}

// ---- building blocks of the torso head (modules/real3d/super_resolution/sr_with_ref.py:16-162) --------------------------------
// Plain nn.Conv2d (k = 1 or 3, stride 1, "same" padding) [+ activation] on the tensor-core path: x [N][H][W][Ip] fp16, weights packed by
// r3dp_sr_tc_pack_weights from the [1][O][I][k][k] fp32 tensor (k = 1: the value sits in tap 4), y [N][H][W][O] fp16.
// act: 0 = linear, 1 = lrelu(0.2)*sqrt2 (bias_act), 2 = nn.LeakyReLU() (slope 0.01).
static int conv_res_impl(const void* x_f16, const void* wp_f16, const float* bias, int N, int Nw, int I, int O, int H, int W, int ksize,
                         int act, const void* residual_f16, void* y_f16, int split, r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && wp_f16 && bias && y_f16, "sr_tc_conv: null pointer");
    R3DP_REQUIRE(N > 0 && (Nw == N || Nw == 1) && W % BM == 0 && O % BN == 0 && O <= 256 && (ksize == 1 || ksize == 3) && act >= 0 && act <= 3,
                 "sr_tc_conv: bad shape / options");
    const float slope = act == 0 ? 1.0f : (act == 1 ? kLreluSlope : (act == 2 ? 0.01f : 0.0f));       // max(v, v*slope): slope 0 = ReLU
    return conv_plain_launch(x_f16, wp_f16, bias, N, Nw, I, O, H, W, ksize, slope, act == 1 ? kLreluGain : 1.0f, residual_f16, y_f16, split, stream);
}
extern "C" int r3dp_sr_tc_conv_res(const void* x_f16, const void* wp_f16, const float* bias, int N, int Nw, int I, int O, int H, int W, int ksize,
                                   int act, const void* residual_f16, void* y_f16, r3dp_stream_t stream) {
    return conv_res_impl(x_f16, wp_f16, bias, N, Nw, I, O, H, W, ksize, act, residual_f16, y_f16, 0, stream);
}
// the same plain convolution with split fp16 operands ([hi | lo] tensors, see the r3dp_sr_tcx_* family): fp32-grade results
extern "C" int r3dp_sr_tcx_conv(const void* x_f16, const void* wp_f16, const float* bias, int N, int Nw, int I, int O, int H, int W, int ksize,
                                int act, void* y_f16, r3dp_stream_t stream) {
    return conv_res_impl(x_f16, wp_f16, bias, N, Nw, I, O, H, W, ksize, act, nullptr, y_f16, 1, stream);
}
// ... with the residual in the output's [hi | lo] layout, added to the activated fp32 value before the split (ResBlock2d of large_sr)
extern "C" int r3dp_sr_tcx_conv_res(const void* x_f16, const void* wp_f16, const float* bias, int N, int Nw, int I, int O, int H, int W, int ksize,
                                    int act, const void* residual_f16, void* y_f16, r3dp_stream_t stream) {
    return conv_res_impl(x_f16, wp_f16, bias, N, Nw, I, O, H, W, ksize, act, residual_f16, y_f16, 1, stream);
}
extern "C" int r3dp_sr_tc_conv(const void* x_f16, const void* wp_f16, const float* bias, int N, int Nw, int I, int O, int H, int W, int ksize,
                               int act, void* y_f16, r3dp_stream_t stream) {
    return r3dp_sr_tc_conv_res(x_f16, wp_f16, bias, N, Nw, I, O, H, W, ksize, act, nullptr, y_f16, stream);
}

// SynthesisBlockNoUp tail (superresolution.py:159-258): conv3x3 (modulated, up == 1) + bias/lrelu -> y, and img_out = img_prev (SAME resolution)
// + ToRGB(y) + brgb.
static int layer_torgb_noup_impl(const void* x_f16, const void* wp_f16, const float* bias, const float* wrgb, const float* brgb,
                                 const float* img_prev, int N, int Nw, int I, int O, int H, int W, void* y_f16, float* img_out, int split,
                                 r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && wp_f16 && bias && wrgb && brgb && y_f16 && img_out, "sr_tc_layer_torgb_noup: null pointer");
    R3DP_REQUIRE(N > 0 && (Nw == N || Nw == 1) && W % BM == 0 && O % BN == 0 && O <= 256, "sr_tc_layer_torgb_noup: bad shape");
    ConvArgs a = {};
    a.n_phases = 1; a.ph[0] = {taps_3x3(0), H, 0, 0};
    set_output(a, kActRgb, y_f16, H, W, O, 1);
    a.bias = bias; a.act_slope = kLreluSlope; a.act_gain = kLreluGain;
    a.wrgb = wrgb; a.brgb = brgb; a.img_prev = img_prev; a.img_out = img_out; a.img_H = H; a.img_W = W; a.skip_same_res = 1;
    a.split = split;
    return run_conv(x_f16, N, H, W, I, wp_f16, Nw, 9, O, a, as_stream(stream));
}
extern "C" int r3dp_sr_tc_layer_torgb_noup(const void* x_f16, const void* wp_f16, const float* bias, const float* wrgb, const float* brgb,
                                           const float* img_prev, int N, int Nw, int I, int O, int H, int W, void* y_f16, float* img_out,
                                           r3dp_stream_t stream) {
    return layer_torgb_noup_impl(x_f16, wp_f16, bias, wrgb, brgb, img_prev, N, Nw, I, O, H, W, y_f16, img_out, 0, stream);
}
extern "C" int r3dp_sr_tcx_layer_torgb_noup(const void* x_f16, const void* wp_f16, const float* bias, const float* wrgb, const float* brgb,
                                            const float* img_prev, int N, int Nw, int I, int O, int H, int W, void* y_f16, float* img_out,
                                            r3dp_stream_t stream) {
    return layer_torgb_noup_impl(x_f16, wp_f16, bias, wrgb, brgb, img_prev, N, Nw, I, O, H, W, y_f16, img_out, 1, stream);
}

// out[n,y,x,:] = [ xa[n,y,x,0:Ca] * alpha[n,y,x] , xb[n,y,x,0:Cb] * (1 - alpha[n,y,x]) ]   (sr_with_ref.py:111,122: alpha-cat fusion), fp16 NHWC
// SPLIT: xa / xb hold [hi | lo] halves (lo at half their pixel stride); hi + lo is scaled in fp32 and the output is the [hi | lo] layout of the
// (Ca + Cb)-channel result: out [N,H,W, 2 (Ca + Cb)], lo at channel Ca + Cb.
// alpha == NULL: the plain concat [xa, xb, xc] (sr_with_ref.py:159, weight_fuse=False); the 8-channel vectors (both halves when SPLIT) are
// copied unchanged.  The LAST operand (xb, or xc when Cc > 0) may hold one frame shared by the batch (hw_last > 0).
template <bool SPLIT>
__global__ void alpha_cat_kernel(const __half* __restrict__ xa, int Ca, int sa, const __half* __restrict__ xb, int Cb, int sb,
                                 const __half* __restrict__ xc, int Cc, int sc, long long hw_last, const float* __restrict__ alpha, long long npix,
                                 __half* __restrict__ out) {
    const int Ct = Ca + Cb + Cc, cv = Ct / 8;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= npix * cv) return;
    const long long pix = idx / cv; const int c8 = (int)(idx - pix * cv), c = c8 * 8;
    const bool first = c < Ca;
    const long long p_last = hw_last > 0 ? pix % hw_last : pix;             // the last operand holds one frame shared by the batch
    const __half* src; int s;
    if (first) { src = xa + pix * sa + c; s = sa; }
    else if (c < Ca + Cb) { src = xb + (Cc > 0 ? pix : p_last) * sb + (c - Ca); s = sb; }
    else { src = xc + p_last * sc + (c - Ca - Cb); s = sc; }
    const uint4 raw = __ldg(reinterpret_cast<const uint4*>(src));
    __half* dst = out + pix * (SPLIT ? 2 : 1) * Ct + c;
    if (!alpha) {
        *reinterpret_cast<uint4*>(dst) = raw;
        if (SPLIT) *reinterpret_cast<uint4*>(dst + Ct) = __ldg(reinterpret_cast<const uint4*>(src + s / 2));
        return;
    }
    const float al = alpha[pix];
    const float m = first ? al : 1.0f - al;
    const __half2* h = reinterpret_cast<const __half2*>(&raw);
    uint4 pk; __half2* ph = reinterpret_cast<__half2*>(&pk);
    if (!SPLIT) {
#pragma unroll
        for (int j = 0; j < 4; ++j) { const float2 f = __half22float2(h[j]); ph[j] = __floats2half2_rn(f.x * m, f.y * m); }
        *reinterpret_cast<uint4*>(dst) = pk;
        return;
    }
    const uint4 rawl = __ldg(reinterpret_cast<const uint4*>(src + s / 2));
    const __half2* hl = reinterpret_cast<const __half2*>(&rawl);
    uint4 pl; __half2* pq = reinterpret_cast<__half2*>(&pl);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(h[j]), g = __half22float2(hl[j]);
        const float v0 = (f.x + g.x) * m, v1 = (f.y + g.y) * m;
        ph[j] = __floats2half2_rn(v0, v1);
        const float2 hf = __half22float2(ph[j]);
        pq[j] = __floats2half2_rn(v0 - hf.x, v1 - hf.y);
    }
    *reinterpret_cast<uint4*>(dst) = pk;
    *reinterpret_cast<uint4*>(dst + Ct) = pl;
}
// Cc == 0: two operands (alpha-cat); alpha == NULL: unweighted concat.  last_shared: the last operand holds one frame [1,H,W,C].
static int alpha_cat_impl(const void* xa_f16, int Ca, int stride_a, const void* xb_f16, int Cb, int stride_b, const void* xc_f16, int Cc,
                          int stride_c, int last_shared, const float* alpha, int N, int H, int W, void* out_f16, int split, r3dp_stream_t stream) {
    const char* what = alpha ? "sr_alpha_cat" : "sr_cat3";
    R3DP_REQUIRE(xa_f16 && xb_f16 && (xc_f16 || Cc == 0) && out_f16, "%s: null pointer", what);
    R3DP_REQUIRE(!alpha || Cc == 0, "%s: alpha weights two operands", what);
    const int wide = split ? 2 : 1;
    R3DP_REQUIRE(N > 0 && H > 0 && W > 0 && Ca % 8 == 0 && Cb % 8 == 0 && Cc % 8 == 0 && Cc >= 0 && stride_a >= wide * Ca && stride_b >= wide * Cb &&
                 stride_a % (8 * wide) == 0 && stride_b % (8 * wide) == 0 && (Cc == 0 || (stride_c >= wide * Cc && stride_c % (8 * wide) == 0)),
                 "%s: bad shape", what);
    const long long npix = (long long)N * H * W, total = npix * ((Ca + Cb + Cc) / 8);
    auto kern = split ? alpha_cat_kernel<true> : alpha_cat_kernel<false>;
    kern<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<const __half*>(xa_f16), Ca, stride_a,
        reinterpret_cast<const __half*>(xb_f16), Cb, stride_b, reinterpret_cast<const __half*>(xc_f16), Cc, stride_c,
        last_shared ? (long long)H * W : 0ll, alpha, npix, reinterpret_cast<__half*>(out_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}
extern "C" int r3dp_sr_alpha_cat_ex(const void* xa_f16, int Ca, int stride_a, const void* xb_f16, int Cb, int stride_b, int xb_shared,
                                    const float* alpha, int N, int H, int W, void* out_f16, r3dp_stream_t stream) {
    R3DP_REQUIRE(alpha, "sr_alpha_cat: null pointer");
    return alpha_cat_impl(xa_f16, Ca, stride_a, xb_f16, Cb, stride_b, nullptr, 0, 0, xb_shared, alpha, N, H, W, out_f16, 0, stream);
}
extern "C" int r3dp_sr_tcx_alpha_cat_ex(const void* xa_f16, int Ca, int stride_a, const void* xb_f16, int Cb, int stride_b, int xb_shared,
                                        const float* alpha, int N, int H, int W, void* out_f16, r3dp_stream_t stream) {
    R3DP_REQUIRE(alpha, "sr_alpha_cat: null pointer");
    return alpha_cat_impl(xa_f16, Ca, stride_a, xb_f16, Cb, stride_b, nullptr, 0, 0, xb_shared, alpha, N, H, W, out_f16, 1, stream);
}
extern "C" int r3dp_sr_cat3(const void* xa_f16, int Ca, int stride_a, const void* xb_f16, int Cb, int stride_b, const void* xc_f16, int Cc,
                            int stride_c, int xc_shared, int N, int H, int W, void* out_f16, r3dp_stream_t stream) {
    return alpha_cat_impl(xa_f16, Ca, stride_a, xb_f16, Cb, stride_b, xc_f16, Cc, stride_c, xc_shared, nullptr, N, H, W, out_f16, 0, stream);
}
extern "C" int r3dp_sr_tcx_cat3(const void* xa_f16, int Ca, int stride_a, const void* xb_f16, int Cb, int stride_b, const void* xc_f16, int Cc,
                                int stride_c, int xc_shared, int N, int H, int W, void* out_f16, r3dp_stream_t stream) {
    return alpha_cat_impl(xa_f16, Ca, stride_a, xb_f16, Cb, stride_b, xc_f16, Cc, stride_c, xc_shared, nullptr, N, H, W, out_f16, 1, stream);
}
extern "C" int r3dp_sr_alpha_cat(const void* xa_f16, int Ca, int stride_a, const void* xb_f16, int Cb, int stride_b, const float* alpha, int N,
                                 int H, int W, void* out_f16, r3dp_stream_t stream) {
    return r3dp_sr_alpha_cat_ex(xa_f16, Ca, stride_a, xb_f16, Cb, stride_b, 0, alpha, N, H, W, out_f16, stream);
}

// out = a * alpha + b * (1 - alpha), fp32 NCHW [N,C,H,W] with alpha [N,1,H,W]  (sr_with_ref.py:110,132)
__global__ void blend_kernel(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ alpha, int C, long long hw,
                             long long total, float* __restrict__ out) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const long long n = idx / (C * hw), p = idx % hw;
    const float al = alpha[n * hw + p];
    out[idx] = a[idx] * al + b[idx] * (1.0f - al);
}
extern "C" int r3dp_sr_blend(const float* a, const float* b, const float* alpha, int N, int C, int H, int W, float* out, r3dp_stream_t stream) {
    R3DP_REQUIRE(a && b && alpha && out && N > 0 && C > 0 && H > 0 && W > 0, "sr_blend: bad arguments");
    const long long hw = (long long)H * W, total = (long long)N * C * hw;
    blend_kernel<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(a, b, alpha, C, hw, total, out);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

// person_occlusion = clamp(torso_occlusion + (w > threshold ? 1 : w), 0, 1)   (sr_with_ref.py:126-131)
__global__ void person_occlusion_kernel(const float* __restrict__ w, const float* __restrict__ torso, float thr, long long total, float* __restrict__ out) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const float h = w[idx] > thr ? 1.0f : w[idx];
    out[idx] = fminf(fmaxf(torso[idx] + h, 0.f), 1.f);
}
extern "C" int r3dp_sr_person_occlusion(const float* head_alpha, const float* torso_occlusion, float threshold, int N, int H, int W, float* out,
                                        r3dp_stream_t stream) {
    R3DP_REQUIRE(head_alpha && torso_occlusion && out && N > 0 && H > 0 && W > 0, "sr_person_occlusion: bad arguments");
    const long long total = (long long)N * H * W;
    person_occlusion_kernel<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(head_alpha, torso_occlusion, threshold, total, out);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

// F.interpolate(scale 1/2, bilinear, align_corners=False, antialias=True) (sr_with_ref.py:79-82): separable triangle filter of support 2,
// taps [1,3,3,1]/8 in the interior, clipped and renormalised at the borders ([3,3,1]/7, [1,3,3]/7).  x [N*C][2h][2w] -> y [N*C][h][w], fp32.
__global__ void aa_down2_kernel(const float* __restrict__ x, int NC, int h, int w, float* __restrict__ y) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)NC * h * w) return;
    const int ox = (int)(idx % w), oy = (int)((idx / w) % h); const long long nc = idx / ((long long)w * h);
    const int H2 = 2 * h, W2 = 2 * w;
    const float* p = x + nc * H2 * W2;
    const float k4[4] = {0.25f, 0.75f, 0.75f, 0.25f};
    float wy[4], wx[4], sy = 0.f, sx = 0.f;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        const int yy = 2 * oy - 1 + t, xx = 2 * ox - 1 + t;
        wy[t] = (yy >= 0 && yy < H2) ? k4[t] : 0.f; wx[t] = (xx >= 0 && xx < W2) ? k4[t] : 0.f;
        sy += wy[t]; sx += wx[t];
    }
    float acc = 0.f;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        if (wy[u] == 0.f) continue;
        const int yy = 2 * oy - 1 + u;
        float row = 0.f;
#pragma unroll
        for (int v = 0; v < 4; ++v) { if (wx[v] != 0.f) row = fmaf(wx[v] / sx, p[(size_t)yy * W2 + 2 * ox - 1 + v], row); }
        acc = fmaf(wy[u] / sy, row, acc);
    }
    y[idx] = acc;
}
extern "C" int r3dp_sr_resize_aa_down2(const float* x, int N, int C, int h_out, int w_out, float* y, r3dp_stream_t stream) {
    R3DP_REQUIRE(x && y && N > 0 && C > 0 && h_out > 0 && w_out > 0, "sr_resize_aa_down2: bad arguments");
    const long long total = (long long)N * C * h_out * w_out;
    aa_down2_kernel<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(x, N * C, h_out, w_out, y);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

// out[n,y,x,0:C] = xa * alpha + xb * (1 - alpha)  (htbsr_head_weight_fuse_mode v1, sr_with_ref.py:98: plain alpha blend of the head and torso features), fp16 NHWC
// SPLIT: xa / xb hold [hi | lo] halves (lo at half their pixel stride); the blend of hi + lo runs in fp32, out [N,H,W,2C] = [hi | lo]
template <bool SPLIT>
__global__ void alpha_mix_kernel(const __half* __restrict__ xa, int sa, const __half* __restrict__ xb, int sb, const float* __restrict__ alpha, int C,
                                 long long npix, __half* __restrict__ out) {
    const int cv = C / 8;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= npix * cv) return;
    const long long pix = idx / cv; const int c8 = (int)(idx - pix * cv);
    const float al = alpha[pix];
    const uint4 ra = __ldg(reinterpret_cast<const uint4*>(xa + pix * sa + c8 * 8)), rb = __ldg(reinterpret_cast<const uint4*>(xb + pix * sb + c8 * 8));
    const __half2* ha = reinterpret_cast<const __half2*>(&ra); const __half2* hb = reinterpret_cast<const __half2*>(&rb);
    uint4 pk; __half2* ph = reinterpret_cast<__half2*>(&pk);
    if (!SPLIT) {
#pragma unroll
        for (int j = 0; j < 4; ++j) { const float2 a = __half22float2(ha[j]), b = __half22float2(hb[j]); ph[j] = __floats2half2_rn(a.x * al + b.x * (1.0f - al), a.y * al + b.y * (1.0f - al)); }
        *reinterpret_cast<uint4*>(out + idx * 8) = pk;
        return;
    }
    const uint4 rla = __ldg(reinterpret_cast<const uint4*>(xa + pix * sa + sa / 2 + c8 * 8)), rlb = __ldg(reinterpret_cast<const uint4*>(xb + pix * sb + sb / 2 + c8 * 8));
    const __half2* la = reinterpret_cast<const __half2*>(&rla); const __half2* lb = reinterpret_cast<const __half2*>(&rlb);
    uint4 pl; __half2* pq = reinterpret_cast<__half2*>(&pl);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float2 a = __half22float2(ha[j]), b = __half22float2(hb[j]), al2 = __half22float2(la[j]), bl2 = __half22float2(lb[j]);
        const float v0 = (a.x + al2.x) * al + (b.x + bl2.x) * (1.0f - al), v1 = (a.y + al2.y) * al + (b.y + bl2.y) * (1.0f - al);
        ph[j] = __floats2half2_rn(v0, v1);
        const float2 hf = __half22float2(ph[j]);
        pq[j] = __floats2half2_rn(v0 - hf.x, v1 - hf.y);
    }
    __half* dst = out + pix * 2 * C + c8 * 8;
    *reinterpret_cast<uint4*>(dst) = pk;
    *reinterpret_cast<uint4*>(dst + C) = pl;
}
static int alpha_mix_impl(const void* xa_f16, int stride_a, const void* xb_f16, int stride_b, const float* alpha, int C, int N, int H, int W,
                          void* out_f16, int split, r3dp_stream_t stream) {
    const int wide = split ? 2 : 1;
    R3DP_REQUIRE(xa_f16 && xb_f16 && alpha && out_f16 && N > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && stride_a >= wide * C && stride_b >= wide * C &&
                 stride_a % (8 * wide) == 0 && stride_b % (8 * wide) == 0, "sr_alpha_mix: bad arguments");
    const long long npix = (long long)N * H * W, total = npix * (C / 8);
    auto kern = split ? alpha_mix_kernel<true> : alpha_mix_kernel<false>;
    kern<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<const __half*>(xa_f16), stride_a,
        reinterpret_cast<const __half*>(xb_f16), stride_b, alpha, C, npix, reinterpret_cast<__half*>(out_f16));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}
extern "C" int r3dp_sr_alpha_mix(const void* xa_f16, int stride_a, const void* xb_f16, int stride_b, const float* alpha, int C, int N, int H, int W,
                                 void* out_f16, r3dp_stream_t stream) {
    return alpha_mix_impl(xa_f16, stride_a, xb_f16, stride_b, alpha, C, N, H, W, out_f16, 0, stream);
}
extern "C" int r3dp_sr_tcx_alpha_mix(const void* xa_f16, int stride_a, const void* xb_f16, int stride_b, const float* alpha, int C, int N, int H, int W,
                                     void* out_f16, r3dp_stream_t stream) {
    return alpha_mix_impl(xa_f16, stride_a, xb_f16, stride_b, alpha, C, N, H, W, out_f16, 1, stream);
}

// out[n,0,y,x] = min(sigmoid(logit), cap[n,0,y,x]) with logit = channel 0 of an NHWC fp16 tensor (+ its lo half lo_off channels further when lo_off > 0):
// the tail of head_torso_alpha_predictor and the `alpha[alpha > weights] = weights` cap of fuse mode v3 (sr_with_ref.py:130-132)
__global__ void alpha_gate_kernel(const __half* __restrict__ y, int stride, int lo_off, const float* __restrict__ cap, long long npix, float* __restrict__ out) {
    const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= npix) return;
    float v = __half2float(y[pix * stride]);
    if (lo_off > 0) v += __half2float(y[pix * stride + lo_off]);
    const float sg = 1.0f / (1.0f + expf(-v));
    out[pix] = fminf(sg, cap[pix]);
}
extern "C" int r3dp_sr_alpha_gate(const void* logits_f16, int stride, int lo_off, const float* cap, int N, int H, int W, float* out, r3dp_stream_t stream) {
    R3DP_REQUIRE(logits_f16 && cap && out && N > 0 && H > 0 && W > 0 && stride > 0 && lo_off >= 0 && lo_off < stride, "sr_alpha_gate: bad arguments");
    const long long npix = (long long)N * H * W;
    alpha_gate_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<const __half*>(logits_f16), stride, lo_off, cap, npix, out);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

// ---- stage 2 of the torso warper (facev2v_warp/network2.py:248-301, Generator) on conv_tc3 -------------------------------------------
// Launch options only: the kernel is the one above.  W a multiple of 64 (64-wide maps use half of each 128-pixel tile), O = 128 | 256 (the
// 64-cout up.1 is packed with zero filters up to 128), act = max(v, v * slope) (1 linear, 0.2 nn.LeakyReLU(0.2), 0 ReLU), gain 1.
static int tw_conv_impl(const void* x_f16, const void* wp_f16, const float* bias, int N, int I, int O, int H, int W, int ksize, float slope,
                        const void* residual_f16, void* y_f16, int split, r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && wp_f16 && bias && y_f16, "tw_conv: null pointer");
    R3DP_REQUIRE(N > 0 && H > 0 && W % 64 == 0 && W > 0 && (O == 128 || O == 256) && (ksize == 1 || ksize == 3) && slope >= 0.f && slope <= 1.f,
                 "tw_conv: bad shape / options");
    return conv_plain_launch(x_f16, wp_f16, bias, N, 1, I, O, H, W, ksize, slope, 1.0f, residual_f16, y_f16, split, stream);
}
extern "C" int r3dp_tw_conv(const void* x_f16, const void* wp_f16, const float* bias, int N, int I, int O, int H, int W, int ksize, float slope,
                            const void* residual_f16, void* y_f16, int split, r3dp_stream_t stream) {
    return tw_conv_impl(x_f16, wp_f16, bias, N, I, O, H, W, ksize, slope, residual_f16, y_f16, split, stream);
}

// nn.Upsample(scale 2, nearest) + 3x3 conv as four output-parity phases of 2x2 taps on the low-resolution input (16 tap GEMMs per input
// pixel instead of 36).  Weights: 4 phase sets packed as [4][9][O][Ip] (r3dp_sr_tc_pack_weights with Nw = 4), set p*2+q holds the composed
// taps of output parity (p, q) at (dy+1)*3 + (dx+1), dy in {-1, 0} for p = 0 and {0, +1} for p = 1 (the same per axis for q, dx).
static int tw_conv_up_nearest_impl(const void* x_f16, const void* wp_f16, const float* bias, int N, int I, int O, int H, int W, float slope,
                                   void* y_f16, int split, r3dp_stream_t stream) {
    R3DP_REQUIRE(x_f16 && wp_f16 && bias && y_f16, "tw_conv_up_nearest: null pointer");
    R3DP_REQUIRE(N > 0 && H > 0 && W % 64 == 0 && W > 0 && (O == 128 || O == 256) && slope >= 0.f && slope <= 1.f, "tw_conv_up_nearest: bad shape / options");
    ConvArgs a = {};
    a.n_phases = 4;
    for (int p = 0; p < 4; ++p) a.ph[p] = {taps_up_nearest(p >> 1, p & 1), H, p >> 1, p & 1};
    set_output(a, kStoreAct, y_f16, 2 * H, 2 * W, O, 2);
    a.bias = bias; a.act_slope = slope; a.act_gain = 1.0f; a.split = split;
    return run_conv(x_f16, N, H, W, I, wp_f16, 1, 36, O, a, as_stream(stream));
}
extern "C" int r3dp_tw_conv_up_nearest(const void* x_f16, const void* wp_f16, const float* bias, int N, int I, int O, int H, int W, float slope,
                                       void* y_f16, int split, r3dp_stream_t stream) {
    return tw_conv_up_nearest_impl(x_f16, wp_f16, bias, N, I, O, H, W, slope, y_f16, split, stream);
}

// Timing of the tensor-core conv launches: r3dp_sr_tc_prof(1) starts recording a CUDA-event pair around every conv_tc3 launch,
// r3dp_sr_tc_prof(0) stops; r3dp_sr_tc_prof_read synchronises the recorded events and returns their summed duration and count.
extern "C" int r3dp_sr_tc_prof(int enable) { g_prof.on = enable != 0; if (enable) g_prof.used = 0; return 0; }
extern "C" int r3dp_sr_tc_prof_read(float* total_ms, int* launches) {
    float sum = 0.f;
    for (size_t i = 0; i + 1 < g_prof.used; i += 2) {
        R3DP_CUDA(cudaEventSynchronize(g_prof.ev[i + 1]));
        float ms = 0.f;
        R3DP_CUDA(cudaEventElapsedTime(&ms, g_prof.ev[i], g_prof.ev[i + 1]));
        sum += ms;
    }
    if (total_ms) *total_ms = sum;
    if (launches) *launches = (int)(g_prof.used / 2);
    return 0;
}

// debug builds (-DR3DP_TC_DEBUG_TIMING=1): device buffer of 32 x 24 uint64; the i-th conv_tc3 launch after this call adds clock sums to row i: [0,8) MMA warp, [8,16) epilogue warp 2 (columns 0-63), [16,24) epilogue warp 6 (columns 64-127)
extern "C" int r3dp_sr_tc_debug_buffer(void* buf) { g_debug_buf = reinterpret_cast<unsigned long long*>(buf); g_debug_launch = 0; return 0; }
