// Streaming fused renderer for single-pass renders (ImportanceRenderer.forward with depth_resolution_importance == 0,
// renderer.py:118-167): one PERSISTENT, warp-specialised CTA per SM in which the tri-plane gather, the OSG decoder on wgmma and the
// ray march of consecutive sample tiles overlap instead of alternating.
//
// Work item   = a group of G rays of one frame (G rows of one image column when the rays form an image: planes 1 and 2 are indexed by
//               (x,z)/(z,x) only, so these rays walk the same texels), streamed front to back in depth chunks of D = 128/G samples per ray.
// Tile        = the G x D = 128 samples of one chunk = two 64-row wgmma tiles; row = ray_local * D + k_local.
// Roles (16 warps = 4 whole warpgroups, mbarrier hand-offs, every ring is filled and drained in tile order):
//   decode  x4  one warpgroup: layer 1 A1 x W1 (3 partial products x 2 k-steps, M64 N64 K16, twice) -> +bias, softplus -> re-split into the
//               A2 atoms; layer 2 A2 x W2 (3 x 4, M64 N48) -> +bias, scaled sigmoid -> fp32 rows (2-deep ring)
//   march   x4  MipRayMarcher2 (ray_marcher.py:26-57) incrementally: alpha / transmittance once per sample (lane = tile row, segmented product
//               scan), colours with lane = channel; accumulators live in registers across the tiles of an item; only the final [32] features,
//               weight sum and depth leave the SM
//   gather  x8  sample depths (renderer.py:223-226) -> positions -> bilinear tap descriptors (smem) -> all 12 x LDG.128 of a sample in flight ->
//               FMAs -> mean feature as fp16 hi|lo halves straight into the swizzled A1 stage (3-stage ring); depths into a small ring
//               for the marcher; L2 look-ahead prefetch of the next frames' planes
// Decoder arithmetic is the split-fp16 scheme of render_shared.cuh (fp32-grade results).
#include "render_shared.cuh"
#include <stdlib.h>

namespace r3dp {
int g_rs_chunk_log2 = -1;
int g_rs_prefetch = -1;                                           // frames of L2 look-ahead (0 = off); r3dp_set_option("rs_prefetch") / R3DP_RS_PREFETCH
namespace rs {

constexpr int kGatherWarps = 8;
// warps 0-3 decode (the warpgroup that issues the MMAs and holds their accumulators), 4-7 march, 8-15 gather.  512 threads leave 128
// registers per thread, enough for the gather warps to keep all twelve 16-byte loads of a sample in flight
constexpr int kFirstGather = 8;
constexpr int kThreads = (kFirstGather + kGatherWarps) * 32;    // 512
constexpr int NS = 3;                                           // A1 stages
constexpr int NR = 2;                                           // decoded-row buffers
constexpr int ND = 8;                                           // depth ring slots
constexpr int kRowF = 33;                                       // floats per decoded row (odd: conflict-free thread-per-row stores)
constexpr int kSPW = 128 / kGatherWarps;                        // samples per gather warp and tile

constexpr int kOffA2 = NS * 16384;
constexpr int kOffW = kOffA2 + 32768;
constexpr int kOffRows = kOffW + 21504;                         // MlpTcImage (20 928 B) padded
constexpr int kOffDep = kOffRows + NR * 128 * kRowF * 4;
constexpr int kOffDsc = kOffDep + ND * 128 * 4;
constexpr int kDscF = 36;                                       // floats per sample descriptor row (28 used by tri-planes, 27 by tri-grids; 36: the four 8-lane groups of a warp read different banks)
constexpr int kOffRay = kOffDsc + kGatherWarps * kSPW * kDscF * 4;
constexpr int kOffBar = kOffRay + kGatherWarps * 8 * 8 * 4;
constexpr int kSmem = kOffBar + 512 + 1024;                     // + alignment slack

struct Bars {
    uint64_t a1_full[NS], a1_empty[NS];
    uint64_t rows_full[NR], rows_empty[NR];
    uint64_t dep_empty[ND], dep_full[ND];
};
static_assert(sizeof(Bars) <= 512, "barrier block");
using tc::mbar_arrive;

template <int LOG2D>
__device__ __forceinline__ int ray_index(const RenderArgs& a, int grp, int r) {
    constexpr int G = 128 >> LOG2D;
    if (a.tile_cols > 0) {
        const int col = grp % a.tile_cols, band = grp / a.tile_cols;
        return (band * G + r) * a.res + col;
    }
    return grp * G + r;
}

template <int LOG2D, bool GRID>
__global__ void __launch_bounds__(kThreads, 1) render_stream_kernel(const RenderArgs a, int items_per_frame, int total_items) {
    constexpr int D = 1 << LOG2D, G = 128 >> LOG2D;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = tc::align_smem_1024(smem_raw);
    uint8_t* a1 = smem;
    uint8_t* a2 = smem + kOffA2;
    uint8_t* wimg = smem + kOffW;
    float* rows = reinterpret_cast<float*>(smem + kOffRows);
    float* dep = reinterpret_cast<float*>(smem + kOffDep);
    float* dsc_all = reinterpret_cast<float*>(smem + kOffDsc);
    float* ray_all = reinterpret_cast<float*>(smem + kOffRay);
    Bars& B = *reinterpret_cast<Bars*>(smem + kOffBar);
    const float* b1s = reinterpret_cast<const float*>(wimg + 20480);
    const float* b2s = b1s + kHidden;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int NT = (a.S + D - 1) >> LOG2D;                                     // tiles per item
    const int my_items = (int)blockIdx.x < total_items ? (total_items - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    const uint32_t total_tiles = (uint32_t)(my_items * NT);

    if (tid == 0) {
        for (int i = 0; i < NS; ++i) { tc::mbar_init(&B.a1_full[i], kGatherWarps); tc::mbar_init(&B.a1_empty[i], 4); }
        for (int i = 0; i < NR; ++i) { tc::mbar_init(&B.rows_full[i], 4); tc::mbar_init(&B.rows_empty[i], 4); }
        for (int i = 0; i < ND; ++i) { tc::mbar_init(&B.dep_empty[i], 4); tc::mbar_init(&B.dep_full[i], kGatherWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    {   // decoder operand image (pre-swizzled fp16 hi/lo atoms + biases) from the call's workspace
        const uint4* src = reinterpret_cast<const uint4*>(a.image);
        uint4* dst = reinterpret_cast<uint4*>(wimg);
        for (int i = tid; i < (int)(sizeof(MlpTcImage) / 16); i += kThreads)
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(tc::smem_u32(dst + i)), "l"(src + i) : "memory");
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();

    if (warp >= kFirstGather) {
        // ===================================================== gather ===========================================================
        constexpr int RPW = kSPW >> LOG2D;                                      // rays per gather warp
        static_assert(RPW >= 1, "D must not exceed the samples of one gather warp");
        const int gw = warp - kFirstGather, sub = lane >> 3, cq = lane & 7;
        float* dsc = dsc_all + gw * kSPW * kDscF;
        float* rayw = ray_all + gw * 64;
        const float scale = 2.0f / a.box_warp;
        const int rs = a.p0.row_stride, ts = a.p0.texel_stride, ss = a.p0.slice_stride;
        float dmin = __int_as_float(0x7f800000), dmax = __int_as_float(0xff800000);
        uint32_t q = 0;
        int pf_next = 0;
        for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
            const int n = item / items_per_frame, grp = item - n * items_per_frame;
            if (gw == 0 && lane == 0 && a.lookahead > 0) {                        // keep `lookahead` frames of planes streaming into L2 ahead of the gather
                for (; pf_next < a.N && pf_next < n + a.lookahead; ++pf_next) {
                    prefetch_frame_l2(a.p0, a.H, a.W, pf_next, blockIdx.x, gridDim.x); prefetch_frame_l2(a.p1, a.H, a.W, pf_next, blockIdx.x, gridDim.x);
                }
            }
            __syncwarp();
            if (lane < RPW) {
                const int m = ray_index<LOG2D>(a, grp, gw * RPW + lane);
                float* rf = rayw + lane * 8;
                if (m < a.M) {
                    Ray r = fetch_ray(a.ray_o, a.ray_d, a.camera, a.res, n, a.M, m);
                    float2 lim = a.limits[(size_t)n * a.M + m];
                    if (!a.valid[(size_t)n * a.M + m] && a.ws->n_valid > 0) {      // renderer.py:125-126 (far end from ray_START, sic)
                        lim.x = ord2f(a.ws->t0_min); lim.y = ord2f(a.ws->t0_max);
                    }
                    rf[0] = r.ox; rf[1] = r.oy; rf[2] = r.oz; rf[3] = r.dx; rf[4] = r.dy; rf[5] = r.dz; rf[6] = lim.x; rf[7] = lim.y;
                } else {
#pragma unroll
                    for (int e = 0; e < 8; ++e) rf[e] = 0.f;
                }
            }
            __syncwarp();
            const float* base0 = a.p0.base + (size_t)n * a.p0.frame_stride;
            const float* base1 = a.p1.base ? a.p1.base + (size_t)n * a.p1.frame_stride : nullptr;
            // this lane's sample of the descriptor phase (lanes 0..kSPW-1): ray rl of the warp, depth index k0 + j
            const int s_rl = (lane & (kSPW - 1)) >> LOG2D, s_j = lane & (D - 1);
            const int s_m = ray_index<LOG2D>(a, grp, gw * RPW + s_rl);
            const float* up = a.u_coarse + ((size_t)n * a.M + (s_m < a.M ? s_m : 0)) * a.S;
            float u_next = (lane < kSPW && s_m < a.M && s_j < a.S) ? __ldg(up + s_j) : 0.f;
            for (int t = 0; t < NT; ++t, ++q) {
                const int k0 = t << LOG2D, stage = q % NS, dslot = q % ND;
                const float u = u_next;
                {
                    const int kn = k0 + D + s_j;
                    u_next = (t + 1 < NT && lane < kSPW && s_m < a.M && kn < a.S) ? __ldg(up + kn) : 0.f;
                }
                tc::mbar_wait(&B.dep_empty[dslot], ((q / ND) & 1) ^ 1);
                if (lane < kSPW) {
                    const int k = k0 + s_j;
                    float* row = dsc + lane * kDscF;
                    float d = 0.f;
                    if (s_m < a.M && k < a.S) {
                        const float* rf = rayw + s_rl * 8;
                        const float t0 = rf[6], t1 = rf[7];
                        const float step = __fdiv_rn((float)k, (float)(a.S - 1));                  // renderer.py:223-226, math_utils.py:101-118
                        d = __fadd_rn(t0, __fmul_rn(step, __fsub_rn(t1, t0)));
                        d = __fadd_rn(d, __fmul_rn(u, __fdiv_rn(__fsub_rn(t1, t0), (float)(a.S - 1))));
                        dmin = fminf(dmin, d); dmax = fmaxf(dmax, d);
                        const float x = __fadd_rn(rf[0], __fmul_rn(d, rf[3]));
                        const float y = __fadd_rn(rf[1], __fmul_rn(d, rf[4]));
                        const float z = __fadd_rn(rf[2], __fmul_rn(d, rf[5]));
                        if (GRID) sample_desc(a.p0, a.H, a.W, scale * x, scale * y, scale * z, row);
                        else sample_desc_split(a.p0, a.H, a.W, scale * x, scale * y, scale * z, row);
                    } else {
#pragma unroll
                        for (int e = 0; e < 28; ++e) row[e] = 0.f;                                 // offset 0, weights 0: a harmless tap
                    }
                    dep[dslot * 128 + gw * kSPW + lane] = d;
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&B.dep_full[dslot]);                // the depths have their own full barrier: the march warps acquire them directly
                tc::mbar_wait(&B.a1_empty[stage], ((q / NS) & 1) ^ 1);
                uint8_t* a1s = a1 + stage * 16384;
#pragma unroll 1
                for (int it = 0; it < kSPW / 4; ++it) {
                    const int s = it * 4 + sub;
                    const float4* rw = reinterpret_cast<const float4*>(dsc + s * kDscF);
                    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (GRID) {
                        float dscv[28];
#pragma unroll
                        for (int e = 0; e < 7; ++e) { const float4 qv = rw[e]; dscv[4 * e] = qv.x; dscv[4 * e + 1] = qv.y; dscv[4 * e + 2] = qv.z; dscv[4 * e + 3] = qv.w; }
                        gather_desc<true>(base0, dscv, rs, ts, ss, cq, acc);
                        if (base1 != nullptr) gather_desc<true>(base1, dscv, rs, ts, ss, cq, acc);
                    } else {
                        // row = [off0 off1 off2 - | 4 weights x 3 planes]: the offsets first, ALL twelve LDG.128 of the sample issued back to back
                        // (48 registers in flight per lane), the weights fetched from smem under their latency, only then the FMAs.  ncu on the
                        // previous form: ptxas interleaved the loads with their uses in 4 groups = 4 exposed L2 round trips per step.
                        const float4 offs = rw[0];
                        gather12(base0, __float_as_int(offs.x), __float_as_int(offs.y), __float_as_int(offs.z), rs, ts, cq, rw + 1, acc);
                        if (base1 != nullptr) gather12(base1, __float_as_int(offs.x), __float_as_int(offs.y), __float_as_int(offs.z), rs, ts, cq, rw + 1, acc);
                    }
                    // mean over the planes as fp16 hi + lo halves into the swizzled A1 stage: lane cq owns K = [4cq, 4cq+4) of both halves
                    const float third = 1.0f / 3.0f;
                    const float f0 = acc.x * third, f1 = acc.y * third, f2 = acc.z * third, f3 = acc.w * third;
                    const __half2 h01 = __floats2half2_rn(f0, f1), h23 = __floats2half2_rn(f2, f3);
                    const float2 g01 = __half22float2(h01), g23 = __half22float2(h23);
                    const __half2 l01 = __floats2half2_rn(f0 - g01.x, f1 - g01.y), l23 = __floats2half2_rn(f2 - g23.x, f3 - g23.y);
                    const int trow = gw * kSPW + s;
                    uint8_t* rp = a1s + (trow >> 3) * 1024 + (trow & 7) * 128 + (cq & 1) * 8;
                    uint2 hv, lv;
                    hv.x = *reinterpret_cast<const uint32_t*>(&h01); hv.y = *reinterpret_cast<const uint32_t*>(&h23);
                    lv.x = *reinterpret_cast<const uint32_t*>(&l01); lv.y = *reinterpret_cast<const uint32_t*>(&l23);
                    *reinterpret_cast<uint2*>(rp + (((cq >> 1) ^ (trow & 7)) << 4)) = hv;
                    *reinterpret_cast<uint2*>(rp + (((4 + (cq >> 1)) ^ (trow & 7)) << 4)) = lv;
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");       // generic-proxy A1 stores -> visible to the tensor core
                __syncwarp();
                if (lane == 0) mbar_arrive(&B.a1_full[stage]);
            }
        }
        // call-wide min/max of the sample depths (ray_marcher.py:50)
        dmin = warp_min(dmin); dmax = warp_max(dmax);
        if (lane == 0 && dmin <= dmax) { atomicMin(&a.ws->d_min, f2ord(dmin)); atomicMax(&a.ws->d_max, f2ord(dmax)); }
    } else if (warp < 4) {
        // ====================================================== decode ==========================================================
        const uint32_t a2_s = tc::smem_u32(a2), w_s = tc::smem_u32(wimg);
        for (uint32_t q = 0; q < total_tiles; ++q) {
            const uint32_t stage = q % NS;
            tc::mbar_wait(&B.a1_full[stage], (q / NS) & 1u);
            const uint32_t a1_s = tc::smem_u32(a1) + stage * 16384u;
            float h[2][32];                                                    // tile rows [0, 64) and [64, 128)
            tc::wg_fence();
#pragma unroll
            for (int b = 0; b < 2; ++b) {                                      // x_hi w_hi + x_lo w_hi + x_hi w_lo, 2 k-steps each
                uint32_t accum = 0;
#pragma unroll
                for (int term = 0; term < 3; ++term) {
                    const uint32_t ao = term == 1 ? 64u : 0u, bo = term == 2 ? 64u : 0u;
#pragma unroll
                    for (int ks = 0; ks < 2; ++ks) {
                        tc::wgmma_m64n64k16(h[b], tc::gmma_desc_sw128(a1_s + b * 8192 + ao + ks * 32), tc::gmma_desc_sw128(w_s + bo + ks * 32), accum);
                        accum = 1;
                    }
                }
            }
            tc::wg_commit();
            tc::wg_wait<0>();
            tc::wg_fence_acc<32>(h[0]); tc::wg_fence_acc<32>(h[1]);
            __syncwarp();
            if (lane == 0) mbar_arrive(&B.a1_empty[stage]);
            // hidden units: +bias, softplus, re-split into the A2 atoms (row = sample of the tile, K = hidden unit)
#pragma unroll
            for (int b = 0; b < 2; ++b)
#pragma unroll
                for (int i = 0; i < 32; i += 2) {
                    const int trow = 64 * b + tc::acc_row(i), j = tc::acc_col(i);
                    const float2 bb = *reinterpret_cast<const float2*>(b1s + j);
                    const float2 hv = softplus2(pk_add(make_float2(h[b][i], h[b][i + 1]), bb));
                    const __half2 hh = __floats2half2_rn(hv.x, hv.y);
                    const float2 hf = __half22float2(hh);
                    const __half2 ll = __floats2half2_rn(hv.x - hf.x, hv.y - hf.y);
                    *reinterpret_cast<__half2*>(a2 + sw128_off(trow, j)) = hh;
                    *reinterpret_cast<__half2*>(a2 + 16384 + sw128_off(trow, j)) = ll;
                }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            asm volatile("bar.sync 1, 128;" ::: "memory");                      // the whole A2 tile is written
            float o[2][24];
            tc::wg_fence();
#pragma unroll
            for (int b = 0; b < 2; ++b) {                                      // h_hi w_hi + h_lo w_hi + h_hi w_lo, 4 k-steps each
                uint32_t accum = 0;
#pragma unroll
                for (int term = 0; term < 3; ++term) {
                    const uint32_t ao = term == 1 ? 16384u : 0u, bo = term == 2 ? (8192u + 6144u) : 8192u;
#pragma unroll
                    for (int ks = 0; ks < 4; ++ks) {
                        tc::wgmma_m64n48k16(o[b], tc::gmma_desc_sw128(a2_s + b * 8192 + ao + ks * 32), tc::gmma_desc_sw128(w_s + bo + ks * 32), accum);
                        accum = 1;
                    }
                }
            }
            tc::wg_commit();
            tc::wg_wait<0>();
            tc::wg_fence_acc<24>(o[0]); tc::wg_fence_acc<24>(o[1]);
            asm volatile("bar.sync 1, 128;" ::: "memory");                      // every warp's layer 2 has read A2 before the next tile rewrites it
            // outputs: sigma raw, colours through the scaled sigmoid
            const uint32_t rb = q % NR;
            tc::mbar_wait(&B.rows_empty[rb], ((q / NR) & 1u) ^ 1u);
#pragma unroll
            for (int b = 0; b < 2; ++b)
#pragma unroll
                for (int i = 0; i < 24; i += 2) {
                    const int trow = 64 * b + tc::acc_row(i), oc = tc::acc_col(i);
                    float* out = rows + (rb * 128 + trow) * kRowF;
                    const float2 sg = sigmoid_scaled2(pk_add(make_float2(o[b][i], o[b][i + 1]), *reinterpret_cast<const float2*>(b2s + oc)));
                    if (oc == 0) out[0] = o[b][i] + b2s[0];
                    else if (oc < kOut) out[oc] = sg.x;
                    if (oc + 1 < kOut) out[oc + 1] = sg.y;
                }
            __syncwarp();
            if (lane == 0) mbar_arrive(&B.rows_full[rb]);
        }
    } else {
        // ====================================================== march ===========================================================
        // ray_marcher.py:26-57, front to back over the tiles of an item.  Warp mw owns RM = G/4 rays = the 32 tile rows [32 mw, 32 mw + 32).
        //   weights  lane = tile row = (ray i = lane >> LOG2D, sample j = lane & (D-1)): alpha of the interval that ENDS at this sample, transmittance by a
        //            segmented product scan over the ray's D lanes times the value carried from the previous tile - one softplus / exp per sample,
        //            not one per sample and colour channel;
        //   colours  lane = channel: 32 (ray, sample) pairs per tile, each weight broadcast by a shuffle; acc += w * mid-point colour.
        constexpr int RM = G / 4;
        static_assert(RM * D == 32, "one warp marches 32 tile rows");
        const int mw = warp - 4, lj = lane & (D - 1), seg_last = lane | (D - 1);
        uint32_t q = 0;
        for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
            const int n = item / items_per_frame, grp = item - n * items_per_frame;
            float Tc = 1.f, last_s = 0.f, last_d = 0.f, wsum = 0.f, dsum = 0.f;        // per tile-row lane; Tc is uniform over the lanes of a ray
            float acc[RM], pc[RM];                                                    // per channel lane
#pragma unroll
            for (int i = 0; i < RM; ++i) { acc[i] = 0.f; pc[i] = 0.f; }
            for (int t = 0; t < NT; ++t, ++q) {
                const uint32_t rb = q % NR, dslot = q % ND;
                tc::mbar_wait(&B.rows_full[rb], (q / NR) & 1u);
                tc::mbar_wait(&B.dep_full[dslot], (q / ND) & 1u);
                const float* rbuf = rows + (rb * 128 + mw * 32) * kRowF;
                const int k = (t << LOG2D) + lj;
                const float s = rbuf[lane * kRowF], d = dep[dslot * 128 + mw * 32 + lane];
                float ps = __shfl_up_sync(0xffffffffu, s, 1), pd = __shfl_up_sync(0xffffffffu, d, 1);
                const float cs = __shfl_sync(0xffffffffu, last_s, seg_last), cd = __shfl_sync(0xffffffffu, last_d, seg_last);
                if (lj == 0) { ps = cs; pd = cd; }
                float alpha = 0.f, om = 1.f, dmid = 0.f;
                if (k > 0 && k < a.S) {
                    const float smid = softplus2(make_float2((ps + s) * 0.5f - 1.0f, 0.f)).x;    // ray_marcher.py:33
                    alpha = 1.0f - __expf(-(smid * (d - pd)));
                    om = 1.0f - alpha + 1e-10f;
                    dmid = 0.5f * (pd + d);
                }
                float incl = om;                                                      // inclusive product over the ray's lanes 0..j
#pragma unroll
                for (int o = 1; o < D; o <<= 1) { const float v = __shfl_up_sync(0xffffffffu, incl, o); if (lj >= o) incl *= v; }
                float excl = __shfl_up_sync(0xffffffffu, incl, 1);
                if (lj == 0) excl = 1.f;
                const float w = alpha * (Tc * excl);                                  // ray_marcher.py:41-42
                Tc *= __shfl_sync(0xffffffffu, incl, seg_last);
                wsum += w;
                dsum = fmaf(w, dmid, dsum);
                last_s = s; last_d = d;
#pragma unroll
                for (int p = 0; p < 32; ++p) {
                    const float wp = __shfl_sync(0xffffffffu, w, p);
                    const float c = rbuf[p * kRowF + 1 + lane];
                    acc[p >> LOG2D] = fmaf(wp, 0.5f * (pc[p >> LOG2D] + c), acc[p >> LOG2D]);
                    pc[p >> LOG2D] = c;
                }
                __syncwarp();
                if (lane == 0) { mbar_arrive(&B.rows_empty[rb]); mbar_arrive(&B.dep_empty[dslot]); }
            }
#pragma unroll
            for (int o = 1; o < D; o <<= 1) { wsum += __shfl_xor_sync(0xffffffffu, wsum, o); dsum += __shfl_xor_sync(0xffffffffu, dsum, o); }
#pragma unroll
            for (int i = 0; i < RM; ++i) {
                const int m = ray_index<LOG2D>(a, grp, mw * RM + i);
                const float wi = __shfl_sync(0xffffffffu, wsum, i << LOG2D), di = __shfl_sync(0xffffffffu, dsum, i << LOG2D);
                if (m < a.M) {
                    const size_t o = (size_t)n * a.M + m;
                    float v = acc[i];
                    if (a.white_back) v = v + 1.0f - wi;
                    a.rgb[o * (kOut - 1) + lane] = v * 2.0f - 1.0f;
                    if (lane == 0) { a.wsum[o] = wi; a.depth[o] = di / wi; }           // 0/0 -> NaN, fixed by depth_clamp_kernel
                }
            }
        }
    }
}

static int chunk_log2() {                          // R3DP_RS_D = 4 | 8 | 16: depth samples per ray and tile (rays per item = 128 / D); A/B knob
    if (g_rs_chunk_log2 < 0) { const char* e = getenv("R3DP_RS_D"); const int d = e ? atoi(e) : 8; g_rs_chunk_log2 = d == 4 ? 2 : (d == 16 ? 4 : 3); }
    return g_rs_chunk_log2;
}

template <int LOG2D, bool GRID>
static int launch(RenderArgs a, cudaStream_t st) {
    constexpr int G = 128 >> LOG2D;
    const bool image = a.res > 0 && a.res * a.res == a.M && (a.res % G) == 0;
    a.tile_cols = image ? a.res : 0;
    const int items_per_frame = (a.M + G - 1) / G;
    const int total = a.N * items_per_frame;
    R3DP_CUDA(cudaFuncSetAttribute(render_stream_kernel<LOG2D, GRID>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
    const int grid = total < sm_count() ? total : sm_count();
    render_stream_kernel<LOG2D, GRID><<<grid, kThreads, kSmem, st>>>(a, items_per_frame, total);
    R3DP_LAUNCH_CHECK();
    return 0;
}

}  // namespace rs

bool render_stream_fits(const RenderArgs& a) {
    if (a.S_imp != 0 || a.S < 2) return false;
    if (a.p1.base && (a.p1.plane_stride != a.p0.plane_stride || a.p1.row_stride != a.p0.row_stride || a.p1.texel_stride != a.p0.texel_stride ||
                      a.p1.depth != a.p0.depth || a.p1.slice_stride != a.p0.slice_stride)) return false;
    return true;
}

int render_lookahead() {                           // R3DP_RS_PREFETCH = frames of planes streamed into L2 ahead of the gather (default 2, 0 = off)
    if (g_rs_prefetch < 0) { const char* e = getenv("R3DP_RS_PREFETCH"); g_rs_prefetch = e ? atoi(e) : 2; if (g_rs_prefetch < 0) g_rs_prefetch = 0; }
    return g_rs_prefetch;
}

int launch_render_stream(const RenderArgs& a, cudaStream_t st) {
    if (a.p0.depth > 1) return rs::launch<3, true>(a, st);                      // tri-grids: D = 8 chunks only
    switch (rs::chunk_log2()) {
        case 2: return rs::launch<2, false>(a, st);
        case 4: return rs::launch<4, false>(a, st);
        default: return rs::launch<3, false>(a, st);
    }
}

}  // namespace r3dp
