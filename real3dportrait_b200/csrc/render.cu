// Fused volumetric renderer: ImportanceRenderer.forward with 'auto' limits (renderer.py:118-167) as three launches after the set-up launch
//   1. ray_limits_kernel   rays (given or generated from cameras) -> (t0,t1,valid) + call-wide min/max of valid t0
//   2. render_stream_kernel (single-pass renders, render_stream.cu) or render_kernel (two-pass importance renders):
//                          depths -> tri-plane gather -> OSG decoder -> ray march [-> importance pass -> merge -> march]
//   3. depth_clamp_kernel  NaN->inf, clamp depth to the call-wide [min,max] sample depth (ray_marcher.py:49-50)
// plus gen_rays (RaySampler.forward) and a stand-alone ray marcher.
#include "render_shared.cuh"

namespace r3dp {


struct RenderWs;
__device__ __forceinline__ void init_ws(RenderWs* ws);
// decoder operand image for the tensor cores (+ the call's workspace header, so that a render needs one set-up launch instead of two)
__global__ void mlp_to_tc_kernel(const r3dp_mlp_t m, MlpTcImage* dst, RenderWs* ws) {
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nt = gridDim.x * blockDim.x;
    if (tid == 0 && ws != nullptr) init_ws(ws);
    const float g1 = 0.17677669529663687f, g2 = 0.125f;        // 1/sqrt(32), 1/sqrt(64)  (networks_stylegan2.py:113)
    for (int i = tid; i < kHidden * kC; i += nt) {
        const int j = i / kC, c = i - j * kC;
        const float w = m.w1[i] * g1;
        const __half hi = __float2half_rn(w), lo = __float2half_rn(w - __half2float(hi));
        *reinterpret_cast<__half*>(dst->w1 + sw128_off(j, c)) = hi;
        *reinterpret_cast<__half*>(dst->w1 + sw128_off(j, kC + c)) = lo;
    }
    for (int i = tid; i < 48 * kHidden; i += nt) {
        const int o = i / kHidden, j = i - o * kHidden;
        const float w = o < kOut ? m.w2[o * kHidden + j] * g2 : 0.f;
        const __half hi = __float2half_rn(w), lo = __float2half_rn(w - __half2float(hi));
        *reinterpret_cast<__half*>(dst->w2hi + sw128_off(o, j)) = hi;
        *reinterpret_cast<__half*>(dst->w2lo + sw128_off(o, j)) = lo;
    }
    for (int i = tid; i < kHidden; i += nt) dst->b1[i] = m.b1[i];
    for (int i = tid; i < 48; i += nt) dst->b2[i] = i < kOut ? m.b2[i] : 0.f;
}
constexpr int kTcThreads = 256;                          // 2 warpgroups: warpgroup g takes rows [64 g, 64 g + 64) of every 128-sample tile
constexpr int kTcA2Bytes = 32768;                        // the two 16 KB A1 tiles of a pass; after layer 1, the two A2 atoms
__device__ __forceinline__ void init_ws(RenderWs* ws) {
    ws->t0_min = 0xffffffffu; ws->t0_max = 0u; ws->d_min = 0xffffffffu; ws->d_max = 0u; ws->n_valid = 0u;
}
__global__ void init_ws_kernel(RenderWs* ws) { init_ws(ws); }

// ---------------------------------------------------------------------------------------------------------------
__global__ void gen_rays_kernel(const float* __restrict__ c2w, const float* __restrict__ K, int N, int res,
                                float* __restrict__ ray_o, float* __restrict__ ray_d) {
    const int M = res * res;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= N * M) return;
    const int n = idx / M, m = idx - n * M;
    Ray r = make_ray(c2w + n * 16, K + n * 9, res, m);
    float* o = ray_o + (size_t)idx * 3; float* d = ray_d + (size_t)idx * 3;
    o[0] = r.ox; o[1] = r.oy; o[2] = r.oz; d[0] = r.dx; d[1] = r.dy; d[2] = r.dz;
}

__global__ void ray_limits_kernel(const float* __restrict__ ray_o, const float* __restrict__ ray_d,
                                  const float* __restrict__ camera, int res, int N, int M, float box,
                                  float2* __restrict__ limits, uint8_t* __restrict__ valid_out, RenderWs* ws) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    float t0 = 0.f, t1 = 0.f; bool valid = false;
    if (idx < N * M) {
        const int n = idx / M, m = idx - n * M;
        Ray r = fetch_ray(ray_o, ray_d, camera, res, n, M, m);
        ray_box(r, box, t0, t1);
        valid = t1 > t0;                                 // renderer.py:122
        limits[idx] = make_float2(t0, t1);
        valid_out[idx] = valid ? 1 : 0;
    }
    // call-wide min / max of the valid ray starts (renderer.py:124-126)
    const unsigned mask = __ballot_sync(0xffffffffu, valid);
    if (mask) {
        float lo = warp_min(valid ? t0 : __int_as_float(0x7f800000));
        float hi = warp_max(valid ? t0 : __int_as_float(0xff800000));
        if ((threadIdx.x & 31) == 0) {
            atomicMin(&ws->t0_min, f2ord(lo));
            atomicMax(&ws->t0_max, f2ord(hi));
            atomicAdd(&ws->n_valid, (unsigned)__popc(mask));
        }
    }
}

__global__ void depth_clamp_kernel(float* __restrict__ depth, int n, const RenderWs* __restrict__ ws) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n) return;
    float d = depth[idx];
    if (d != d) d = __int_as_float(0x7f800000);         // nan_to_num(nan=inf); +-inf are then clamped below
    const float lo = ord2f(ws->d_min), hi = ord2f(ws->d_max);
    depth[idx] = fminf(fmaxf(d, lo), hi);
}

// ---------------------------------------------------------------------------------------------------------------
constexpr int kRenderThreads = 192;

// R rays per CTA.  If the rays form a res x res image we take them as a COLUMN strip (R rows, 1 col): planes 1 and 2
// are indexed by (x,z)/(z,x) only, so rays that differ only in image row share their footprints in L1.
template <int R>
__device__ __forceinline__ int ray_of(const RenderArgs& a, int tile, int r) {
    if (a.tile_cols > 0) {
        const int col = tile % a.tile_cols, band = tile / a.tile_cols;
        return (band * R + r) * a.res + col;
    }
    return tile * R + r;
}

// Two-pass (importance) renders; single-pass renders run the streaming kernel of render_stream.cu.
// TC = false: decoder weights staged in smem, CUDA-core decoder, two samples per thread (passes that do not fit the tensor-core tiles)
// TC = decoder on wgmma (passes of R*max(S, S_imp) <= 256 samples; 256 threads, 2 CTAs/SM); see the MlpTcImage comment
constexpr int kPfCtas = 32;                            // CTAs of a frame that issue its L2 prefetches
template <int R, bool TC>
__global__ void __launch_bounds__(TC ? kTcThreads : kRenderThreads, 2) render_kernel(const RenderArgs a) {
    extern __shared__ __align__(16) float smem[];
    constexpr int kRenderThreads = TC ? kTcThreads : r3dp::kRenderThreads;     // shadows the namespace constant inside this kernel
    const int ST = a.S + a.S_imp;                         // samples per ray after the importance pass
    MlpSmem& mlp = *reinterpret_cast<MlpSmem*>(smem);
    float* rows = smem + sizeof(MlpSmem) / 4;               // [R*ST][kRow]   features -> (sigma, colours)
    float* dep = rows + R * ST * kRow;                     // [R*ST]          sample depths
    float* wts = dep + R * ST;                             // [R*ST]          coarse interval weights
    float* cdf = wts + R * ST;                             // [R*ST]          importance cdf
    float* rayf = cdf + R * ST;                            // [R][8]          ox oy oz dx dy dz t0 t1
    int* ord = reinterpret_cast<int*>(rayf + R * 8);       // [R*ST]          depth order of the merged samples
    // TC layout (1024-aligned): [A1 tiles (2) = A2 atoms] [W image + biases] rows dep wts cdf rayf ord
    // The decoded rows of pass 1 must survive pass 2, so they get their own region (and hold the tap descriptors of the samples in flight,
    // like the CUDA-core decoder); A2 reuses the (by then consumed) A1 tiles.
    uint8_t* a1 = nullptr; uint8_t* a2 = nullptr; uint8_t* wimg = nullptr; float* b1s = nullptr; float* b2s = nullptr;
    if (TC) {
        a1 = tc::align_smem_1024(reinterpret_cast<uint8_t*>(smem));
        a2 = a1;
        wimg = a1 + kTcA2Bytes;
        b1s = reinterpret_cast<float*>(wimg + 20480); b2s = b1s + kHidden;
        rows = b2s + 48;
        dep = rows + R * ST * kRow; wts = dep + R * ST; cdf = wts + R * ST;
        rayf = cdf + R * ST;
        ord = reinterpret_cast<int*>(rayf + R * 8);
    }

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int kWarps = kRenderThreads / 32;
    const int n = blockIdx.y, tile = blockIdx.x;

    if (a.lookahead > 0 && tid == 0 && tile < kPfCtas) {    // the first CTAs of frame n ask the TMA unit for frame n + lookahead (frame 0's also for the first frames)
        if (n == 0)
            for (int f = 0; f < a.lookahead && f < a.N; ++f) { prefetch_frame_l2(a.p0, a.H, a.W, f, tile, kPfCtas); prefetch_frame_l2(a.p1, a.H, a.W, f, tile, kPfCtas); }
        if (n + a.lookahead < a.N) { prefetch_frame_l2(a.p0, a.H, a.W, n + a.lookahead, tile, kPfCtas); prefetch_frame_l2(a.p1, a.H, a.W, n + a.lookahead, tile, kPfCtas); }
    }
    if (!TC) load_mlp_smem(mlp, a.mlp, tid, kRenderThreads);
    if (TC) {
        // decoder weight image (pre-swizzled fp16 hi/lo atoms + biases): 20 928 B from L2
        const uint4* src = reinterpret_cast<const uint4*>(a.image);
        uint4* dst = reinterpret_cast<uint4*>(wimg);
        for (int i = tid; i < (int)(sizeof(MlpTcImage) / 16); i += kRenderThreads)       // LDGSTS: lands while the rays / depths / taps are computed
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(tc::smem_u32(dst + i)), "l"(src + i) : "memory");
        asm volatile("cp.async.commit_group;" ::: "memory");
    }

    // ---- rays + limits -------------------------------------------------------------------------------------
    if (tid < R) {
        const int m = ray_of<R>(a, tile, tid);
        float* rf = rayf + tid * 8;
        if (m < a.M) {
            Ray r = fetch_ray(a.ray_o, a.ray_d, a.camera, a.res, n, a.M, m);
            float2 lim = a.limits[(size_t)n * a.M + m];
            if (!a.valid[(size_t)n * a.M + m] && a.ws->n_valid > 0) {      // renderer.py:125-126 (far end from ray_START, sic)
                lim.x = ord2f(a.ws->t0_min); lim.y = ord2f(a.ws->t0_max);
            }
            rf[0] = r.ox; rf[1] = r.oy; rf[2] = r.oz; rf[3] = r.dx; rf[4] = r.dy; rf[5] = r.dz; rf[6] = lim.x; rf[7] = lim.y;
        } else {
#pragma unroll
            for (int q = 0; q < 8; ++q) rf[q] = 0.f;
        }
    }
    __syncthreads();

    // ---- coarse depths (renderer.py:223-226, math_utils.py:101-118) -----------------------------------------
    float dmin = __int_as_float(0x7f800000), dmax = __int_as_float(0xff800000);
    for (int q = tid; q < R * a.S; q += kRenderThreads) {
        const int r = q / a.S, k = q - r * a.S;
        const int m = ray_of<R>(a, tile, r);
        float d = 0.f;
        if (m < a.M) {
            const float t0 = rayf[r * 8 + 6], t1 = rayf[r * 8 + 7];
            const float u = a.u_coarse[((size_t)n * a.M + m) * a.S + k];
            const float step = __fdiv_rn((float)k, (float)(a.S - 1));
            d = __fadd_rn(t0, __fmul_rn(step, __fsub_rn(t1, t0)));
            d = __fadd_rn(d, __fmul_rn(u, __fdiv_rn(__fsub_rn(t1, t0), (float)(a.S - 1))));
            dmin = fminf(dmin, d); dmax = fmaxf(dmax, d);
        }
        dep[r * ST + k] = d;
    }
    __syncthreads();

    const float* base0 = a.p0.base + (size_t)n * a.p0.frame_stride;
    const float* base1 = a.p1.base ? a.p1.base + (size_t)n * a.p1.frame_stride : nullptr;     // optional second plane set (same strides)
    const int rowstep = a.p0.row_stride, texstep = a.p0.texel_stride;
    const float pscale = 2.0f / a.box_warp;

    // One "pass" = gather + decode for samples k in [k0, k0+kn) of every ray.
    auto run_pass = [&](int k0, int kn) {
        const int nsamp = R * kn;
        // (1) one thread per sample: position -> three tap descriptors (texel offset + 4 bilinear weights with the zero padding
        //     folded in) written into the sample's own row; done ONCE per sample instead of once per lane of the gather group
        for (int q = tid; q < nsamp; q += kRenderThreads) {
            const int r = q / kn, k = k0 + (q - r * kn);
            const float* rf = rayf + r * 8;
            const float d = dep[r * ST + k];
            const float x = __fadd_rn(rf[0], __fmul_rn(d, rf[3]));
            const float y = __fadd_rn(rf[1], __fmul_rn(d, rf[4]));
            const float z = __fadd_rn(rf[2], __fmul_rn(d, rf[5]));
            float* row = rows + (size_t)(r * ST + k) * kRow;
            sample_desc(a.p0, a.H, a.W, pscale * x, pscale * y, pscale * z, row);       // 15 floats (tri-planes) | 27 (tri-grids)
        }
        __syncthreads();
        // (2) gather: each warp takes 4 samples per iteration, 8 lanes x float4 per sample; the row's descriptor is read by all 8
        //     lanes and then overwritten by the 32 mean features
        const int sub = lane >> 3, cq = lane & 7;
        for (int q4 = warp * 4; q4 < nsamp; q4 += kWarps * 4) {
            const int q = q4 + sub;
            if (q < nsamp) {
                const int r = q / kn, k = k0 + (q - r * kn);
                float* row = rows + (size_t)(r * ST + k) * kRow;
                float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
                if (a.p0.depth > 1) {                                    // tri-grids
                    float dg[27];
#pragma unroll
                    for (int e = 0; e < 27; ++e) dg[e] = row[e];
                    gather_desc<true>(base0, dg, rowstep, texstep, a.p0.slice_stride, cq, acc);
                    if (base1 != nullptr) gather_desc<true>(base1, dg, rowstep, texstep, a.p0.slice_stride, cq, acc);
                } else {
                    float dp[15];
#pragma unroll
                    for (int e = 0; e < 15; ++e) dp[e] = row[e];
                    gather_desc<false>(base0, dp, rowstep, texstep, 0, cq, acc);
                    if (base1 != nullptr) gather_desc<false>(base1, dp, rowstep, texstep, 0, cq, acc);
                }
                const float third = 1.0f / 3.0f;
                if (TC) {
                    // mean features as fp16 hi + lo halves straight into the swizzled A1 tile: lane cq owns K = [4cq, 4cq+4) of both halves
                    const float f0 = acc.x * third, f1 = acc.y * third, f2 = acc.z * third, f3 = acc.w * third;
                    const __half2 h01 = __floats2half2_rn(f0, f1), h23 = __floats2half2_rn(f2, f3);
                    const float2 g01 = __half22float2(h01), g23 = __half22float2(h23);
                    const __half2 l01 = __floats2half2_rn(f0 - g01.x, f1 - g01.y), l23 = __floats2half2_rn(f2 - g23.x, f3 - g23.y);
                    const int trow = q & 127;
                    uint8_t* rp = a1 + (q >> 7) * 16384 + (trow >> 3) * 1024 + (trow & 7) * 128 + (cq & 1) * 8;
                    uint2 hv, lv;
                    hv.x = *reinterpret_cast<const uint32_t*>(&h01); hv.y = *reinterpret_cast<const uint32_t*>(&h23);
                    lv.x = *reinterpret_cast<const uint32_t*>(&l01); lv.y = *reinterpret_cast<const uint32_t*>(&l23);
                    *reinterpret_cast<uint2*>(rp + (((cq >> 1) ^ (trow & 7)) << 4)) = hv;
                    *reinterpret_cast<uint2*>(rp + (((4 + (cq >> 1)) ^ (trow & 7)) << 4)) = lv;
                } else {
                    __syncwarp(__activemask());
                    row[cq * 4 + 0] = acc.x * third; row[cq * 4 + 1] = acc.y * third;
                    row[cq * 4 + 2] = acc.z * third; row[cq * 4 + 3] = acc.w * third;
                }
            }
        }
        if (TC) {
            // ---- decoder on the tensor core: warpgroup wg computes rows [64 wg, 64 wg + 64) of every 128-sample tile ---------------------
            const int nt = (nsamp + 127) >> 7, wg = warp >> 2;
            asm volatile("cp.async.wait_group 0;" ::: "memory");                // the weight image has landed
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");        // this thread's A1 (and W) stores -> visible to the async proxy
            __syncthreads();
            const uint32_t a1_s = tc::smem_u32(a1) + wg * 8192, a2_s = tc::smem_u32(a2) + wg * 8192, w_s = tc::smem_u32(wimg);
            auto layer1 = [&](int t, float* acc) {                             // x_hi w_hi + x_lo w_hi + x_hi w_lo, 2 k-steps each
                uint32_t accum = 0;
#pragma unroll
                for (int term = 0; term < 3; ++term) {
                    const uint32_t ao = term == 1 ? 64u : 0u, bo = term == 2 ? 64u : 0u;
#pragma unroll
                    for (int ks = 0; ks < 2; ++ks) {
                        tc::wgmma_m64n64k16(acc, tc::gmma_desc_sw128(a1_s + t * 16384 + ao + ks * 32), tc::gmma_desc_sw128(w_s + bo + ks * 32), accum);
                        accum = 1;
                    }
                }
            };
            float h[32], hn[32];                                               // layer-1 accumulators of the current and the next tile
            tc::wg_fence();
            layer1(0, h);
            if (nt > 1) layer1(1, hn);                                         // A2 overlays the A1 tiles: every layer-1 product is taken first
            tc::wg_commit();
            tc::wg_wait<0>();
            tc::wg_fence_acc<32>(h); tc::wg_fence_acc<32>(hn);
            for (int t = 0; t < nt; ++t) {
                // hidden units of tile t: +bias, softplus, re-split into the A2 atoms (row = sample, K = hidden unit)
#pragma unroll
                for (int i = 0; i < 32; i += 2) {
                    const int trow = 64 * wg + tc::acc_row(i), j = tc::acc_col(i);
                    const float h0 = softplus_fast(h[i] + b1s[j]), h1 = softplus_fast(h[i + 1] + b1s[j + 1]);
                    const __half2 hh = __floats2half2_rn(h0, h1);
                    const float2 hf = __half22float2(hh);
                    const __half2 ll = __floats2half2_rn(h0 - hf.x, h1 - hf.y);
                    *reinterpret_cast<__half2*>(a2 + sw128_off(trow, j)) = hh;
                    *reinterpret_cast<__half2*>(a2 + 16384 + sw128_off(trow, j)) = ll;
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                __syncthreads();
                float o[24];
                tc::wg_fence();
                {                                                              // layer 2: h_hi w_hi + h_lo w_hi + h_hi w_lo, 4 k-steps each
                    uint32_t accum = 0;
#pragma unroll
                    for (int term = 0; term < 3; ++term) {
                        const uint32_t ao = term == 1 ? 16384u : 0u, bo = term == 2 ? (8192u + 6144u) : 8192u;
#pragma unroll
                        for (int ks = 0; ks < 4; ++ks) {
                            tc::wgmma_m64n48k16(o, tc::gmma_desc_sw128(a2_s + ao + ks * 32), tc::gmma_desc_sw128(w_s + bo + ks * 32), accum);
                            accum = 1;
                        }
                    }
                }
                tc::wg_commit();
                tc::wg_wait<0>();
                tc::wg_fence_acc<24>(o);
                __syncthreads();                                               // both warpgroups are done reading A2
                // outputs of tile t: bias, sigma raw, colours through the scaled sigmoid
#pragma unroll
                for (int i = 0; i < 24; ++i) {
                    const int sidx = t * 128 + 64 * wg + tc::acc_row(i), oc = tc::acc_col(i);
                    if (oc < kOut && sidx < nsamp) {
                        const int r = sidx / kn, k = k0 + (sidx - r * kn);
                        float* out = rows + (size_t)(r * ST + k) * kRow;
                        out[oc] = oc == 0 ? o[i] + b2s[0] : sigmoid_fast(o[i] + b2s[oc]) * 1.002f - 0.001f;
                    }
                }
#pragma unroll
                for (int i = 0; i < 32; ++i) h[i] = hn[i];
            }
            __syncthreads();
            return;
        }
        __syncthreads();
        // decode: two samples per thread
        const int half = (nsamp + 1) >> 1;
        for (int p = tid; p < half; p += kRenderThreads) {
            const int qa = p, qb = p + half;
            const int ra = qa / kn, ka = k0 + (qa - ra * kn);
            const bool has_b = qb < nsamp;
            const int rb = has_b ? qb / kn : ra, kb = has_b ? k0 + (qb - rb * kn) : ka;
            decode_pair(mlp, rows + (size_t)(ra * ST + ka) * kRow, rows + (size_t)(rb * ST + kb) * kRow, has_b);
        }
        __syncthreads();
    };

    // Ray march (ray_marcher.py:26-57) over `cnt` samples of ray r taken in the order idx[0..cnt), one warp per ray:
    //   (1) lane l owns a contiguous chunk of intervals: alpha_k from the midpoint density, local transmittance products;
    //   (2) exclusive warp scan of the chunk products -> T_k, w_k = alpha_k T_k; sums of w and w*mid-depth by warp reduction;
    //   (3) lane = colour channel: rgb = sum_k v_k c_k with v_k = (w_{k-1} + w_k)/2  (== sum_k w_k (c_k + c_{k+1})/2).
    // `wbuf` (>= cnt floats) receives w_k (k < cnt-1); `vbuf` is scratch for v_k.
    auto march = [&](int r, int cnt, const int* idx, bool write_out, float* wbuf, float* vbuf) {
        const float* rr = rows + (size_t)r * ST * kRow;
        const float* dd = dep + r * ST;
        const int nint = cnt - 1;
        const int chunk = (nint + 31) >> 5;                                   // intervals per lane (2 for 47, 3 for 95)
        const int kb = lane * chunk, ke = min(kb + chunk, nint);
        float prod = 1.0f;
        for (int k = kb; k < ke; ++k) {
            const int ia = idx ? idx[k] : k, ib = idx ? idx[k + 1] : k + 1;
            const float delta = dd[ib] - dd[ia];
            const float smid = softplus_fast((rr[ia * kRow] + rr[ib * kRow]) * 0.5f - 1.0f);     // ray_marcher.py:33
            const float alpha = 1.0f - __expf(-(smid * delta));
            wbuf[k] = alpha;                                                  // alpha for now, weight below
            prod *= (1.0f - alpha + 1e-10f);
        }
        float incl = prod;                                                    // inclusive scan of the chunk products
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const float t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl *= t; }
        float T = __shfl_up_sync(0xffffffffu, incl, 1);
        if (lane == 0) T = 1.0f;
        float wsum = 0.f, dsum = 0.f;
        for (int k = kb; k < ke; ++k) {
            const int ia = idx ? idx[k] : k, ib = idx ? idx[k + 1] : k + 1;
            const float alpha = wbuf[k];
            const float w = alpha * T;
            T *= (1.0f - alpha + 1e-10f);
            wbuf[k] = w;
            wsum += w; dsum = fmaf(w, (dd[ia] + dd[ib]) * 0.5f, dsum);
        }
        __syncwarp();
        if (!write_out) return;
#pragma unroll
        for (int o = 16; o; o >>= 1) { wsum += __shfl_xor_sync(0xffffffffu, wsum, o); dsum += __shfl_xor_sync(0xffffffffu, dsum, o); }
        for (int k = lane; k < cnt; k += 32) vbuf[k] = 0.5f * ((k > 0 ? wbuf[k - 1] : 0.f) + (k < nint ? wbuf[k] : 0.f));
        __syncwarp();
        float acc = 0.f;
#pragma unroll 4
        for (int k = 0; k < cnt; ++k) {
            const int ia = idx ? idx[k] : k;
            acc = fmaf(vbuf[k], rr[ia * kRow + 1 + lane], acc);
        }
        const int m = ray_of<R>(a, tile, r);
        if (m < a.M) {
            const size_t o = (size_t)n * a.M + m;
            if (a.white_back) acc = acc + 1.0f - wsum;
            a.rgb[o * (kOut - 1) + lane] = acc * 2.0f - 1.0f;
            if (lane == 0) { a.wsum[o] = wsum; a.depth[o] = dsum / wsum; }       // 0/0 -> NaN, fixed by depth_clamp_kernel
        }
    };

    run_pass(0, a.S);

    const int S = a.S, Ni = a.S_imp;
    for (int r = warp; r < R; r += kWarps) {
        float* w = wts + r * ST; float* cd = cdf + r * ST; float* dd = dep + r * ST;
        march(r, S, nullptr, false, w, cd);                                   // coarse weights w[0..S-2]
        __syncwarp();
        // renderer.py:245-247: max_pool1d(2,1,pad 1) -> avg_pool1d(2,1) -> +0.01 ; a_i, i = 0..S-2
        // pdf over p_i = a_{i+1} + 1e-5, i = 0..S-4 ; cdf has S-2 entries (renderer.py:272-276)
        float total = 0.f;
        for (int i = 0; i < S - 3; ++i) {              // every lane computes the same serial sums (torch.cumsum order)
            const int j = i + 1;                                             // index into a
            const float m0 = fmaxf(w[j - 1], w[j]), m1 = fmaxf(w[j], w[j + 1]);   // 1 <= j <= S-3: no -inf padding reached
            total += (0.5f * (m0 + m1) + 0.01f) + 1e-5f;
        }
        float run = 0.f;
        if (lane == 0) cd[0] = 0.f;
        for (int i = 0; i < S - 3; ++i) {
            const int j = i + 1;
            const float m0 = fmaxf(w[j - 1], w[j]), m1 = fmaxf(w[j], w[j + 1]);
            run += __fdiv_rn((0.5f * (m0 + m1) + 0.01f) + 1e-5f, total);
            if (lane == 0) cd[i + 1] = run;
        }
        __syncwarp();
        const int ncdf = S - 2;
        const int m_ray = ray_of<R>(a, tile, r);
        for (int j = lane; j < Ni; j += 32) {
            float dfine = 0.f;
            if (m_ray < a.M) {
                const float u = a.u_fine[((size_t)n * a.M + m_ray) * Ni + j];
                int idx = 0;                                                 // searchsorted(cdf, u, right=True)
                while (idx < ncdf && cd[idx] <= u) ++idx;
                const int lo = max(idx - 1, 0), hi = min(idx, S - 3);
                const float c_lo = cd[lo], c_hi = cd[hi];
                float den = c_hi - c_lo;
                if (den < 1e-5f) den = 1.0f;
                const float b_lo = 0.5f * (dd[lo] + dd[lo + 1]), b_hi = 0.5f * (dd[hi] + dd[hi + 1]);
                dfine = b_lo + __fdiv_rn(u - c_lo, den) * (b_hi - b_lo);
                dmin = fminf(dmin, dfine); dmax = fmaxf(dmax, dfine);
            }
            dd[S + j] = dfine;
        }
    }
    __syncthreads();
    run_pass(S, Ni);
    // merge: stable rank of every sample among the ray's ST depths (== torch.sort order when depths are distinct)
    for (int r = warp; r < R; r += kWarps) {
        const float* dd = dep + r * ST; int* od = ord + r * ST;
        for (int i = lane; i < ST; i += 32) {
            // total order (torch.sort puts NaN last, -0 == +0): every sample gets a distinct rank even for NaN depths (degenerate
            // cameras), so `ord` never holds an unwritten slot
            const unsigned ki = sort_key(dd[i]);
            int rank = 0;
            for (int j = 0; j < ST; ++j) { const unsigned kj = sort_key(dd[j]); rank += (kj < ki) || (kj == ki && j < i); }
            od[rank] = i;
        }
        __syncwarp();
        march(r, ST, od, true, wts + r * ST, cdf + r * ST);
    }

    // call-wide min/max of the sample depths (ray_marcher.py:50)
    dmin = warp_min(dmin); dmax = warp_max(dmax);
    if (lane == 0 && dmin <= dmax) { atomicMin(&a.ws->d_min, f2ord(dmin)); atomicMax(&a.ws->d_max, f2ord(dmax)); }
}

// Stand-alone marcher: one warp per ray, lane = channel (C <= 32 per pass, loops for wider C).
__global__ void ray_march_kernel(const float* __restrict__ colors, const float* __restrict__ sigmas,
                                 const float* __restrict__ depths, int NM, int S, int C, int white_back,
                                 float* __restrict__ rgb, float* __restrict__ depth, float* __restrict__ weights, RenderWs* ws) {
    const int ray = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    float dmin = __int_as_float(0x7f800000), dmax = __int_as_float(0xff800000);
    if (ray < NM) {
        const float* dd = depths + (size_t)ray * S; const float* ss = sigmas + (size_t)ray * S;
        const float* cc = colors + (size_t)ray * S * C;
        for (int i = lane; i < S; i += 32) { dmin = fminf(dmin, dd[i]); dmax = fmaxf(dmax, dd[i]); }
        for (int c0 = 0; c0 < C; c0 += 32) {
            const int c = c0 + lane; const bool on = c < C;
            float T = 1.f, acc = 0.f, wsum = 0.f, dsum = 0.f;
            for (int i = 0; i + 1 < S; ++i) {
                const float delta = dd[i + 1] - dd[i];
                const float smid = softplus_fast((ss[i] + ss[i + 1]) * 0.5f - 1.0f);
                const float alpha = 1.0f - __expf(-(smid * delta));
                const float w = alpha * T;
                T *= (1.0f - alpha + 1e-10f);
                if (on) acc = fmaf(w, (cc[(size_t)i * C + c] + cc[(size_t)(i + 1) * C + c]) * 0.5f, acc);
                wsum += w; dsum = fmaf(w, (dd[i] + dd[i + 1]) * 0.5f, dsum);
                if (c0 == 0 && lane == 0) weights[(size_t)ray * (S - 1) + i] = w;
            }
            if (white_back) acc = acc + 1.0f - wsum;
            if (on) rgb[(size_t)ray * C + c] = acc * 2.0f - 1.0f;
            if (c0 == 0 && lane == 0) depth[ray] = dsum / wsum;
        }
    }
    dmin = warp_min(dmin); dmax = warp_max(dmax);
    if (lane == 0 && dmin <= dmax) { atomicMin(&ws->d_min, f2ord(dmin)); atomicMax(&ws->d_max, f2ord(dmax)); }
}

static size_t render_smem_bytes(int R, int ST) {
    return sizeof(MlpSmem) + (size_t)R * ST * kRow * 4 + 3 * (size_t)R * ST * 4 + (size_t)R * 8 * 4 + (size_t)R * ST * 4;
}

static size_t render_tc_smem(int R, int S, int S_imp) {
    const int ST = S + S_imp;
    return 1024 + kTcA2Bytes + 20480 + (kHidden + 48) * 4 + (size_t)R * ST * (kRow + 4) * 4 + (size_t)R * 8 * 4;
}
// the tensor-core decoder needs each pass of its CTA tile to fit the two 128-sample A tiles, and two CTAs per SM (2 x 113 KB of shared memory)
static bool render_tc_fits(int R, int S, int S_imp) {
    const int per_pass = R * (S > S_imp ? S : S_imp);
    return per_pass <= 256 && render_tc_smem(R, S, S_imp) <= 113 * 1024;
}
template <int R>
static int launch_render_tc(const RenderArgs& a, cudaStream_t st) {
    const size_t smem = render_tc_smem(R, a.S, a.S_imp);
    R3DP_CUDA(cudaFuncSetAttribute(render_kernel<R, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid(a.tiles_per_frame, a.N);                     // (the decoder image was written by r3dp_render_ex's set-up launch)
    render_kernel<R, true><<<grid, kTcThreads, smem, st>>>(a);
    R3DP_LAUNCH_CHECK();
    return 0;
}

template <int R>
static int launch_render_v(const RenderArgs& a, cudaStream_t st) {
    const size_t smem = render_smem_bytes(R, a.S + a.S_imp);
    R3DP_CUDA(cudaFuncSetAttribute(render_kernel<R, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid(a.tiles_per_frame, a.N);
    render_kernel<R, false><<<grid, kRenderThreads, smem, st>>>(a);
    R3DP_LAUNCH_CHECK();
    return 0;
}
template <int R>
static int launch_render(const RenderArgs& a, bool tc, cudaStream_t st) {
    R3DP_REQUIRE(a.S_imp > 0, "render: the tile kernel runs two-pass renders only (S_imp = %d)", a.S_imp);
    return tc ? launch_render_tc<R>(a, st) : launch_render_v<R>(a, st);
}

static int tile_rays(int ST) { return ST <= 48 ? 8 : ST <= 96 ? 4 : ST <= 192 ? 2 : 1; }     // rays per CTA of the tile kernel

// The kernel a render runs (r3dp_render_ex dispatches on this, r3dp_render_path reports it): 0 = streaming kernel (single-pass renders),
// 1 = tile kernel with the tensor-core decoder (two-pass renders whose passes fit its tiles), 2 = tile kernel with the smem-weights
// CUDA-core decoder (the other two-pass renders); both tile decoders keep the decoder in per-call storage
static int render_path(const RenderArgs& a) {
    if (a.S_imp == 0) return 0;
    return render_tc_fits(tile_rays(a.S + a.S_imp), a.S, a.S_imp) ? 1 : 2;
}

// the fields of the kernel arguments that follow from the caller's argument block alone (not from the workspace)
static RenderArgs render_args(const r3dp_render_args_t* g) {
    RenderArgs a = {};
    a.p0.base = g->planes; a.p0.frame_stride = g->layout.frame_stride; a.p0.plane_stride = g->layout.plane_stride;
    a.p0.row_stride = g->layout.row_stride; a.p0.texel_stride = g->layout.texel_stride; a.p0.depth = g->layout.depth; a.p0.slice_stride = g->layout.slice_stride;
    if (g->planes2) {
        a.p1.base = g->planes2; a.p1.frame_stride = g->layout2.frame_stride; a.p1.plane_stride = g->layout2.plane_stride;
        a.p1.row_stride = g->layout2.row_stride; a.p1.texel_stride = g->layout2.texel_stride; a.p1.depth = g->layout2.depth; a.p1.slice_stride = g->layout2.slice_stride;
    }
    a.N = g->N; a.H = g->H; a.W = g->W; a.ray_o = g->ray_o; a.ray_d = g->ray_d; a.camera = g->camera; a.M = g->M; a.res = g->res;
    a.S = g->S; a.S_imp = g->S_imp; a.box_warp = g->box_warp; a.white_back = g->white_back; a.u_coarse = g->u_coarse; a.u_fine = g->u_fine;
    a.mlp = *g->mlp;
    a.rgb = g->rgb; a.depth = g->depth; a.wsum = g->weights_sum; a.valid = g->is_ray_valid;
    return a;
}

}  // namespace r3dp

using namespace r3dp;

extern "C" int r3dp_gen_rays(const float* cam2world, const float* intrinsics, int N, int res, float* ray_o, float* ray_d,
                             r3dp_stream_t stream) {
    R3DP_REQUIRE(N > 0 && res > 0, "gen_rays: N and res must be positive (got %d, %d)", N, res);
    R3DP_REQUIRE(cam2world && intrinsics && ray_o && ray_d, "gen_rays: null pointer");
    const int total = N * res * res;
    gen_rays_kernel<<<(total + 255) / 256, 256, 0, as_stream(stream)>>>(cam2world, intrinsics, N, res, ray_o, ray_d);
    count_launches(1);
    R3DP_LAUNCH_CHECK();
    return 0;
}

extern "C" size_t r3dp_render_workspace_bytes(int N, int M) {
    return kWsLimitsOff + (size_t)N * M * sizeof(float2);
}

static int check_mlp(const r3dp_mlp_t* mlp, int C) {
    R3DP_REQUIRE(mlp && mlp->w1 && mlp->b1 && mlp->w2 && mlp->b2, "decoder: null parameter pointer");
    R3DP_REQUIRE(mlp->in_features == kC && mlp->hidden == kHidden && mlp->out_dim == kOut - 1 && C == kC,
                 "decoder: only the OSGDecoder shape 32->64->1+32 is built (got %d->%d->1+%d, C=%d)",
                 mlp->in_features, mlp->hidden, mlp->out_dim, C);
    return 0;
}

static int check_layout(const r3dp_plane_layout_t& l, int H, int W, const char* what) {
    R3DP_REQUIRE(l.plane_stride > 0 && l.row_stride > 0 && l.texel_stride >= kC && l.frame_stride >= 0, "render: bad %s plane strides", what);
    R3DP_REQUIRE((l.plane_stride % 4) == 0 && (l.row_stride % 4) == 0 && (l.texel_stride % 4) == 0 && (l.frame_stride % 4) == 0 && (l.slice_stride % 4) == 0,
                 "render: %s plane strides must keep texels 16-byte aligned", what);
    R3DP_REQUIRE(l.depth <= 1 || (l.depth <= 64 && l.slice_stride > 0), "render: tri-grids need 2 <= depth <= 64 slices and a slice stride (%s set)", what);
    const long long span = 2ll * l.plane_stride + (long long)(l.depth > 1 ? l.depth - 1 : 0) * l.slice_stride + (long long)(H - 1) * l.row_stride +
                           (long long)(W - 1) * l.texel_stride + kC;
    R3DP_REQUIRE(span < (1ll << 31), "render: %s planes of %dx%d exceed the 32-bit texel offsets of the tap descriptors", what, H, W);
    return 0;
}

extern "C" int r3dp_render_ex(const r3dp_render_args_t* g, r3dp_stream_t stream) {
    R3DP_REQUIRE(g != nullptr, "render: null argument block");
    if (check_mlp(g->mlp, g->C)) return 1;
    const int N = g->N, M = g->M, H = g->H, W = g->W, S = g->S, S_imp = g->S_imp, res = g->res;
    R3DP_REQUIRE(g->planes && g->u_coarse && g->rgb && g->depth && g->weights_sum && g->is_ray_valid && g->workspace, "render: null pointer");
    R3DP_REQUIRE(N > 0 && M > 0 && H >= 2 && W >= 2, "render: bad shape N=%d M=%d H=%d W=%d (planes must be at least 2x2)", N, M, H, W);
    R3DP_REQUIRE(S >= 4, "render: depth_resolution must be >= 4 (got %d)", S);
    R3DP_REQUIRE(S_imp >= 0 && (S_imp == 0 || g->u_fine), "render: depth_resolution_importance=%d needs u_fine", S_imp);
    R3DP_REQUIRE(g->box_warp > 0.f, "render: box_warp must be positive");
    R3DP_REQUIRE((g->ray_o && g->ray_d) || (g->camera && res > 0 && res * res == M), "render: need rays, or camera with M == res*res");
    R3DP_REQUIRE(g->workspace_bytes >= r3dp_render_workspace_bytes(N, M), "render: workspace too small");
    R3DP_REQUIRE((reinterpret_cast<uintptr_t>(g->workspace) & 15) == 0 && (reinterpret_cast<uintptr_t>(g->planes) & 15) == 0, "render: workspace and planes must be 16-byte aligned");
    const int ST = S + S_imp;
    R3DP_REQUIRE(ST <= 384, "render: at most 384 samples per ray are supported (got %d)", ST);
    if (check_layout(g->layout, H, W, "first")) return 1;
    if (g->planes2) {
        if (check_layout(g->layout2, H, W, "second")) return 1;
        R3DP_REQUIRE(g->layout2.plane_stride == g->layout.plane_stride && g->layout2.row_stride == g->layout.row_stride &&
                     g->layout2.texel_stride == g->layout.texel_stride && g->layout2.depth == g->layout.depth &&
                     g->layout2.slice_stride == g->layout.slice_stride && (reinterpret_cast<uintptr_t>(g->planes2) & 15) == 0,
                     "render: the second plane set must use the strides of the first (only its frame stride may differ)");
    }
    cudaStream_t st = as_stream(stream);

    char* wsb = reinterpret_cast<char*>(g->workspace);
    RenderWs* ws = reinterpret_cast<RenderWs*>(wsb);
    float2* limits = reinterpret_cast<float2*>(wsb + kWsLimitsOff);
    mlp_to_tc_kernel<<<4, 256, 0, st>>>(*g->mlp, reinterpret_cast<MlpTcImage*>(wsb + kWsImageOff), ws);      // + workspace header
    const int total = N * M;
    ray_limits_kernel<<<(total + 255) / 256, 256, 0, st>>>(g->ray_o, g->ray_d, g->camera, res, N, M, g->box_warp, limits, g->is_ray_valid, ws);
    R3DP_LAUNCH_CHECK();

    RenderArgs a = render_args(g);
    a.image = reinterpret_cast<const MlpTcImage*>(wsb + kWsImageOff); a.limits = limits; a.ws = ws;
    a.lookahead = kRenderLookahead;
    int rc;
    const int path = render_path(a);
    if (path == 0) {
        rc = launch_render_stream(a, st);
    } else {
        const int R = tile_rays(ST);
        const bool image = res > 0 && res * res == M && (res % R) == 0;
        a.tile_cols = image ? res : 0;
        a.tiles_per_frame = (M + R - 1) / R;
        const bool tc = path == 1;
        rc = R == 8 ? launch_render<8>(a, tc, st) : R == 4 ? launch_render<4>(a, tc, st) : R == 2 ? launch_render<2>(a, tc, st) : launch_render<1>(a, tc, st);
    }
    if (rc) return rc;
    count_launches(4);
    depth_clamp_kernel<<<(total + 255) / 256, 256, 0, st>>>(g->depth, total, ws);
    R3DP_LAUNCH_CHECK();
    return 0;
}

extern "C" int r3dp_render_path(const r3dp_render_args_t* g) {
    if (g == nullptr || g->mlp == nullptr) { set_error("render_path: null argument block or decoder"); return -1; }
    return render_path(render_args(g));
}

extern "C" int r3dp_ray_march(const float* colors, const float* sigmas, const float* depths, int N, int M, int S, int C,
                              int white_back, float* rgb, float* depth, float* weights, void* workspace, r3dp_stream_t stream) {
    R3DP_REQUIRE(colors && sigmas && depths && rgb && depth && weights && workspace, "ray_march: null pointer");
    R3DP_REQUIRE(N > 0 && M > 0 && S >= 2 && C > 0, "ray_march: bad shape");
    cudaStream_t st = as_stream(stream);
    RenderWs* ws = reinterpret_cast<RenderWs*>(workspace);
    init_ws_kernel<<<1, 1, 0, st>>>(ws);
    const int NM = N * M;
    ray_march_kernel<<<(NM + 7) / 8, 256, 0, st>>>(colors, sigmas, depths, NM, S, C, white_back, rgb, depth, weights, ws);
    depth_clamp_kernel<<<(NM + 255) / 256, 256, 0, st>>>(depth, NM, ws);
    count_launches(3);
    R3DP_LAUNCH_CHECK();
    return 0;
}
