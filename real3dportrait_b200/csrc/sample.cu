// Stand-alone tri-plane ops behind the reference's public sampler API:
//   planes_to_channels_last   [N,3,C,H,W] -> [N,3,H,W,C]        (HBM-bound transposition)
//   triplane_sample           sample_from_planes (renderer.py:65-75): the HBM-roofline gather, write-dominated
//   run_model                 ImportanceRenderer.run_model (renderer.py:169-188): gather + OSG decoder
#include "render_shared.cuh"
#include <stdlib.h>

namespace r3dp {

// ---- layout change ------------------------------------------------------------------------------------------------
// One CTA moves a [32 ch][128 px] tile through shared memory: reads are 512 B contiguous per channel row (float4 per
// lane), writes are 128 B contiguous per pixel (float4 per lane, 8 lanes per pixel).
constexpr int kTilePx = 128;
// D = depth slices per plane (1: tri-planes).  Source channel index = c*D + d (the reference views [N,3,C*D,H,W] as [N*3,C,D,H,W],
// renderer.py:83); destination [N,3,D,H,W,C]: every slice is a channels-last plane.
__global__ void __launch_bounds__(256) planes_to_cl_kernel(const float* __restrict__ src, float* __restrict__ dst, int HW, int D) {
    __shared__ float tile[kC][kTilePx + 1];
    const int plane = blockIdx.y / D, dsl = blockIdx.y - plane * D;        // plane = n*3 + p
    const int px0 = blockIdx.x * kTilePx;
    const float* s = src + ((size_t)plane * kC * D + dsl) * HW;
    float* d = dst + ((size_t)plane * D + dsl) * HW * kC;
    const size_t cstride = (size_t)D * HW;
    const int tid = threadIdx.x;
    const bool full = (px0 + kTilePx <= HW) && ((HW & 3) == 0);
    if (full) {
#pragma unroll
        for (int it = 0; it < (kC * kTilePx / 4) / 256; ++it) {       // 4 iterations
            const int v = it * 256 + tid;                              // float4 index in tile
            const int c = v / (kTilePx / 4), p4 = v % (kTilePx / 4);
            const float4 f = ldg_nc_f4(s + (size_t)c * cstride + px0 + p4 * 4);
            tile[c][p4 * 4 + 0] = f.x; tile[c][p4 * 4 + 1] = f.y; tile[c][p4 * 4 + 2] = f.z; tile[c][p4 * 4 + 3] = f.w;
        }
    } else {
        for (int v = tid; v < kC * kTilePx; v += 256) {
            const int c = v / kTilePx, p = v % kTilePx;
            tile[c][p] = (px0 + p < HW) ? s[(size_t)c * cstride + px0 + p] : 0.f;
        }
    }
    __syncthreads();
#pragma unroll
    for (int it = 0; it < (kC * kTilePx / 4) / 256; ++it) {
        const int v = it * 256 + tid;
        const int p = v / (kC / 4), c4 = v % (kC / 4);
        if (px0 + p < HW) {
            float4 f = make_float4(tile[c4 * 4 + 0][p], tile[c4 * 4 + 1][p], tile[c4 * 4 + 2][p], tile[c4 * 4 + 3][p]);
            *reinterpret_cast<float4*>(d + (size_t)(px0 + p) * kC + c4 * 4) = f;
        }
    }
}

// ---- sample_from_trigrids (renderer.py:78-89) on [N,3,D,H,W,C] -----------------------------------------------------------------------
// warp = 4 points x 8 lanes x float4; per plane one descriptor (8 trilinear taps), results per plane as the reference returns them.
__global__ void __launch_bounds__(256, 3) trigrid_sample_kernel(const float* __restrict__ grids, int N, int D, int H, int W,
                                                                const float* __restrict__ coords, int P, float scale, float* __restrict__ out) {
    const int lane = threadIdx.x & 31, sub = lane >> 3, cq = lane & 7;
    const long long total4 = ((long long)N * P + 3) / 4;
    const long long wstride = (long long)gridDim.x * (blockDim.x >> 5);
    const int ts = kC, rs = W * kC, ss = H * W * kC, ps = D * ss;
    for (long long g = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); g < total4; g += wstride) {
        const long long pt = g * 4 + sub;
        if (pt >= (long long)N * P) continue;
        const int n = (int)(pt / P); const int s = (int)(pt - (long long)n * P);
        const float* c = coords + pt * 3;
        const float gx = scale * __ldg(c), gy = scale * __ldg(c + 1), gz = scale * __ldg(c + 2);
        const float* base = grids + (size_t)n * 3 * ps;
#pragma unroll
        for (int p = 0; p < 3; ++p) {
            float d[9];
            const float gu = p == 2 ? gz : gx, gv = p == 0 ? gy : (p == 1 ? gz : gx), gw = p == 0 ? gz : gy;
            tap_desc_grid(gu, gv, gw, H, W, D, p * ps, ss, rs, ts, d);
            const float* b = base + __float_as_int(d[0]) + cq * 4;
            const float4 t0 = ldg_nc_f4(b), t1 = ldg_nc_f4(b + ts), t2 = ldg_nc_f4(b + rs), t3 = ldg_nc_f4(b + rs + ts);
            const float4 u0 = ldg_nc_f4(b + ss), u1 = ldg_nc_f4(b + ss + ts), u2 = ldg_nc_f4(b + ss + rs), u3 = ldg_nc_f4(b + ss + rs + ts);
            float4 r;
            r.x = t0.x * d[1] + t1.x * d[2] + t2.x * d[3] + t3.x * d[4] + u0.x * d[5] + u1.x * d[6] + u2.x * d[7] + u3.x * d[8];
            r.y = t0.y * d[1] + t1.y * d[2] + t2.y * d[3] + t3.y * d[4] + u0.y * d[5] + u1.y * d[6] + u2.y * d[7] + u3.y * d[8];
            r.z = t0.z * d[1] + t1.z * d[2] + t2.z * d[3] + t3.z * d[4] + u0.z * d[5] + u1.z * d[6] + u2.z * d[7] + u3.z * d[8];
            r.w = t0.w * d[1] + t1.w * d[2] + t2.w * d[3] + t3.w * d[4] + u0.w * d[5] + u1.w * d[6] + u2.w * d[7] + u3.w * d[8];
            stg_cs_f4(out + (((size_t)n * 3 + p) * P + s) * kC + cq * 4, r);
        }
    }
}

// ---- sample_from_planes ---------------------------------------------------------------------------------------------
// Persistent kernel, a warp owns chunks of 32 CONSECUTIVE points (chunk-cyclic over the grid; consecutive points are consecutive depths of a
// ray in the renderer's use, so the (x,y)-plane taps of a chunk hit L1).  Per chunk: lane = point computes the three tap descriptors ONCE
// (zero padding folded into the weights: no bounds checks, no predicated loads) into a 2 KB shared-memory block; then 8 steps of 4 points,
// 8 lanes x float4 = one 128-byte texel line per tap, ALL twelve 16-byte loads of a point issued before the first use, streaming stores
// (the output is never re-read here).  The coordinates of the next chunk are requested before this chunk's taps.
// Earlier forms: descriptors recomputed by all 8 lanes of a point + loads split into dependent groups at 64
// registers -> 59 % of the HBM peak with 60 % issue-active; MINB = resident CTAs per SM the register allocation targets.
template <int MINB>
__global__ void __launch_bounds__(256, MINB) triplane_sample_kernel(const float* __restrict__ planes, int N, int H, int W,
                                                                    const float* __restrict__ coords, int P, float scale,
                                                                    float* __restrict__ out) {
    __shared__ __align__(16) float s_desc[8][32][16];           // per warp: [point][off0 off1 off2 frame | 4 weights x 3 planes]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, sub = lane >> 3, cq = lane & 7;
    const long long NP = (long long)N * P, n_chunks = (NP + 31) / 32;
    const long long wstride = (long long)gridDim.x * 8;
    long long chunk = (long long)blockIdx.x * 8 + warp;
    float (*row)[16] = s_desc[warp];
    const size_t fstride = (size_t)3 * H * W * kC;
    const int rs = W * kC;
    float nx = 0.f, ny = 0.f, nz = 0.f;
    if (chunk < n_chunks && chunk * 32 + lane < NP) { const float* c = coords + (chunk * 32 + lane) * 3; nx = __ldg(c); ny = __ldg(c + 1); nz = __ldg(c + 2); }
    for (; chunk < n_chunks; chunk += wstride) {
        const long long pt0 = chunk * 32;
        const float gx = scale * nx, gy = scale * ny, gz = scale * nz;
        {
            const long long pt2 = (chunk + wstride) * 32 + lane;
            if (chunk + wstride < n_chunks && pt2 < NP) { const float* c = coords + pt2 * 3; nx = __ldg(c); ny = __ldg(c + 1); nz = __ldg(c + 2); }
        }
        {   // plane 0 <- (x,y), plane 1 <- (x,z), plane 2 <- (z,x)   (generate_planes + project_onto_planes, renderer.py:30-63)
            float t[5];
            float* r = row[lane];
            tap_desc(gx, gy, H, W, 0, t); r[0] = t[0]; r[4] = t[1]; r[5] = t[2]; r[6] = t[3]; r[7] = t[4];
            tap_desc(gx, gz, H, W, 1, t); r[1] = t[0]; r[8] = t[1]; r[9] = t[2]; r[10] = t[3]; r[11] = t[4];
            tap_desc(gz, gx, H, W, 2, t); r[2] = t[0]; r[12] = t[1]; r[13] = t[2]; r[14] = t[3]; r[15] = t[4];
        }
        __syncwarp();
#pragma unroll 1
        for (int it = 0; it < 8; ++it) {
            const int sp = it * 4 + sub;
            const long long pt = pt0 + sp;
            if (pt >= NP) break;                                                  // only the last chunk; whole 8-lane groups leave together
            const int n = (int)(pt / P); const int s = (int)(pt - (long long)n * P);
            const float4* rw = reinterpret_cast<const float4*>(row[sp]);
            const float4 offs = rw[0];
            const float* base = planes + (size_t)n * fstride + cq * 4;
            float4 t[12];
            {
                const float* b = base + __float_as_int(offs.x);
                t[0] = ldg_nc_f4(b); t[1] = ldg_nc_f4(b + kC); t[2] = ldg_nc_f4(b + rs); t[3] = ldg_nc_f4(b + rs + kC);
                b = base + __float_as_int(offs.y);
                t[4] = ldg_nc_f4(b); t[5] = ldg_nc_f4(b + kC); t[6] = ldg_nc_f4(b + rs); t[7] = ldg_nc_f4(b + rs + kC);
                b = base + __float_as_int(offs.z);
                t[8] = ldg_nc_f4(b); t[9] = ldg_nc_f4(b + kC); t[10] = ldg_nc_f4(b + rs); t[11] = ldg_nc_f4(b + rs + kC);
            }
            float* o = out + (((size_t)n * 3) * P + s) * kC + cq * 4;
#pragma unroll
            for (int p = 0; p < 3; ++p) {
                const float4 w = rw[1 + p];
                float4 r;
                r.x = t[4 * p].x * w.x + t[4 * p + 1].x * w.y + t[4 * p + 2].x * w.z + t[4 * p + 3].x * w.w;
                r.y = t[4 * p].y * w.x + t[4 * p + 1].y * w.y + t[4 * p + 2].y * w.z + t[4 * p + 3].y * w.w;
                r.z = t[4 * p].z * w.x + t[4 * p + 1].z * w.y + t[4 * p + 2].z * w.z + t[4 * p + 3].z * w.w;
                r.w = t[4 * p].w * w.x + t[4 * p + 1].w * w.y + t[4 * p + 2].w * w.z + t[4 * p + 3].w * w.w;
                stg_cs_f4(o + (size_t)p * P * kC, r);
            }
        }
        __syncwarp();
    }
}

// ---- run_model ----------------------------------------------------------------------------------------------------
constexpr int kRmThreads = 192, kRmPoints = 384;
__global__ void __launch_bounds__(kRmThreads, 2) run_model_kernel(const PlaneSet ps, int N, int H, int W,
                                                                 const float* __restrict__ coords, int P, float scale,
                                                                 const r3dp_mlp_t m, float* __restrict__ rgb,
                                                                 float* __restrict__ sigma) {
    extern __shared__ __align__(16) float smem[];
    MlpSmem& mlp = *reinterpret_cast<MlpSmem*>(smem);
    float* rows = smem + sizeof(MlpSmem) / 4;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, sub = lane >> 3, cq = lane & 7;
    const int n = blockIdx.y, p0 = blockIdx.x * kRmPoints;
    const int cnt = min(kRmPoints, P - p0);
    load_mlp_smem(mlp, m, tid, kRmThreads);
    const float* base = ps.base + (size_t)n * ps.frame_stride;
    for (int q4 = warp * 4; q4 < cnt; q4 += (kRmThreads / 32) * 4) {
        const int q = q4 + sub;
        if (q < cnt) {
            const float* c = coords + ((size_t)n * P + p0 + q) * 3;
            const float gx = scale * __ldg(c), gy = scale * __ldg(c + 1), gz = scale * __ldg(c + 2);
            float d[27];
            sample_desc(ps, H, W, gx, gy, gz, d);
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            if (ps.depth > 1) gather_desc<true>(base, d, ps.row_stride, ps.texel_stride, ps.slice_stride, cq, acc);
            else gather_desc<false>(base, d, ps.row_stride, ps.texel_stride, 0, cq, acc);
            float* row = rows + (size_t)q * kRow + cq * 4;
            const float third = 1.0f / 3.0f;
            row[0] = acc.x * third; row[1] = acc.y * third; row[2] = acc.z * third; row[3] = acc.w * third;
        }
    }
    __syncthreads();
    const int half = (cnt + 1) >> 1;
    for (int p = tid; p < half; p += kRmThreads) {
        const bool has_b = p + half < cnt;
        decode_pair(mlp, rows + (size_t)p * kRow, rows + (size_t)(has_b ? p + half : p) * kRow, has_b);
    }
    __syncthreads();
    float* o = rgb + ((size_t)n * P + p0) * (kOut - 1);
    for (int i = tid; i < cnt * (kOut - 1); i += kRmThreads) {
        const int q = i >> 5, c = i & 31;
        o[i] = rows[(size_t)q * kRow + 1 + c];
    }
    for (int q = tid; q < cnt; q += kRmThreads) sigma[(size_t)n * P + p0 + q] = rows[(size_t)q * kRow];
}

// ---- OSGDecoder.forward on caller-supplied features (triplane.py:133-146) -------------------------------------------
// feat [N,K,P,C] with K = 3 (mean over planes, triplane.py:135-136) or K = 1 (already aggregated).
__global__ void __launch_bounds__(kRmThreads, 2) decode_kernel(const float* __restrict__ feat, int K, int P, const r3dp_mlp_t m,
                                                              float* __restrict__ rgb, float* __restrict__ sigma) {
    extern __shared__ __align__(16) float smem[];
    MlpSmem& mlp = *reinterpret_cast<MlpSmem*>(smem);
    float* rows = smem + sizeof(MlpSmem) / 4;
    const int tid = threadIdx.x;
    const int n = blockIdx.y, p0 = blockIdx.x * kRmPoints;
    const int cnt = min(kRmPoints, P - p0);
    load_mlp_smem(mlp, m, tid, kRmThreads);
    const float invk = 1.0f / (float)K;
    for (int i = tid; i < cnt * kC; i += kRmThreads) {
        const int q = i >> 5, c = i & 31;
        float acc = 0.f;
        for (int k = 0; k < K; ++k) acc += feat[(((size_t)n * K + k) * P + p0 + q) * kC + c];
        rows[(size_t)q * kRow + c] = K == 1 ? acc : acc * invk;
    }
    __syncthreads();
    const int half = (cnt + 1) >> 1;
    for (int p = tid; p < half; p += kRmThreads) {
        const bool has_b = p + half < cnt;
        decode_pair(mlp, rows + (size_t)p * kRow, rows + (size_t)(has_b ? p + half : p) * kRow, has_b);
    }
    __syncthreads();
    float* o = rgb + ((size_t)n * P + p0) * (kOut - 1);
    for (int i = tid; i < cnt * (kOut - 1); i += kRmThreads) o[i] = rows[(size_t)(i >> 5) * kRow + 1 + (i & 31)];
    for (int q = tid; q < cnt; q += kRmThreads) sigma[(size_t)n * P + p0 + q] = rows[(size_t)q * kRow];
}

}  // namespace r3dp

using namespace r3dp;

extern "C" int r3dp_grids_to_channels_last(const float* grids_nchw, int N, int C, int D, int H, int W, float* grids_cl, r3dp_stream_t stream) {
    R3DP_REQUIRE(grids_nchw && grids_cl, "grids_to_channels_last: null pointer");
    R3DP_REQUIRE(C == kC, "grids_to_channels_last: C must be %d (got %d)", kC, C);
    R3DP_REQUIRE(N > 0 && H > 0 && W > 0 && D >= 1 && (long long)N * 3 * D <= 65535, "grids_to_channels_last: bad shape");
    const int HW = H * W;
    dim3 grid((HW + kTilePx - 1) / kTilePx, N * 3 * D);
    planes_to_cl_kernel<<<grid, 256, 0, as_stream(stream)>>>(grids_nchw, grids_cl, HW, D);
    count_launches(1);
    R3DP_LAUNCH_CHECK();
    return 0;
}
extern "C" int r3dp_planes_to_channels_last(const float* planes_nchw, int N, int C, int H, int W, float* planes_cl,
                                            r3dp_stream_t stream) {
    return r3dp_grids_to_channels_last(planes_nchw, N, C, 1, H, W, planes_cl, stream);
}

extern "C" int r3dp_trigrid_sample(const float* grids_cl, int N, int C, int D, int H, int W, const float* coords, int P, float box_warp,
                                   float* out, r3dp_stream_t stream) {
    R3DP_REQUIRE(grids_cl && coords && out, "trigrid_sample: null pointer");
    R3DP_REQUIRE(C == kC && D >= 2 && N > 0 && P > 0 && H >= 2 && W >= 2 && box_warp > 0.f, "trigrid_sample: bad shape (C = 32, depth >= 2)");
    R3DP_REQUIRE((long long)3 * D * H * W * kC < (1ll << 31), "trigrid_sample: grids exceed the 32-bit texel offsets");
    const long long warps = ((long long)N * P + 3) / 4;
    const long long need = (warps + 7) / 8, cap = (long long)sm_count() * 3;
    trigrid_sample_kernel<<<(unsigned)(need < cap ? need : cap), 256, 0, as_stream(stream)>>>(grids_cl, N, D, H, W, coords, P, 2.0f / box_warp, out);
    count_launches(1);
    R3DP_LAUNCH_CHECK();
    return 0;
}

extern "C" int r3dp_triplane_sample(const float* planes_cl, int N, int C, int H, int W, const float* coords, int P,
                                    float box_warp, float* out, r3dp_stream_t stream) {
    R3DP_REQUIRE(planes_cl && coords && out, "triplane_sample: null pointer");
    R3DP_REQUIRE(C == kC, "triplane_sample: C must be %d (got %d)", kC, C);
    R3DP_REQUIRE(N > 0 && P > 0 && H > 0 && W > 0 && box_warp > 0.f, "triplane_sample: bad shape");
    const long long chunks = ((long long)N * P + 31) / 32;          // one warp-chunk = 32 consecutive points
    long long need = (chunks + 7) / 8;
    static int minb = -1;                          // R3DP_SAMPLE_MINB = 2 | 3 | 4 (register/occupancy trade-off: A/B knob)
    if (minb < 0) { const char* e = getenv("R3DP_SAMPLE_MINB"); minb = e ? atoi(e) : 3; if (minb < 2 || minb > 4) minb = 3; }
    const long long cap = (long long)sm_count() * minb;
    const unsigned blocks = (unsigned)(need < cap ? need : cap);
    const float sc = 2.0f / box_warp;
    cudaStream_t st = as_stream(stream);
    switch (minb) {
        case 2: triplane_sample_kernel<2><<<blocks, 256, 0, st>>>(planes_cl, N, H, W, coords, P, sc, out); break;
        case 4: triplane_sample_kernel<4><<<blocks, 256, 0, st>>>(planes_cl, N, H, W, coords, P, sc, out); break;
        default: triplane_sample_kernel<3><<<blocks, 256, 0, st>>>(planes_cl, N, H, W, coords, P, sc, out); break;
    }
    R3DP_LAUNCH_CHECK();
    return 0;
}

extern "C" int r3dp_run_model_grid(const float* planes_cl, int N, int C, int D, int H, int W, const float* coords, int P, float box_warp,
                                   const r3dp_mlp_t* mlp, float* rgb, float* sigma, r3dp_stream_t stream) {
    R3DP_REQUIRE(planes_cl && coords && rgb && sigma && mlp, "run_model: null pointer");
    R3DP_REQUIRE(mlp->in_features == kC && mlp->hidden == kHidden && mlp->out_dim == kOut - 1 && C == kC,
                 "run_model: only the OSGDecoder shape 32->64->1+32 is built");
    R3DP_REQUIRE(N > 0 && P > 0 && H >= 2 && W >= 2 && D >= 1 && box_warp > 0.f, "run_model: bad shape");
    R3DP_REQUIRE((long long)3 * D * H * W * kC < (1ll << 31), "run_model: planes exceed the 32-bit texel offsets");
    const size_t smem = sizeof(MlpSmem) + (size_t)kRmPoints * kRow * 4;
    R3DP_CUDA(cudaFuncSetAttribute(run_model_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    PlaneSet ps;
    ps.base = planes_cl; ps.depth = D; ps.slice_stride = H * W * kC; ps.plane_stride = D * H * W * kC; ps.frame_stride = 3ll * ps.plane_stride;
    ps.row_stride = W * kC; ps.texel_stride = kC;
    dim3 grid((P + kRmPoints - 1) / kRmPoints, N);
    run_model_kernel<<<grid, kRmThreads, smem, as_stream(stream)>>>(ps, N, H, W, coords, P, 2.0f / box_warp, *mlp, rgb, sigma);
    count_launches(1);
    R3DP_LAUNCH_CHECK();
    return 0;
}
extern "C" int r3dp_run_model(const float* planes_cl, int N, int C, int H, int W, const float* coords, int P, float box_warp,
                              const r3dp_mlp_t* mlp, float* rgb, float* sigma, r3dp_stream_t stream) {
    return r3dp_run_model_grid(planes_cl, N, C, 1, H, W, coords, P, box_warp, mlp, rgb, sigma, stream);
}

extern "C" int r3dp_decode(const float* feat, int N, int K, int P, int C, const r3dp_mlp_t* mlp, float* rgb, float* sigma,
                           r3dp_stream_t stream) {
    R3DP_REQUIRE(feat && rgb && sigma && mlp, "decode: null pointer");
    R3DP_REQUIRE(mlp->in_features == kC && mlp->hidden == kHidden && mlp->out_dim == kOut - 1 && C == kC,
                 "decode: only the OSGDecoder shape 32->64->1+32 is built");
    R3DP_REQUIRE(N > 0 && P > 0 && (K == 1 || K == 3), "decode: bad shape (K must be 1 or 3, got %d)", K);
    const size_t smem = sizeof(MlpSmem) + (size_t)kRmPoints * kRow * 4;
    R3DP_CUDA(cudaFuncSetAttribute(decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid((P + kRmPoints - 1) / kRmPoints, N);
    decode_kernel<<<grid, kRmThreads, smem, as_stream(stream)>>>(feat, K, P, *mlp, rgb, sigma);
    count_launches(1);
    R3DP_LAUNCH_CHECK();
    return 0;
}
