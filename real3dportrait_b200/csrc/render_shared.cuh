// Structures shared by the two fused-render translation units:
//   render.cu         entry points, limits / clamp kernels, the CTA-per-ray-tile kernel (two-pass importance renders, odd shapes)
//   render_stream.cu  the warp-specialised streaming kernel (single-pass renders: gather || wgmma decode || march overlap)
#pragma once
#include "render_core.cuh"
#include "tc_prims.cuh"

namespace r3dp {

// ---- tensor-core decoder operand image --------------------------------------------------------------------------------------------
// The OSG decoder is two GEMMs over the samples: [M x 32] x [32 x 64] -> softplus -> [M x 64] x [64 x 33].  They run on wgmma with
// fp16 operands and fp32 accumulation in registers; fp32 accuracy is kept by splitting every operand into two fp16 halves
// (v = hi + lo exactly to 2^-22 |v|) and summing the three significant partial products hi*hi + lo*hi + hi*lo (lo*lo ~ 2^-22 is dropped).
// Operand images (K-major, 128-byte swizzle: one 128 B row = 64 fp16, 8-row groups 1024 B apart):
//   A1 tile  128 samples x [x_hi(32) | x_lo(32)]             written by the gather
//   W1       64 hidden   x [w_hi(32) | w_lo(32)]             k-steps 0,1 = hi, 2,3 = lo
//   A2 tile  128 samples x [h_hi(64)] , [h_lo(64)]           two atoms, written by the layer-1 epilogue
//   W2       48 outputs  x [w_hi(64)] , [w_lo(64)]           two atoms, rows >= 33 are zero (N = 48: a multiple of 16)
struct alignas(16) MlpTcImage {
    uint8_t w1[kHidden * 128];
    uint8_t w2hi[48 * 128];
    uint8_t w2lo[48 * 128];
    float b1[kHidden];
    float b2[48];
};
static_assert(sizeof(MlpTcImage) == 8192 + 6144 + 6144 + 256 + 192, "MlpTcImage layout");

__device__ __forceinline__ uint32_t sw128_off(int row, int k) {                // byte offset of fp16 element (row, k) of a swizzled atom
    return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + ((((k >> 3) ^ (row & 7))) << 4) + (k & 7) * 2);
}

// ---- per-call workspace ---------------------------------------------------------------------------------------------------------------
// [RenderWs | MlpTcImage | MlpConst-free padding | limits float2[N*M]]: the decoder operand image lives in the CALLER's workspace, so two
// renders with different decoders on different streams never share state.
struct RenderWs {
    unsigned t0_min, t0_max;   // ordered-uint encoded floats over valid rays
    unsigned d_min, d_max;     // over every sample depth of the call
    unsigned n_valid;
    unsigned pad[3];
};
static_assert(sizeof(RenderWs) == 32, "ws header");
constexpr size_t kWsImageOff = 256;                                              // MlpTcImage (16-byte aligned)
constexpr size_t kWsLimitsOff = kWsImageOff + ((sizeof(MlpTcImage) + 255) / 256) * 256;

// channels-last plane addressing, strides in floats: texel (plane p, row y, col x) of frame n starts at
//   base + n*frame_stride + p*plane_stride + y*row_stride + x*texel_stride    and holds kC contiguous floats.
// [N,3,H,W,C]: plane = H*W*C, row = W*C, texel = C.   [N,H,W,3,C] (= torch channels_last of the producer's [N,3*C,H,W]): plane = C, row = W*3*C, texel = 3*C.
// Tri-grids (`triplane_feature_type: trigrid / trigrid_v2`, renderer.py:78-89): each plane is a stack of `depth` slices, slice d of plane p
// starts slice_stride floats further; depth <= 1 = plain tri-planes.
struct PlaneSet {
    const float* base;
    long long frame_stride;
    int plane_stride, row_stride, texel_stride;
    int depth, slice_stride;
};

struct RenderArgs {
    PlaneSet p0, p1;                    // p1.base == nullptr: single set; else both sets are sampled at the same points and added
    int N, H, W;
    const float* ray_o; const float* ray_d; const float* camera; int M, res;
    int S, S_imp; float box_warp; int white_back;
    const float* u_coarse; const float* u_fine;
    r3dp_mlp_t mlp;
    const MlpTcImage* image;            // tensor-core decoder operands (workspace)
    float* rgb; float* depth; float* wsum;
    const float2* limits; const uint8_t* valid; RenderWs* ws;
    int tiles_per_frame, tile_cols;     // ray tiling of the CTA-per-tile kernel (see ray_of)
    int lookahead;                      // frames of planes streamed DRAM -> L2 ahead of the gather (0 = off)
};

// DRAM -> L2 prefetch of one frame's planes: share `part` of `parts` (32 KB chunks, round-robin).  The gather is
// latency-bound - a warp iteration waits for the slowest of its 48 texel lines, and with cold planes one of them nearly always comes from
// DRAM.  The TMA unit streams the planes into L2 ahead of the demand loads, which then pay the L2 latency only.
__device__ __forceinline__ void prefetch_frame_l2(const PlaneSet& ps, int H, int W, int n, int part, int parts) {
    if (ps.base == nullptr || (ps.frame_stride == 0 && n > 0)) return;
    const long long span = (2ll * ps.plane_stride + (long long)(ps.depth > 1 ? ps.depth - 1 : 0) * ps.slice_stride + (long long)(H - 1) * ps.row_stride +
                            (long long)(W - 1) * ps.texel_stride + kC) * 4;          // bytes from the frame's first to its last texel
    const char* base = reinterpret_cast<const char*>(ps.base + (size_t)n * ps.frame_stride);
    constexpr long long kChunk = 32768;
    for (long long off = (long long)part * kChunk; off < span; off += (long long)parts * kChunk) {
        const long long left = span - off;
        const uint32_t bytes = (uint32_t)((left < kChunk ? left : kChunk) & ~15ll);
        if (bytes) asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(base + off), "r"(bytes) : "memory");
    }
}

__device__ __forceinline__ Ray fetch_ray(const float* __restrict__ ray_o, const float* __restrict__ ray_d,
                                         const float* __restrict__ camera, int res, int n, int M, int m) {
    if (ray_o != nullptr) {
        const float* o = ray_o + ((size_t)n * M + m) * 3; const float* d = ray_d + ((size_t)n * M + m) * 3;
        Ray r; r.ox = o[0]; r.oy = o[1]; r.oz = o[2]; r.dx = d[0]; r.dy = d[1]; r.dz = d[2];
        return r;
    }
    return make_ray(camera + n * 25, camera + n * 25 + 16, res, m);
}

// Descriptor of one bilinear tap quad with explicit strides: out[0] = float-punned offset (in floats, from the frame's base) of the
// 2x2 texel block (shifted inside the plane; outside taps get weight 0, see axis_taps), out[1..4] = weights.
__device__ __forceinline__ void tap_desc_s(float gu, float gv, int H, int W, int plane_off, int row_stride, int texel_stride, float* out) {
    const float px = ((gu + 1.0f) * (float)W - 1.0f) * 0.5f;      // align_corners=False
    const float py = ((gv + 1.0f) * (float)H - 1.0f) * 0.5f;
    int bx, by; float wxa, wxb, wya, wyb;
    axis_taps(px, W, bx, wxa, wxb);
    axis_taps(py, H, by, wya, wyb);
    out[0] = __int_as_float(plane_off + by * row_stride + bx * texel_stride);
    out[1] = wxa * wya; out[2] = wxb * wya; out[3] = wxa * wyb; out[4] = wxb * wyb;
}

// Tri-grid descriptor (sample_from_trigrids, renderer.py:78-89: 3-D grid_sample, zero padding, align_corners=False): out[0] = offset of the
// 2x2x2 texel block (shifted inside the grid), out[1..4] = weights of the four taps in slice z, out[5..8] = in slice z+1.  D >= 2.
__device__ __forceinline__ void tap_desc_grid(float gu, float gv, float gw, int H, int W, int D, int plane_off, int slice_stride, int row_stride,
                                              int texel_stride, float* out) {
    const float px = ((gu + 1.0f) * (float)W - 1.0f) * 0.5f;
    const float py = ((gv + 1.0f) * (float)H - 1.0f) * 0.5f;
    const float pz = ((gw + 1.0f) * (float)D - 1.0f) * 0.5f;
    int bx, by, bz; float wxa, wxb, wya, wyb, wza, wzb;
    axis_taps(px, W, bx, wxa, wxb);
    axis_taps(py, H, by, wya, wyb);
    axis_taps(pz, D, bz, wza, wzb);
    out[0] = __int_as_float(plane_off + bz * slice_stride + by * row_stride + bx * texel_stride);
    const float w00 = wxa * wya, w10 = wxb * wya, w01 = wxa * wyb, w11 = wxb * wyb;
    out[1] = w00 * wza; out[2] = w10 * wza; out[3] = w01 * wza; out[4] = w11 * wza;
    out[5] = w00 * wzb; out[6] = w10 * wzb; out[7] = w01 * wzb; out[8] = w11 * wzb;
}

// the three descriptors of one sample position: plane 0 <- (x, y | z), plane 1 <- (x, z | y), plane 2 <- (z, x | y)
// (generate_planes + project_onto_planes, renderer.py:30-63); 15 floats for tri-planes, 27 for tri-grids
__device__ __forceinline__ void sample_desc(const PlaneSet& ps, int H, int W, float gx, float gy, float gz, float* row) {
    if (ps.depth > 1) {
        tap_desc_grid(gx, gy, gz, H, W, ps.depth, 0, ps.slice_stride, ps.row_stride, ps.texel_stride, row);
        tap_desc_grid(gx, gz, gy, H, W, ps.depth, ps.plane_stride, ps.slice_stride, ps.row_stride, ps.texel_stride, row + 9);
        tap_desc_grid(gz, gx, gy, H, W, ps.depth, 2 * ps.plane_stride, ps.slice_stride, ps.row_stride, ps.texel_stride, row + 18);
    } else {
        tap_desc_s(gx, gy, H, W, 0, ps.row_stride, ps.texel_stride, row);
        tap_desc_s(gx, gz, H, W, ps.plane_stride, ps.row_stride, ps.texel_stride, row + 5);
        tap_desc_s(gz, gx, H, W, 2 * ps.plane_stride, ps.row_stride, ps.texel_stride, row + 10);
    }
}

// ---- 2 x fp32 arithmetic on value pairs and the decoder activations on top of it --------------------------------------------------------
__device__ __forceinline__ float2 pk_fma(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 pk_mul(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 pk_add(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float ex2_approx(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float lg2_approx(float x) { float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rcp_approx(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
// torch.nn.Softplus(beta=1) of two values in the overflow-free form max(x,0) + ln(1 + exp(-|x|)) (exact for every x, so the reference's
// threshold = 20 switch - where softplus(x) = x to 2e-9 - needs no branch): 2 x (FMUL, EX2, LG2, FMNMX) + FADD2 + FFMA2
__device__ __forceinline__ float2 softplus2(float2 x) {
    const float2 e = make_float2(ex2_approx(fabsf(x.x) * -1.4426950408889634f), ex2_approx(fabsf(x.y) * -1.4426950408889634f));
    const float2 u = pk_add(e, make_float2(1.0f, 1.0f));
    const float2 l = make_float2(lg2_approx(u.x), lg2_approx(u.y));
    return pk_fma(l, make_float2(0.6931471805599453f, 0.6931471805599453f), make_float2(fmaxf(x.x, 0.f), fmaxf(x.y, 0.f)));
}
// sigmoid(x) * 1.002 - 0.001 of two values (OSGDecoder, triplane.py:143): FMUL2, 2 x EX2, FADD2, 2 x RCP, FFMA2
__device__ __forceinline__ float2 sigmoid_scaled2(float2 x) {
    const float2 t = pk_mul(x, make_float2(-1.4426950408889634f, -1.4426950408889634f));
    const float2 u = pk_add(make_float2(ex2_approx(t.x), ex2_approx(t.y)), make_float2(1.0f, 1.0f));
    return pk_fma(make_float2(rcp_approx(u.x), rcp_approx(u.y)), make_float2(1.002f, 1.002f), make_float2(-0.001f, -0.001f));
}

// tri-plane descriptor in the split layout of the streaming kernel: row[0..2] = the three texel-block offsets, row[4 + 8p .. 11 + 8p] = the four
// weights of plane p, each stored TWICE (w0 w0 w1 w1 w2 w2 w3 w3) so that one LDS.128 yields two aligned (w,w) pairs for float2 FMAs
__device__ __forceinline__ void sample_desc_split(const PlaneSet& ps, int H, int W, float gx, float gy, float gz, float* row) {
    float t[5];
    tap_desc_s(gx, gy, H, W, 0, ps.row_stride, ps.texel_stride, t);
    row[0] = t[0];
    reinterpret_cast<float4*>(row)[1] = make_float4(t[1], t[1], t[2], t[2]); reinterpret_cast<float4*>(row)[2] = make_float4(t[3], t[3], t[4], t[4]);
    tap_desc_s(gx, gz, H, W, ps.plane_stride, ps.row_stride, ps.texel_stride, t);
    row[1] = t[0];
    reinterpret_cast<float4*>(row)[3] = make_float4(t[1], t[1], t[2], t[2]); reinterpret_cast<float4*>(row)[4] = make_float4(t[3], t[3], t[4], t[4]);
    tap_desc_s(gz, gx, H, W, 2 * ps.plane_stride, ps.row_stride, ps.texel_stride, t);
    row[2] = t[0];
    reinterpret_cast<float4*>(row)[5] = make_float4(t[1], t[1], t[2], t[2]); reinterpret_cast<float4*>(row)[6] = make_float4(t[3], t[3], t[4], t[4]);
}

// the twelve taps of one tri-plane sample with every load issued before the first use: `wrow` points at the 6 x float4 duplicated weights in shared memory
__device__ __forceinline__ void gather12(const float* __restrict__ base, int o0, int o1, int o2, int rs, int ts, int cq, const float4* wrow, float4& acc) {
    float4 t[12];
    {
        const float* b = base + o0 + cq * 4;
        t[0] = ldg_nc_f4(b); t[1] = ldg_nc_f4(b + ts); t[2] = ldg_nc_f4(b + rs); t[3] = ldg_nc_f4(b + rs + ts);
        b = base + o1 + cq * 4;
        t[4] = ldg_nc_f4(b); t[5] = ldg_nc_f4(b + ts); t[6] = ldg_nc_f4(b + rs); t[7] = ldg_nc_f4(b + rs + ts);
        b = base + o2 + cq * 4;
        t[8] = ldg_nc_f4(b); t[9] = ldg_nc_f4(b + ts); t[10] = ldg_nc_f4(b + rs); t[11] = ldg_nc_f4(b + rs + ts);
    }
    // scheduling fence: every value above is an operand of these (empty) statements, so no use can be hoisted above the last load
    asm volatile("" : "+f"(t[0].x), "+f"(t[0].y), "+f"(t[0].z), "+f"(t[0].w), "+f"(t[1].x), "+f"(t[1].y), "+f"(t[1].z), "+f"(t[1].w),
                      "+f"(t[2].x), "+f"(t[2].y), "+f"(t[2].z), "+f"(t[2].w), "+f"(t[3].x), "+f"(t[3].y), "+f"(t[3].z), "+f"(t[3].w));
    asm volatile("" : "+f"(t[4].x), "+f"(t[4].y), "+f"(t[4].z), "+f"(t[4].w), "+f"(t[5].x), "+f"(t[5].y), "+f"(t[5].z), "+f"(t[5].w),
                      "+f"(t[6].x), "+f"(t[6].y), "+f"(t[6].z), "+f"(t[6].w), "+f"(t[7].x), "+f"(t[7].y), "+f"(t[7].z), "+f"(t[7].w));
    asm volatile("" : "+f"(t[8].x), "+f"(t[8].y), "+f"(t[8].z), "+f"(t[8].w), "+f"(t[9].x), "+f"(t[9].y), "+f"(t[9].z), "+f"(t[9].w),
                      "+f"(t[10].x), "+f"(t[10].y), "+f"(t[10].z), "+f"(t[10].w), "+f"(t[11].x), "+f"(t[11].y), "+f"(t[11].z), "+f"(t[11].w));
    float2 lo = make_float2(acc.x, acc.y), hi = make_float2(acc.z, acc.w);       // channel pairs (0,1) and (2,3): 24 packed FMAs instead of 48 + 12
#pragma unroll
    for (int p = 0; p < 3; ++p) {
        const float4 wa = wrow[2 * p], wb = wrow[2 * p + 1];                   // (w0 w0 w1 w1), (w2 w2 w3 w3)
        lo = pk_fma(make_float2(t[4 * p].x, t[4 * p].y), make_float2(wa.x, wa.y), lo);         hi = pk_fma(make_float2(t[4 * p].z, t[4 * p].w), make_float2(wa.x, wa.y), hi);
        lo = pk_fma(make_float2(t[4 * p + 1].x, t[4 * p + 1].y), make_float2(wa.z, wa.w), lo); hi = pk_fma(make_float2(t[4 * p + 1].z, t[4 * p + 1].w), make_float2(wa.z, wa.w), hi);
        lo = pk_fma(make_float2(t[4 * p + 2].x, t[4 * p + 2].y), make_float2(wb.x, wb.y), lo); hi = pk_fma(make_float2(t[4 * p + 2].z, t[4 * p + 2].w), make_float2(wb.x, wb.y), hi);
        lo = pk_fma(make_float2(t[4 * p + 3].x, t[4 * p + 3].y), make_float2(wb.z, wb.w), lo); hi = pk_fma(make_float2(t[4 * p + 3].z, t[4 * p + 3].w), make_float2(wb.z, wb.w), hi);
    }
    acc = make_float4(lo.x, lo.y, hi.x, hi.y);
}

// gather of one sample by an 8-lane group (lane cq owns channels 4cq..4cq+3): SUM over the three planes of the (bi|tri)linear taps
// described by `d` (15 or 27 floats, already in registers), read from `base`.  GRID is a compile-time flag.
template <bool GRID>
__device__ __forceinline__ void gather_desc(const float* __restrict__ base, const float* d, int rs, int ts, int ss, int cq, float4& acc) {
    constexpr int kStep = GRID ? 9 : 5;
#pragma unroll
    for (int p = 0; p < 3; ++p) {
        const float* b = base + __float_as_int(d[kStep * p]) + cq * 4;
        const float4 t00 = ldg_nc_f4(b), t10 = ldg_nc_f4(b + ts), t01 = ldg_nc_f4(b + rs), t11 = ldg_nc_f4(b + rs + ts);
        const float w00 = d[kStep * p + 1], w10 = d[kStep * p + 2], w01 = d[kStep * p + 3], w11 = d[kStep * p + 4];
        acc.x += t00.x * w00 + t10.x * w10 + t01.x * w01 + t11.x * w11;
        acc.y += t00.y * w00 + t10.y * w10 + t01.y * w01 + t11.y * w11;
        acc.z += t00.z * w00 + t10.z * w10 + t01.z * w01 + t11.z * w11;
        acc.w += t00.w * w00 + t10.w * w10 + t01.w * w01 + t11.w * w11;
        if (GRID) {
            const float* c = b + ss;
            const float4 u00 = ldg_nc_f4(c), u10 = ldg_nc_f4(c + ts), u01 = ldg_nc_f4(c + rs), u11 = ldg_nc_f4(c + rs + ts);
            const float v00 = d[kStep * p + 5], v10 = d[kStep * p + 6], v01 = d[kStep * p + 7], v11 = d[kStep * p + 8];
            acc.x += u00.x * v00 + u10.x * v10 + u01.x * v01 + u11.x * v11;
            acc.y += u00.y * v00 + u10.y * v10 + u01.y * v01 + u11.y * v11;
            acc.z += u00.z * v00 + u10.z * v10 + u01.z * v01 + u11.z * v11;
            acc.w += u00.w * v00 + u10.w * v10 + u01.w * v01 + u11.w * v11;
        }
    }
}

// order-preserving key of a depth for the merge sort: NaN last (as torch.sort), -0 == +0
__device__ __forceinline__ unsigned sort_key(float d) {
    if (d != d) return 0xffffffffu;
    return f2ord(d == 0.f ? 0.f : d);
}

// render_stream.cu
extern int g_rs_chunk_log2;      // A/B knob (r3dp_set_option / R3DP_RS_D)
extern int g_rs_prefetch;        // frames of L2 look-ahead of the streaming kernel (r3dp_set_option / R3DP_RS_PREFETCH)
bool render_stream_fits(const RenderArgs& a);
int launch_render_stream(const RenderArgs& a, cudaStream_t st);
int render_lookahead();

}  // namespace r3dp
