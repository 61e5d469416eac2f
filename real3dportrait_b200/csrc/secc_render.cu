// SECC_Renderer (deep_3drecon/secc_renderer.py) on sm_90a: the BFM face mesh from 3DMM coefficients, rasterised and shaded with the NCC code.
//   secc_vertices_kernel   shape = basis . [id | exp] + mean (bfm.py:102-115), pose v = R s + t (bfm.py:204-238, 260-270), to_camera z = 10 - z,
//                          the renderer's x negation (mesh_renderer.py:69-71), FoV projection -> (x_ndc, y_ndc, z_view, 0) per vertex.
//                          One warp per vertex holds its three basis rows in registers and loops over the frames of its block's frame
//                          chunk (blockIdx.y): the basis (61.7 MB for the BFM) is read from memory once per chunk.  A mesh with enough vertices
//                          to fill the GPU runs one chunk of every frame; a small one (the 68 key points of motion.py) splits the frames into
//                          chunks of whole 32-frame tiles, which computes every frame exactly as one chunk does.
//   secc_raster_kernel     one thread per (frame, face): pytorch3d's per-face culls, then every pixel centre of the face's bounding box; a covered
//                          centre does a 64-bit atomicMin of (bits of pz) << 32 | face into the frame's key buffer: nearest pz, ties to the lower face.
//   secc_resolve_kernel    one thread per pixel: decodes the key, recomputes the winner's corrected barycentrics, interpolates the NCC code
//                          -> secc = 2 mask sum_i w_i ncc_i - 1 (and the mask), and resets the key to empty for the next call.
// pytorch3d's rules (rasterize_meshes, blur 0, faces_per_pixel 1, perspective-correct, no culling / clipping) are restated in DESIGN.md.
#include "common.cuh"
#include <math.h>

namespace r3dp {
namespace secc {

constexpr int kMaxK = 256;                // id + exp coefficients per frame (the BFM has 80 + 64)
constexpr int kFrameTile = 32;            // frames whose coefficients sit in shared memory at once
constexpr int kVertWarps = 8;             // vertices per block of the vertex pass
constexpr int kMaxChunks = 3 * kMaxK / 4 / 32;      // float4 chunks of a vertex's three basis rows per lane
constexpr float kEps = 1e-8f;             // pytorch3d's kEpsilon
constexpr unsigned long long kEmpty = ~0ull;
constexpr float kInvPi = 0.318309886183790672f;

inline unsigned blocks(long long n, int t) { return (unsigned)((n + t - 1) / t); }

__global__ void __launch_bounds__(kVertWarps * 32) secc_vertices_kernel(const float* __restrict__ basis, const float* __restrict__ mean, int N,
                                                                        int n_id, int n_exp, const float* __restrict__ id, int ids,
                                                                        const float* __restrict__ exp, int exps, const float* __restrict__ euler,
                                                                        const float* __restrict__ trans, int B, int chunk, float cam_dist,
                                                                        float tan_half, float4* __restrict__ verts) {
    __shared__ __align__(16) float s_coef[kFrameTile * kMaxK];
    __shared__ float s_pose[kFrameTile * 12];                      // R row-major (9), t (3)
    const int K = n_id + n_exp, K4 = K / 4;
    const int lane = threadIdx.x & 31;
    const int v = blockIdx.x * kVertWarps + (threadIdx.x >> 5);
    const bool live = v < N;
    // this vertex's three basis rows (3K contiguous floats) in registers: chunk j = lane + 32 i covers row j / K4, coefficients 4 (j % K4) ..
    float4 bas[kMaxChunks];
#pragma unroll
    for (int i = 0; i < kMaxChunks; ++i) {
        const int j = lane + 32 * i;
        bas[i] = (live && j < 3 * K4) ? __ldg(reinterpret_cast<const float4*>(basis + (size_t)v * 3 * K) + j) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float m0 = 0.f, m1 = 0.f, m2 = 0.f;
    if (live) {
        m0 = mean[3 * v]; m1 = mean[3 * v + 1]; m2 = mean[3 * v + 2];
    }
    {                                                              // this block's chunk of frames (chunk: a multiple of kFrameTile)
        const int f0 = blockIdx.y * chunk;
        B = min(chunk, B - f0);
        id += (size_t)f0 * ids;
        exp += (size_t)f0 * exps;
        if (euler) euler += 3 * f0;
        if (trans) trans += 3 * f0;
        verts += (size_t)f0 * N;
    }
    for (int b0 = 0; b0 < B; b0 += kFrameTile) {
        const int nb = min(kFrameTile, B - b0);
        __syncthreads();                                           // the previous tile's coefficients are no longer read
        for (int i = threadIdx.x; i < nb * K; i += blockDim.x) {
            const int b = i / K, k = i % K;
            s_coef[b * K + k] = k < n_id ? id[(size_t)(b0 + b) * ids + k] : exp[(size_t)(b0 + b) * exps + (k - n_id)];
        }
        for (int b = threadIdx.x; b < nb; b += blockDim.x) {
            float sx = 0.f, cx = 1.f, sy = 0.f, cy = 1.f, sz = 0.f, cz = 1.f;
            if (euler) {                                           // sincospif: an exact argument reduction, no local-memory Payne-Hanek path
                sincospif(euler[(b0 + b) * 3 + 0] * kInvPi, &sx, &cx);
                sincospif(euler[(b0 + b) * 3 + 1] * kInvPi, &sy, &cy);
                sincospif(euler[(b0 + b) * 3 + 2] * kInvPi, &sz, &cz);
            }
            // R = Rz Ry Rx (bfm.py:214-238); the reference's rot is R^T applied to row vectors, i.e. v = R s
            float* r = s_pose + b * 12;
            r[0] = cz * cy; r[1] = cz * sy * sx - sz * cx; r[2] = cz * sy * cx + sz * sx;
            r[3] = sz * cy; r[4] = sz * sy * sx + cz * cx; r[5] = sz * sy * cx - cz * sx;
            r[6] = -sy;     r[7] = cy * sx;                r[8] = cy * cx;
            r[9] = trans ? trans[(b0 + b) * 3 + 0] : 0.f;
            r[10] = trans ? trans[(b0 + b) * 3 + 1] : 0.f;
            r[11] = trans ? trans[(b0 + b) * 3 + 2] : 0.f;
        }
        __syncthreads();
        if (!live) continue;
        float k0 = 0.f, k1 = 0.f, k2 = 0.f;                        // the dot products of frame b0 + (b & ~31) + lane, kept by that lane
        for (int b = 0; b < nb; ++b) {
            const float* c = s_coef + b * K;
            float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f;
#pragma unroll
            for (int i = 0; i < kMaxChunks; ++i) {
                const int j = lane + 32 * i;
                if (j < 3 * K4) {
                    const int row = j / K4, k = 4 * (j - row * K4);
                    const float4 cc = *reinterpret_cast<const float4*>(c + k);
                    float d = bas[i].x * cc.x;
                    d = fmaf(bas[i].y, cc.y, d);
                    d = fmaf(bas[i].z, cc.z, d);
                    d = fmaf(bas[i].w, cc.w, d);
                    acc0 += row == 0 ? d : 0.f;             // selects, not a dynamically indexed (local-memory) array
                    acc1 += row == 1 ? d : 0.f;
                    acc2 += row == 2 ? d : 0.f;
                }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                acc0 += __shfl_xor_sync(0xffffffffu, acc0, o);
                acc1 += __shfl_xor_sync(0xffffffffu, acc1, o);
                acc2 += __shfl_xor_sync(0xffffffffu, acc2, o);
            }
            if (lane == (b & 31)) {
                k0 = acc0; k1 = acc1; k2 = acc2;
            }
            // every 32 frames the lanes finish one frame each: pose, projection and the store run 32-wide, not on lane 0 alone
            if (((b & 31) == 31 || b == nb - 1) && lane <= (b & 31)) {
                const int fb = (b & ~31) + lane;
                const float* r = s_pose + fb * 12;
                const float s0 = k0 + m0, s1 = k1 + m1, s2 = k2 + m2;
                const float vx = fmaf(r[0], s0, fmaf(r[1], s1, fmaf(r[2], s2, r[9])));
                const float vy = fmaf(r[3], s0, fmaf(r[4], s1, fmaf(r[5], s2, r[10])));
                const float vz = fmaf(r[6], s0, fmaf(r[7], s1, fmaf(r[8], s2, r[11])));
                const float z = cam_dist - vz;                    // to_camera (bfm.py:241-243)
                const float zt = z * tan_half;
                // mesh_renderer.py negates x; FoVPerspectiveCameras: x_ndc = x / (z tan(fov/2)); the rasteriser keeps the view-space z
                verts[(size_t)(b0 + fb) * N + v] = make_float4(-vx / zt, vy / zt, z, 0.f);
            }
        }
    }
}

// pytorch3d EdgeFunctionForward(p, v0, v1)
__device__ __forceinline__ float edge_fn(float px, float py, float ax, float ay, float bx, float by) {
    return (px - ax) * (by - ay) - (py - ay) * (bx - ax);
}

// Corrected barycentrics of pixel centre (px, py) in the face (a, b, c); false when the centre is not strictly inside.
__device__ __forceinline__ bool bary(float px, float py, const float4& a, const float4& b, const float4& c, float& w0, float& w1, float& w2) {
    const float area = edge_fn(c.x, c.y, a.x, a.y, b.x, b.y) + kEps;              // BarycentricCoordsForward
    const float b0 = edge_fn(px, py, b.x, b.y, c.x, c.y) / area;
    const float b1 = edge_fn(px, py, c.x, c.y, a.x, a.y) / area;
    const float b2 = edge_fn(px, py, a.x, a.y, b.x, b.y) / area;
    const float t0 = b0 * b.z * c.z, t1 = a.z * b1 * c.z, t2 = a.z * b.z * b2;      // BarycentricPerspectiveCorrectionForward
    const float den = fmaxf(t0 + t1 + t2, kEps);
    w0 = t0 / den; w1 = t1 / den; w2 = t2 / den;
    return w0 > 0.f && w1 > 0.f && w2 > 0.f;
}

// pixel index -> NDC centre as pytorch3d computes it (PixToNonSquareNdc on the flipped index: +X left, +Y up)
__device__ __forceinline__ float pix_ndc(int i, int S) { return -1.0f + (2.0f * (float)(S - 1 - i) + 1.0f) / (float)S; }

__global__ void __launch_bounds__(256) secc_raster_kernel(const float4* __restrict__ verts, int N, const int* __restrict__ faces, int F, int B,
                                                          int S, unsigned long long* __restrict__ keys) {
    const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;        // B F < 2^31 (checked by the entry point): 32-bit division
    if (idx >= (unsigned)B * (unsigned)F) return;
    const int b = (int)(idx / (unsigned)F), f = (int)(idx % (unsigned)F);
    const float4* vb = verts + (size_t)b * N;
    const float4 a = vb[faces[3 * f]], bb = vb[faces[3 * f + 1]], c = vb[faces[3 * f + 2]];
    const float zmax = fmaxf(a.z, fmaxf(bb.z, c.z));
    const float A = edge_fn(a.x, a.y, bb.x, bb.y, c.x, c.y);                        // face_area
    if (zmax < 0.f || (A <= kEps && A >= -kEps)) return;
    const float xmin = fminf(a.x, fminf(bb.x, c.x)), xmax = fmaxf(a.x, fmaxf(bb.x, c.x));
    const float ymin = fminf(a.y, fminf(bb.y, c.y)), ymax = fmaxf(a.y, fmaxf(bb.y, c.y));
    if (!(xmax >= -1.5f && xmin <= 1.5f && ymax >= -1.5f && ymin <= 1.5f)) return;      // off screen (and NaN vertices)
    // candidate columns / rows from x = 1 - (2c+1)/S, widened by one: the exact test below decides
    const float hs = 0.5f * (float)S, lo = -2.f, hi = (float)S + 1.f;             // clamped before the int conversion
    const int c0 = max(0, (int)floorf(fminf(fmaxf(hs * (1.f - xmax) - 0.5f, lo), hi)) - 1);
    const int c1 = min(S - 1, (int)ceilf(fminf(fmaxf(hs * (1.f - xmin) - 0.5f, lo), hi)) + 1);
    const int r0 = max(0, (int)floorf(fminf(fmaxf(hs * (1.f - ymax) - 0.5f, lo), hi)) - 1);
    const int r1 = min(S - 1, (int)ceilf(fminf(fmaxf(hs * (1.f - ymin) - 0.5f, lo), hi)) + 1);
    unsigned long long* kb = keys + (size_t)b * S * S;
    for (int r = r0; r <= r1; ++r) {
        const float py = pix_ndc(r, S);
        if (py > ymax || py < ymin) continue;                                       // CheckPointOutsideBoundingBox
        for (int cc = c0; cc <= c1; ++cc) {
            const float px = pix_ndc(cc, S);
            if (px > xmax || px < xmin) continue;
            float w0, w1, w2;
            if (!bary(px, py, a, bb, c, w0, w1, w2)) continue;
            const float pz = w0 * a.z + w1 * bb.z + w2 * c.z;
            if (pz < 0.f) continue;
            const unsigned long long key = ((unsigned long long)(__float_as_uint(pz) & 0x7fffffffu) << 32) | (unsigned)f;   // -0 -> +0
            atomicMin(kb + (size_t)r * S + cc, key);
        }
    }
}

__global__ void __launch_bounds__(256) secc_resolve_kernel(const float4* __restrict__ verts, int N, const int* __restrict__ faces,
                                                           const float4* __restrict__ ncc, int B, int S, int drop_face0,
                                                           unsigned long long* __restrict__ keys, float* __restrict__ secc,
                                                           float* __restrict__ mask) {
    const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;        // B S^2 < 2^31 (checked by the entry point): 32-bit division
    const unsigned SS = (unsigned)S * (unsigned)S;
    if (idx >= (unsigned)B * SS) return;
    const int b = (int)(idx / SS);
    const unsigned p = idx - (unsigned)b * SS;
    const int r = (int)(p / (unsigned)S), cc = (int)(p % (unsigned)S);
    const unsigned long long key = keys[idx];
    keys[idx] = kEmpty;
    float o0 = -1.f, o1 = -1.f, o2 = -1.f, m = 0.f;
    const int f = (int)(unsigned)(key & 0xffffffffull);
    // pix_to_face > 0 on the packed face index (mesh_renderer.py:116): face 0 of image 0 of a call is background
    if (key != kEmpty && !(drop_face0 && b == 0 && f == 0)) {
        const float4* vb = verts + (size_t)b * N;
        const int i0 = faces[3 * f], i1 = faces[3 * f + 1], i2 = faces[3 * f + 2];
        float w0, w1, w2;
        bary(pix_ndc(cc, S), pix_ndc(r, S), vb[i0], vb[i1], vb[i2], w0, w1, w2);
        const float4 n0 = ncc[i0], n1 = ncc[i1], n2 = ncc[i2];
        // interpolate_face_attributes: sum_i w_i attr_i, then (x - 0.5) / 0.5
        o0 = 2.f * (w0 * n0.x + w1 * n1.x + w2 * n2.x) - 1.f;
        o1 = 2.f * (w0 * n0.y + w1 * n1.y + w2 * n2.y) - 1.f;
        o2 = 2.f * (w0 * n0.z + w1 * n1.z + w2 * n2.z) - 1.f;
        m = 1.f;
    }
    float* sb = secc + (size_t)b * 3 * SS + p;
    sb[0] = o0; sb[SS] = o1; sb[2 * SS] = o2;
    if (mask) mask[idx] = m;
}

}  // namespace secc
}  // namespace r3dp

using namespace r3dp;
using namespace r3dp::secc;

extern "C" int r3dp_secc_vertices(const float* basis, const float* mean, int N, int n_id, int n_exp, const float* id, int ids, const float* exp,
                                  int exps, const float* euler, const float* trans, int B, float cam_dist, float tan_half, float* verts,
                                  r3dp_stream_t stream) {
    R3DP_REQUIRE(basis && mean && id && exp && verts, "secc_vertices: null pointer");
    const int K = n_id + n_exp;
    R3DP_REQUIRE(N > 0 && B > 0 && n_id >= 0 && n_exp >= 0 && K > 0 && K % 4 == 0 && K <= kMaxK, "secc_vertices: bad shape (0 < id+exp <= %d, a multiple of 4)", kMaxK);
    R3DP_REQUIRE((ids >= n_id || ids == 0) && (exps >= n_exp || exps == 0), "secc_vertices: bad row strides");
    R3DP_REQUIRE(((uintptr_t)basis & 15) == 0 && ((uintptr_t)verts & 15) == 0, "secc_vertices: basis and verts must be 16-byte aligned");
    // fewer vertex blocks than two waves of the GPU: split the frames into chunks of whole tiles so the grid fills it
    const unsigned vb = blocks(N, kVertWarps);
    const int tiles = (B + kFrameTile - 1) / kFrameTile, want = 2 * sm_count();
    const int split = (int)vb >= want ? 1 : min(tiles, (want + (int)vb - 1) / (int)vb);
    const int chunk = (tiles + split - 1) / split * kFrameTile;
    const dim3 grid(vb, (unsigned)((B + chunk - 1) / chunk));
    secc_vertices_kernel<<<grid, kVertWarps * 32, 0, as_stream(stream)>>>(basis, mean, N, n_id, n_exp, id, ids, exp, exps, euler, trans, B, chunk,
                                                                         cam_dist, tan_half, reinterpret_cast<float4*>(verts));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_secc_raster(const float* verts, int N, const int* faces, int F, int B, int S, void* keys, r3dp_stream_t stream) {
    R3DP_REQUIRE(verts && faces && keys, "secc_raster: null pointer");
    R3DP_REQUIRE(N > 0 && F > 0 && B > 0 && S > 0 && S <= 4096, "secc_raster: bad shape");
    R3DP_REQUIRE((long long)B * F < (1ll << 31) && (long long)B * S * S < (1ll << 31), "secc_raster: B*F and B*S*S must be below 2^31");
    R3DP_REQUIRE(((uintptr_t)verts & 15) == 0 && ((uintptr_t)keys & 7) == 0, "secc_raster: misaligned buffer");
    secc_raster_kernel<<<blocks((long long)B * F, 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<const float4*>(verts), N, faces, F, B, S,
                                                                                     reinterpret_cast<unsigned long long*>(keys));
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_secc_resolve(const float* verts, int N, const int* faces, const float* ncc, int B, int S, int drop_face0, void* keys,
                                 float* secc, float* mask, r3dp_stream_t stream) {
    R3DP_REQUIRE(verts && faces && ncc && keys && secc, "secc_resolve: null pointer");
    R3DP_REQUIRE(N > 0 && B > 0 && S > 0 && S <= 4096, "secc_resolve: bad shape");
    R3DP_REQUIRE((long long)B * S * S < (1ll << 31), "secc_resolve: B*S*S must be below 2^31");
    R3DP_REQUIRE(((uintptr_t)verts & 15) == 0 && ((uintptr_t)ncc & 15) == 0 && ((uintptr_t)keys & 7) == 0, "secc_resolve: misaligned buffer");
    secc_resolve_kernel<<<blocks((long long)B * S * S, 256), 256, 0, as_stream(stream)>>>(
        reinterpret_cast<const float4*>(verts), N, faces, reinterpret_cast<const float4*>(ncc), B, S, drop_face0,
        reinterpret_cast<unsigned long long*>(keys), secc, mask);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}
