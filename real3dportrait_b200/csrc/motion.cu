// Clip motion on sm_90a: each frame's camera and the torso head's key points from the clip's pose and 3DMM coefficients (DESIGN.md, "Clip
// motion"; real3d_infer.py:271-321, 428-452).
//   motion_camera_kernel     one thread per frame: the frame's pose (mirror_index into the driving pose, z translation of frame 0, mapping to
//                            the source pose; fp32 as the reference), written out for the key-point pass, then the camera smoothed over the
//                            truncated 7-frame window (smooth_camera_sequence): the thread recomputes the raw camera of each of its <= 7
//                            neighbours from their poses, which costs less than a second launch and a [T,16] round trip through memory.
//                            Rotation mean = scipy's Rotation.mean: the eigenvector of the largest eigenvalue of sum q q^T (4x4 Jacobi, double).
//   motion_keypoints_kernel  one thread per (frame, key point): kp = clamp(-(x_ndc, y_ndc), -1, 1) of r3dp_secc_vertices' output at the key
//                            points (= the reference's (lm2d - 0.5) / 0.5), the 7-tap box filter over frames with the edge frames mirrored
//                            (smooth_features_xd), z = 0; kp_s unsmoothed.
//   motion_lm2d_kernel       lm2d = (1 - (x_ndc, y_ndc)) / 2, Face3DHelper.reconstruct_lm2d's image coordinates in [0, 1].
#include "common.cuh"
#include <math.h>

namespace r3dp {
namespace motion {

constexpr int kHalf = 3;                           // smooth_camera_sequence and smooth_features_xd with kernel_size 7
constexpr float kInvPi = 0.318309886183790672f;

inline unsigned blocks(long long n, int t) { return (unsigned)((n + t - 1) / t); }

// infer_utils.py:24-38: forward on even turns, reversed on odd turns
__device__ __forceinline__ int mirror_index(int i, int P) {
    const int turn = i / P, res = i - turn * P;
    return (turn & 1) ? P - res - 1 : res;
}

// real3d_infer.py:282-309 for frame i, in fp32 as the reference computes it: drv = the source pose for 'static' (P = 1)
__device__ __forceinline__ void frame_pose(int i, const float* src_e, const float* src_t, const float* drv_e, const float* drv_t, int P, int map,
                                           float e[3], float t[3]) {
    const int j = mirror_index(i, P);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        e[k] = drv_e[3 * j + k];
        t[k] = drv_t[3 * j + k];
    }
    t[2] = drv_t[2];                               // trans[:, -1] = trans[0, -1] (frame 0 is driving row mirror_index(0, P) = 0)
    if (map) {                                     // + (src - pose[0]), pose[0] taken after the z fix
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            e[k] = __fadd_rn(e[k], __fsub_rn(src_e[k], drv_e[k]));
            t[k] = __fadd_rn(t[k], __fsub_rn(src_t[k], drv_t[k]));
        }
    }
}

// get_eg3d_convention_camera_pose_intrinsic (convert_to_eg3d_convention.py:109-139): R = compute_rotation(euler) = (Rz Ry Rx)^T,
// c = 0.27 (-R (t - [0,0,10])) + [0, 0.006, 0.161], c2w rotation M = R diag(1,-1,-1).  R in fp32 from sincospif (no local-memory
// Payne-Hanek path), the rest in double.
__device__ __forceinline__ void raw_camera(const float e[3], const float t[3], double M[9], double c[3]) {
    float sx, cx, sy, cy, sz, cz;
    sincospif(e[0] * kInvPi, &sx, &cx);
    sincospif(e[1] * kInvPi, &sy, &cy);
    sincospif(e[2] * kInvPi, &sz, &cz);
    // r = Rz Ry Rx row-major (as secc_vertices_kernel); R = r^T
    const float r[9] = {cz * cy, cz * sy * sx - sz * cx, cz * sy * cx + sz * sx,
                        sz * cy, sz * sy * sx + cz * cx, sz * sy * cx - cz * sx,
                        -sy,     cy * sx,                cy * cx};
    const double d0 = t[0], d1 = t[1], d2 = (double)t[2] - 10.0;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const double R0 = r[0 * 3 + a], R1 = r[1 * 3 + a], R2 = r[2 * 3 + a];      // row a of R = column a of r
        c[a] = -(R0 * d0 + R1 * d1 + R2 * d2) * 0.27;
        M[3 * a + 0] = R0;
        M[3 * a + 1] = -R1;
        M[3 * a + 2] = -R2;
    }
    c[1] += 0.006;
    c[2] += 0.161;
}

// scipy's Rotation.from_matrix: (x, y, z, w) from the largest of the trace and the diagonal, normalised
__device__ __forceinline__ void quat_of(const double m[9], double q[4]) {
    const double tr = m[0] + m[4] + m[8];
    if (tr >= m[0] && tr >= m[4] && tr >= m[8]) {
        q[0] = m[7] - m[5]; q[1] = m[2] - m[6]; q[2] = m[3] - m[1]; q[3] = 1.0 + tr;
    } else if (m[0] >= m[4] && m[0] >= m[8]) {
        q[0] = 1.0 + 2.0 * m[0] - tr; q[1] = m[1] + m[3]; q[2] = m[2] + m[6]; q[3] = m[7] - m[5];
    } else if (m[4] >= m[8]) {
        q[0] = m[1] + m[3]; q[1] = 1.0 + 2.0 * m[4] - tr; q[2] = m[5] + m[7]; q[3] = m[2] - m[6];
    } else {
        q[0] = m[2] + m[6]; q[1] = m[5] + m[7]; q[2] = 1.0 + 2.0 * m[8] - tr; q[3] = m[3] - m[1];
    }
    const double n = rsqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
#pragma unroll
    for (int k = 0; k < 4; ++k) q[k] *= n;
}

// The unit eigenvector of the largest eigenvalue of the symmetric 4x4 a (cyclic Jacobi; a is destroyed).
__device__ void top_eigenvector(double a[4][4], double q[4]) {
    double v[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) v[i][j] = i == j ? 1.0 : 0.0;
    const double tr = a[0][0] + a[1][1] + a[2][2] + a[3][3];
    for (int sweep = 0; sweep < 16; ++sweep) {
        double off = 0.0;
#pragma unroll
        for (int p = 0; p < 3; ++p)
#pragma unroll
            for (int r = p + 1; r < 4; ++r) off += a[p][r] * a[p][r];
        if (off <= 1e-40 * tr * tr) break;
#pragma unroll
        for (int p = 0; p < 3; ++p) {
#pragma unroll
            for (int r = p + 1; r < 4; ++r) {
                const double apr = a[p][r];
                if (apr == 0.0) continue;
                // Numerical Recipes' rotation: t = sgn(theta) / (|theta| + sqrt(theta^2 + 1)), theta = (a_rr - a_pp) / (2 a_pr)
                const double theta = (a[r][r] - a[p][p]) / (2.0 * apr);
                const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = rsqrt(t * t + 1.0), s = t * c;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const double x = a[k][p], y = a[k][r];
                    a[k][p] = c * x - s * y;
                    a[k][r] = s * x + c * y;
                }
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const double x = a[p][k], y = a[r][k];
                    a[p][k] = c * x - s * y;
                    a[r][k] = s * x + c * y;
                }
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const double x = v[k][p], y = v[k][r];
                    v[k][p] = c * x - s * y;
                    v[k][r] = s * x + c * y;
                }
            }
        }
    }
    double top = a[0][0];                          // column selects, not a dynamically indexed (local-memory) array
#pragma unroll
    for (int k = 0; k < 4; ++k) q[k] = v[k][0];
#pragma unroll
    for (int j = 1; j < 4; ++j) {
        const bool better = a[j][j] > top;
        top = better ? a[j][j] : top;
#pragma unroll
        for (int k = 0; k < 4; ++k) q[k] = better ? v[k][j] : q[k];
    }
    double n = 0.0;
#pragma unroll
    for (int k = 0; k < 4; ++k) n += q[k] * q[k];
    n = rsqrt(n);
#pragma unroll
    for (int k = 0; k < 4; ++k) q[k] *= n;
}

__global__ void __launch_bounds__(128) motion_camera_kernel(const float* __restrict__ src_e, const float* __restrict__ src_t,
                                                            const float* __restrict__ drv_e, const float* __restrict__ drv_t, int P, int T,
                                                            int map, float* __restrict__ euler, float* __restrict__ trans,
                                                            float* __restrict__ cameras) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= T) return;
    float e[3], t[3];
    frame_pose(i, src_e, src_t, drv_e, drv_t, P, map, e, t);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        euler[3 * i + k] = e[k];
        trans[3 * i + k] = t[k];
    }
    // smooth_camera_sequence (infer_utils.py:40-69): window [max(0, i-3), min(T, i+4)); translation mean, Rotation.mean.  Its except branch
    // needs det <= 0, and these rotations have det +1, so it is not built.
    const int j0 = max(0, i - kHalf), j1 = min(T, i + kHalf + 1);
    double A[4][4] = {}, cs[3] = {0.0, 0.0, 0.0};
    for (int j = j0; j < j1; ++j) {
        float ej[3], tj[3];
        frame_pose(j, src_e, src_t, drv_e, drv_t, P, map, ej, tj);
        double M[9], c[3], q[4];
        raw_camera(ej, tj, M, c);
        quat_of(M, q);
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b) A[a][b] += q[a] * q[b];
#pragma unroll
        for (int k = 0; k < 3; ++k) cs[k] += c[k];
    }
    double q[4];
    top_eigenvector(A, q);
    const double x = q[0], y = q[1], z = q[2], w = q[3], n = (double)(j1 - j0);
    const double R[9] = {1.0 - 2.0 * (y * y + z * z), 2.0 * (x * y - z * w),       2.0 * (x * z + y * w),
                         2.0 * (x * y + z * w),       1.0 - 2.0 * (x * x + z * z), 2.0 * (y * z - x * w),
                         2.0 * (x * z - y * w),       2.0 * (y * z + x * w),       1.0 - 2.0 * (x * x + y * y)};
    float* o = cameras + (size_t)i * 25;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        o[4 * a + 0] = (float)R[3 * a + 0];
        o[4 * a + 1] = (float)R[3 * a + 1];
        o[4 * a + 2] = (float)R[3 * a + 2];
        o[4 * a + 3] = (float)(cs[a] / n);
    }
    o[12] = 0.f; o[13] = 0.f; o[14] = 0.f; o[15] = 1.f;
    // _fix_intrinsics (convert_to_eg3d_convention.py:8-27)
    const float f = (float)(2985.29 / 700.0);
    o[16] = f;   o[17] = 0.f; o[18] = 0.5f;
    o[19] = 0.f; o[20] = f;   o[21] = 0.5f;
    o[22] = 0.f; o[23] = 0.f; o[24] = 1.f;
}

// torch.clamp: NaN stays NaN
__device__ __forceinline__ float clamp1(float v) { return v != v ? v : fminf(fmaxf(v, -1.f), 1.f); }

__global__ void __launch_bounds__(256) motion_keypoints_kernel(const float4* __restrict__ verts_s, const float4* __restrict__ verts_d, int T, int K,
                                                               float* __restrict__ kp_s, float* __restrict__ kp_d) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;              // T K < 2^31 (checked by the entry point)
    if (idx >= (T + 1) * K) return;
    if (idx >= T * K) {                                                 // the source frame: clamped, not smoothed
        const int k = idx - T * K;
        const float4 v = verts_s[k];
        kp_s[3 * k + 0] = clamp1(-v.x);
        kp_s[3 * k + 1] = clamp1(-v.y);
        kp_s[3 * k + 2] = 0.f;
        return;
    }
    const int t = idx / K, k = idx - t * K;
    // smooth_features_xd (infer_utils.py:71-102): frames padded with the flipped first and last three (index -1 - i before 0, 2T - 1 - i
    // after T - 1), then a 7-tap box filter; summed in double, rounded once
    double sx = 0.0, sy = 0.0;
#pragma unroll
    for (int d = -kHalf; d <= kHalf; ++d) {
        int s = t + d;
        s = s < 0 ? -1 - s : (s >= T ? 2 * T - 1 - s : s);
        const float4 v = verts_d[(size_t)s * K + k];
        sx += (double)clamp1(-v.x);
        sy += (double)clamp1(-v.y);
    }
    float* o = kp_d + (size_t)idx * 3;
    o[0] = (float)(sx / (2 * kHalf + 1));
    o[1] = (float)(sy / (2 * kHalf + 1));
    o[2] = 0.f;
}

__global__ void __launch_bounds__(256) motion_lm2d_kernel(const float4* __restrict__ verts, long long n, float* __restrict__ lm2d) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 v = verts[i];
    // face_proj = f x / z + c, y flipped about 224, / 224: (1 - x_ndc) / 2 with x_ndc = -x / (z tan_half), tan_half = c / f
    lm2d[2 * i + 0] = 0.5f - 0.5f * v.x;
    lm2d[2 * i + 1] = 0.5f - 0.5f * v.y;
}

}  // namespace motion
}  // namespace r3dp

using namespace r3dp;
using namespace r3dp::motion;

extern "C" int r3dp_motion_camera(const float* src_euler, const float* src_trans, const float* drv_euler, const float* drv_trans, int P, int T,
                                  int map_to_init_pose, float* euler, float* trans, float* cameras, r3dp_stream_t stream) {
    R3DP_REQUIRE(src_euler && src_trans && drv_euler && drv_trans && euler && trans && cameras, "motion_camera: null pointer");
    R3DP_REQUIRE(P >= 1 && T >= 1, "motion_camera: need P >= 1 and T >= 1");
    motion_camera_kernel<<<blocks(T, 128), 128, 0, as_stream(stream)>>>(src_euler, src_trans, drv_euler, drv_trans, P, T, map_to_init_pose ? 1 : 0,
                                                                        euler, trans, cameras);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_motion_keypoints(const float* verts_s, const float* verts_d, int T, int K, float* kp_s, float* kp_d, r3dp_stream_t stream) {
    R3DP_REQUIRE(verts_s && verts_d && kp_s && kp_d, "motion_keypoints: null pointer");
    R3DP_REQUIRE(T >= 3 && K >= 1, "motion_keypoints: need T >= 3 (the 7-frame smoothing mirrors three frames at each end) and K >= 1");
    R3DP_REQUIRE((long long)(T + 1) * K < (1ll << 31), "motion_keypoints: (T + 1) K must be below 2^31");
    R3DP_REQUIRE(((uintptr_t)verts_s & 15) == 0 && ((uintptr_t)verts_d & 15) == 0, "motion_keypoints: verts must be 16-byte aligned");
    motion_keypoints_kernel<<<blocks((long long)(T + 1) * K, 256), 256, 0, as_stream(stream)>>>(
        reinterpret_cast<const float4*>(verts_s), reinterpret_cast<const float4*>(verts_d), T, K, kp_s, kp_d);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_motion_lm2d(const float* verts, long long n, float* lm2d, r3dp_stream_t stream) {
    R3DP_REQUIRE(verts && lm2d, "motion_lm2d: null pointer");
    R3DP_REQUIRE(n >= 1, "motion_lm2d: need n >= 1");
    R3DP_REQUIRE(((uintptr_t)verts & 15) == 0, "motion_lm2d: verts must be 16-byte aligned");
    motion_lm2d_kernel<<<blocks(n, 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<const float4*>(verts), n, lm2d);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}
