// 3DMM landmark fit on sm_90a (DESIGN.md, "3DMM fit"; data_gen/utils/process_{image,video}/fit_3dmm_landmark.py): one iteration of the
// reference's Adam loop is two launches.
//   fit_grad_kernel  grid (frame-tile CTAs, 8 key-point chunks of 64 points, the 468 padded to 512 with weight 0).  Each CTA keeps its
//                    chunk's basis [192 rows (x | y | z blocks), 144] in shared memory and walks frame tiles of 64:
//                      S = Q B^T      the chunk's key shapes, Q = [id | exp] [64,144] (stage 1: the mean shape, no GEMM)
//                      epilogue       rotate, translate, project, weighted residual against the landmarks, and the chain rule back to the
//                                     vertices: dS [64,192], and per frame the 3x3 dL/dR and dL/dtrans summed over the chunk's points
//                      dQ = dS B      the coefficient gradients: exp rows per (chunk, frame), the global id summed over the CTA's frames
//                    Each thread owns 8 frames x 2 key points (lanes l and l + 32 of a warp share the warp's 8 frames), so a key point's three
//                    coordinates sit in one thread.  The GEMMs are fp32 FMAs on the CUDA cores; the epilogue (pose, projection, residual,
//                    chain rule and the per-frame sums) runs in fp64, where the residual's cancellation against the landmark would otherwise
//                    cost most of fp32's digits.  The chunk partials are written, never accumulated with atomics, so a rerun is bit-identical.
//   fit_adam_kernel  one thread per parameter: the chunk partials summed in a fixed order (the id over every CTA too), the regulariser
//                    and Laplacian gradients (frames t - 2 .. t + 2 of the current parameters), and torch's Adam step into the other buffer
//                    of a ping-pong pair, each group with its own step counter.  The parameters and Adam's moments are fp64.
#include "common.cuh"
#include <math.h>

namespace r3dp {
namespace fit {

constexpr int kKp = 468, kChunk = 64, kChunks = 8, kRows = 3 * kChunk;
constexpr int kNid = 80, kNexp = 64, kNq = kNid + kNexp;
constexpr int kRowP = kNexp + 6;                   // per-frame parameters: exp 64, euler 3, trans 3
constexpr int kFrames = 64;                        // frames per tile
constexpr int kMaxCtas = 16;                       // frame-tile CTAs per chunk (one 167 KB CTA per SM: 8 x 16 of the H100's 132 SMs)
constexpr int kThreads = 256;
constexpr int kBS = kNq + 1;                       // basis row stride: lanes l and l + 32 read rows l, l + 32 at one k without bank conflicts
constexpr int kQS = kFrames + 4;                   // Q^T row stride (float4 reads of a warp's 8 frames)
constexpr int kDS = kFrames + 2;                   // dS^T row stride (float2 reads; 2-way conflicts on the epilogue's stores)
constexpr int kPart = 12;                          // per (chunk, frame): dL/dR (3x3, row-major) and dL/dtrans
constexpr float kFocal = 1015.f, kCenter = 112.f, kDistance = 10.f;

struct Smem {
    float B[kRows * kBS];
    union {
        float Qt[kNq * kQS];
        float dSt[kRows * kDS];
    } u;
    double pose[kFrames][12];                      // R = Rz Ry Rx row-major, trans
    float mean[kRows];
    float w[kChunk];
    double idred[kThreads / 32][kNid];
};

inline int grid_x(int T) { return std::min((T + kFrames - 1) / kFrames, kMaxCtas); }

template <typename F>
__device__ __forceinline__ void mat3_mul(const F a[9], const F b[9], F c[9]) {
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) c[3 * i + j] = a[3 * i] * b[j] + a[3 * i + 1] * b[3 + j] + a[3 * i + 2] * b[6 + j];
}

// compute_rotation's factors (bfm.py:204-238; the reference multiplies row vectors by their product's transpose): Rx, Ry, Rz and, for
// angle d >= 0, that factor's derivative in its place
__device__ __forceinline__ void rotation(const double e[3], double R[9], int d = -1) {
    double sx, cx, sy, cy, sz, cz;
    sincos(e[0], &sx, &cx);
    sincos(e[1], &sy, &cy);
    sincos(e[2], &sz, &cz);
    const double rx[9] = {1, 0, 0, 0, cx, -sx, 0, sx, cx}, drx[9] = {0, 0, 0, 0, -sx, -cx, 0, cx, -sx};
    const double ry[9] = {cy, 0, sy, 0, 1, 0, -sy, 0, cy}, dry[9] = {-sy, 0, cy, 0, 0, 0, -cy, 0, -sy};
    const double rz[9] = {cz, -sz, 0, sz, cz, 0, 0, 0, 1}, drz[9] = {-sz, -cz, 0, cz, -sz, 0, 0, 0, 0};
    double fx[9], fy[9], fz[9], t[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) {                  // selects, not a dynamically chosen (local-memory) array
        fx[i] = d == 0 ? drx[i] : rx[i];
        fy[i] = d == 1 ? dry[i] : ry[i];
        fz[i] = d == 2 ? drz[i] : rz[i];
    }
    mat3_mul(fz, fy, t);
    mat3_mul(t, fx, R);
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// x: the parameters [id 80 | per frame: exp 64, euler 3, trans 3].  lms [T, L, 2] mediapipe pixels (y down), H the image side, sf = H / 224
// as fp32 (the reference's y = H - y, then / sf).  gscale = 2 / (T 468 2): d mean(w r^2) / d proj = gscale w r.
template <bool kGemm>
__global__ void __launch_bounds__(kThreads, 1) fit_grad_kernel(const float* __restrict__ basis, const float* __restrict__ mean,
                                                               const float* __restrict__ weight, const float* __restrict__ lms, int T, int L,
                                                               float H, float sf, const double* __restrict__ x, float gscale,
                                                               double* __restrict__ part_frame, float* __restrict__ part_exp,
                                                               double* __restrict__ part_id) {
    extern __shared__ float4 smem_raw[];
    Smem& s = *reinterpret_cast<Smem*>(smem_raw);
    const int c = blockIdx.y, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (kGemm)
        for (int i = tid; i < kRows * kNq; i += kThreads) {
            const int r = i / kNq, k = i - r * kNq;
            s.B[r * kBS + k] = basis[(size_t)c * kRows * kNq + i];
        }
    for (int i = tid; i < kRows; i += kThreads) s.mean[i] = mean[c * kRows + i];
    if (tid < kChunk) s.w[tid] = weight[c * kChunk + tid];
    double idacc[3] = {0.0, 0.0, 0.0};             // dL/did[lane + 32 i] over this CTA's frames (k < 80), in fp64: a sum over the clip
    const int ntiles = (T + kFrames - 1) / kFrames;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int f0 = tile * kFrames;
        __syncthreads();                           // the previous tile's dS^T reads are done
        if (tid < kFrames) {
            const int f = f0 + tid;
            double e[3] = {0.0, 0.0, 0.0}, R[9];
            if (f < T) {
                const double* p = x + kNid + (size_t)f * kRowP + kNexp;
#pragma unroll
                for (int a = 0; a < 3; ++a) {
                    e[a] = p[a];
                    s.pose[tid][9 + a] = p[3 + a];
                }
            } else {
#pragma unroll
                for (int a = 0; a < 3; ++a) s.pose[tid][9 + a] = 0.0;
            }
            rotation(e, R);
#pragma unroll
            for (int a = 0; a < 9; ++a) s.pose[tid][a] = R[a];
        }
        float acc[8][2][3];
#pragma unroll
        for (int f = 0; f < 8; ++f)
#pragma unroll
            for (int j2 = 0; j2 < 2; ++j2)
#pragma unroll
                for (int a = 0; a < 3; ++a) acc[f][j2][a] = 0.f;
        if (kGemm) {
            for (int i = tid; i < kFrames * kNq; i += kThreads) {
                const int fl = i / kNq, k = i - fl * kNq, f = f0 + fl;
                float q = 0.f;
                if (f < T) q = (float)(k < kNid ? x[k] : x[kNid + (size_t)f * kRowP + (k - kNid)]);
                s.u.Qt[k * kQS + fl] = q;
            }
            __syncthreads();
            const float* qb = s.u.Qt + 8 * warp;
#pragma unroll 2
            for (int k = 0; k < kNq; ++k) {
                const float4 qa = *reinterpret_cast<const float4*>(qb + k * kQS), qc = *reinterpret_cast<const float4*>(qb + k * kQS + 4);
                const float q[8] = {qa.x, qa.y, qa.z, qa.w, qc.x, qc.y, qc.z, qc.w};
                float b[2][3];
#pragma unroll
                for (int j2 = 0; j2 < 2; ++j2)
#pragma unroll
                    for (int a = 0; a < 3; ++a) b[j2][a] = s.B[(a * kChunk + lane + 32 * j2) * kBS + k];
#pragma unroll
                for (int f = 0; f < 8; ++f)
#pragma unroll
                    for (int j2 = 0; j2 < 2; ++j2)
#pragma unroll
                        for (int a = 0; a < 3; ++a) acc[f][j2][a] = fmaf(q[f], b[j2][a], acc[f][j2][a]);
            }
        }
        __syncthreads();                           // Q^T reads are done (dS^T shares its memory); the poses are visible
        // ---- epilogue: projection, residual, chain rule --------------------------------------------------------------------------------
#pragma unroll
        for (int f = 0; f < 8; ++f) {
            const int fl = 8 * warp + f, frame = f0 + fl;
            double R[9], t[3];
#pragma unroll
            for (int a = 0; a < 9; ++a) R[a] = s.pose[fl][a];
#pragma unroll
            for (int a = 0; a < 3; ++a) t[a] = s.pose[fl][9 + a];
            double red[kPart];
#pragma unroll
            for (int i = 0; i < kPart; ++i) red[i] = 0.0;
#pragma unroll
            for (int j2 = 0; j2 < 2; ++j2) {
                const int j = lane + 32 * j2, kp = c * kChunk + j;
                double sh[3], dp[3] = {0.0, 0.0, 0.0};
#pragma unroll
                for (int a = 0; a < 3; ++a) sh[a] = (double)s.mean[a * kChunk + j] + (double)acc[f][j2][a];
                const float w = s.w[j];
                if (frame < T && w != 0.f) {
                    double p[3];
#pragma unroll
                    for (int a = 0; a < 3; ++a) p[a] = R[3 * a] * sh[0] + R[3 * a + 1] * sh[1] + R[3 * a + 2] * sh[2] + t[a];
                    const double inv = 1.0 / ((double)kDistance - p[2]);
                    const float2 lm = *reinterpret_cast<const float2*>(lms + ((size_t)frame * L + kp) * 2);
                    const double ru = ((double)kFocal * p[0] * inv + kCenter) - (double)__fdiv_rn(lm.x, sf);
                    const double rv = ((double)kFocal * p[1] * inv + kCenter) - (double)__fdiv_rn(__fsub_rn(H, lm.y), sf);
                    dp[0] = gscale * w * ru * kFocal * inv;
                    dp[1] = gscale * w * rv * kFocal * inv;
                    dp[2] = (dp[0] * p[0] + dp[1] * p[1]) * inv;
                }
#pragma unroll
                for (int a = 0; a < 3; ++a) {
#pragma unroll
                    for (int b = 0; b < 3; ++b) red[3 * a + b] = fma(dp[a], sh[b], red[3 * a + b]);
                    red[9 + a] += dp[a];
                }
#pragma unroll
                for (int b = 0; b < 3; ++b) s.u.dSt[(b * kChunk + j) * kDS + fl] = (float)(R[b] * dp[0] + R[3 + b] * dp[1] + R[6 + b] * dp[2]);
            }
#pragma unroll
            for (int i = 0; i < kPart; ++i) red[i] = warp_sum(red[i]);
            if (lane < kPart && frame < T) {
                double v = red[0];
#pragma unroll
                for (int i = 1; i < kPart; ++i) v = lane == i ? red[i] : v;
                part_frame[((size_t)c * T + frame) * kPart + lane] = v;
            }
        }
        if (kGemm) {
        __syncthreads();
        // ---- dQ = dS B: lane owns k = lane + 32 i ----------------------------------------------------------------------------------------
        float acc2[8][5];
#pragma unroll
        for (int f = 0; f < 8; ++f)
#pragma unroll
            for (int i = 0; i < 5; ++i) acc2[f][i] = 0.f;
        const float* db = s.u.dSt + 8 * warp;
#pragma unroll 2
        for (int r = 0; r < kRows; ++r) {
            float d[8];
#pragma unroll
            for (int h = 0; h < 4; ++h) {
                const float2 v = *reinterpret_cast<const float2*>(db + r * kDS + 2 * h);
                d[2 * h] = v.x;
                d[2 * h + 1] = v.y;
            }
            float b[5];
#pragma unroll
            for (int i = 0; i < 5; ++i) b[i] = (i < 4 || lane < 16) ? s.B[r * kBS + lane + 32 * i] : 0.f;
#pragma unroll
            for (int f = 0; f < 8; ++f)
#pragma unroll
                for (int i = 0; i < 5; ++i) acc2[f][i] = fmaf(d[f], b[i], acc2[f][i]);
        }
#pragma unroll
        for (int i = 0; i < 5; ++i) {
            const int k = lane + 32 * i;
            if (k < kNid) {
#pragma unroll
                for (int f = 0; f < 8; ++f) idacc[i < 3 ? i : 0] += acc2[f][i];
            } else if (k < kNq) {
#pragma unroll
                for (int f = 0; f < 8; ++f) {
                    const int frame = f0 + 8 * warp + f;
                    if (frame < T) part_exp[((size_t)c * T + frame) * kNexp + (k - kNid)] = acc2[f][i];
                }
            }
        }
        }
    }
    if (!kGemm) return;
#pragma unroll
    for (int i = 0; i < 3; ++i)
        if (lane + 32 * i < kNid) s.idred[warp][lane + 32 * i] = idacc[i];
    __syncthreads();
    if (tid < kNid) {
        double v = 0.0;
#pragma unroll
        for (int w = 0; w < kThreads / 32; ++w) v += s.idred[w][tid];
        part_id[((size_t)c * gridDim.x + blockIdx.x) * kNid + tid] = v;
    }
}

struct AdamArgs {
    double step_frame, bc2_frame, step_idexp, bc2_idexp;   // step sizes lr / (1 - 0.9^t) and sqrt(1 - 0.999^t) per group (t = 0: frozen)
    double lam_id, lam_exp, lam_lap;
};

// cal_lap_loss's gradient at frame t of a column of C values with row stride ld over T frames (x[-1] = x[0], x[T] = x[T-1]), before the
// 2 / (C T) factor
__device__ __forceinline__ double lap_grad(const double* x, int ld, int t, int T) {
    auto at = [&](int i) { return x[(size_t)min(max(i, 0), T - 1) * ld]; };
    auto o = [&](int i) { return at(i) - 0.5 * (at(i - 1) + at(i + 1)); };
    double g = o(t);
    if (t + 1 <= T - 1) g -= 0.5 * o(t + 1);
    if (t == 0) g -= 0.5 * o(0);
    if (t >= 1) g -= 0.5 * o(t - 1);
    if (t == T - 1) g -= 0.5 * o(T - 1);
    return g;
}

// torch.optim.Adam (betas 0.9, 0.999, eps 1e-8): m.lerp_(g, 0.1), v = 0.999 v + 0.001 g^2, p += -step_size m / (sqrt(v) / bc2 + eps)
__device__ __forceinline__ double adam(double p, double g, double* m, double* v, double step_size, double bc2) {
    const double mm = *m + 0.1 * (g - *m);
    const double vv = *v * 0.999 + g * g * 0.001;
    *m = mm;
    *v = vv;
    return p - step_size * (mm / (sqrt(vv) / bc2 + 1e-8));
}

// The parameters, Adam's moments and this step are fp64: near convergence the loop amplifies any per-step perturbation by orders of
// magnitude (DESIGN.md, "3DMM fit"), and fp32 storage of the parameters would be the largest such perturbation.
__global__ void __launch_bounds__(256) fit_adam_kernel(const double* __restrict__ part_frame, const float* __restrict__ part_exp,
                                                       const double* __restrict__ part_id, int T, int nb, AdamArgs a,
                                                       const double* __restrict__ x, double* __restrict__ xn, double* __restrict__ m,
                                                       double* __restrict__ v, double* __restrict__ grad) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= kNid + (long long)T * kRowP) return;
    const bool stage2 = a.step_idexp > 0.0;
    double g, step_size = a.step_frame, bc2 = a.bc2_frame;
    if (idx < kNid) {
        if (!stage2) {
            xn[idx] = x[idx];
            return;
        }
        g = 0.0;
        for (int c = 0; c < kChunks; ++c)
            for (int b = 0; b < nb; ++b) g += part_id[((size_t)c * nb + b) * kNid + idx];
        g += (2.0 * a.lam_id / kNid) * x[idx];
        step_size = a.step_idexp;
        bc2 = a.bc2_idexp;
    } else {
        const int t = (int)((idx - kNid) / kRowP), j = (int)((idx - kNid) - (long long)t * kRowP);
        const double* col = x + kNid + j;
        if (j < kNexp) {
            if (!stage2) {
                xn[idx] = x[idx];
                return;
            }
            g = 0.0;
            for (int c = 0; c < kChunks; ++c) g += part_exp[((size_t)c * T + t) * kNexp + j];
            g += (2.0 * a.lam_exp / ((double)kNexp * T)) * x[idx];
            if (a.lam_lap != 0.0) g += (2.0 * a.lam_lap / ((double)kNexp * T)) * lap_grad(col, kRowP, t, T);
            step_size = a.step_idexp;
            bc2 = a.bc2_idexp;
        } else {
            double G[kPart];
#pragma unroll
            for (int i = 0; i < kPart; ++i) G[i] = 0.0;
            for (int c = 0; c < kChunks; ++c) {
                const double* p = part_frame + ((size_t)c * T + t) * kPart;
#pragma unroll
                for (int i = 0; i < kPart; ++i) G[i] += p[i];
            }
            if (j < kNexp + 3) {                   // euler: sum over dL/dR * dR/de
                const double* e = x + kNid + (size_t)t * kRowP + kNexp;
                const double ee[3] = {e[0], e[1], e[2]};
                double dR[9];
                rotation(ee, dR, j - kNexp);
                g = 0.0;
#pragma unroll
                for (int i = 0; i < 9; ++i) g = fma(G[i], dR[i], g);
            } else {
                g = G[9 + j - kNexp - 3];
            }
            if (stage2 && a.lam_lap != 0.0) g += (2.0 * 0.3 * a.lam_lap / (3.0 * T)) * lap_grad(col, kRowP, t, T);
        }
    }
    if (grad) grad[idx] = g;
    xn[idx] = adam(x[idx], g, m + idx, v + idx, step_size, bc2);
}

}  // namespace fit
}  // namespace r3dp

using namespace r3dp;
using namespace r3dp::fit;

extern "C" int r3dp_fit_grad(const float* basis, const float* mean, const float* weight, const float* lms, int T, int L, int img_size,
                             const double* x, int stage, double* part_frame, float* part_exp, double* part_id, r3dp_stream_t stream) {
    R3DP_REQUIRE(mean && weight && lms && x && part_frame, "fit_grad: null pointer");
    R3DP_REQUIRE(stage == 1 || (stage == 2 && basis && part_exp && part_id), "fit_grad: stage 1, or stage 2 with basis, part_exp and part_id");
    R3DP_REQUIRE(T >= 1 && L >= kKp && img_size >= 1, "fit_grad: need T >= 1, at least 468 landmarks per frame and img_size >= 1");
    R3DP_REQUIRE(((uintptr_t)lms & 7) == 0, "fit_grad: lms must be 8-byte aligned");
    const int smem = (int)sizeof(Smem);
    const dim3 grid(grid_x(T), kChunks);
    const float sf = (float)(img_size / (2.0 * kCenter)), gscale = (float)(2.0 / ((double)T * kKp * 2));
    if (stage == 2) {
        R3DP_CUDA(cudaFuncSetAttribute(fit_grad_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        fit_grad_kernel<true><<<grid, kThreads, smem, as_stream(stream)>>>(basis, mean, weight, lms, T, L, (float)img_size, sf, x, gscale,
                                                                           part_frame, part_exp, part_id);
    } else {
        R3DP_CUDA(cudaFuncSetAttribute(fit_grad_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        fit_grad_kernel<false><<<grid, kThreads, smem, as_stream(stream)>>>(basis, mean, weight, lms, T, L, (float)img_size, sf, x, gscale,
                                                                            part_frame, part_exp, part_id);
    }
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}

extern "C" int r3dp_fit_adam(const double* part_frame, const float* part_exp, const double* part_id, int T, int step_frame, int step_idexp,
                             double lr, double lam_id, double lam_exp, double lam_lap, const double* x, double* x_next, double* m,
                             double* v, double* grad, r3dp_stream_t stream) {
    R3DP_REQUIRE(part_frame && x && x_next && m && v && x != x_next, "fit_adam: null pointer, or x_next aliases x");
    R3DP_REQUIRE(T >= 1 && step_frame >= 1 && step_idexp >= 0, "fit_adam: need T >= 1, step_frame >= 1 and step_idexp >= 0");
    R3DP_REQUIRE(step_idexp == 0 || (part_exp && part_id), "fit_adam: stage 2 needs part_exp and part_id");
    AdamArgs a;
    auto sizes = [](int t, double lr_, double& step_size, double& bc2) {
        step_size = t ? lr_ / (1.0 - pow(0.9, t)) : 0.0;
        bc2 = t ? sqrt(1.0 - pow(0.999, t)) : 1.0;
    };
    sizes(step_frame, lr, a.step_frame, a.bc2_frame);
    sizes(step_idexp, lr, a.step_idexp, a.bc2_idexp);
    a.lam_id = lam_id;
    a.lam_exp = lam_exp;
    a.lam_lap = lam_lap;
    const long long n = kNid + (long long)T * kRowP;
    fit_adam_kernel<<<(unsigned)((n + 255) / 256), 256, 0, as_stream(stream)>>>(part_frame, part_exp, part_id, T, grid_x(T), a, x, x_next, m, v,
                                                                               grad);
    R3DP_LAUNCH_CHECK();
    count_launches(1);
    return 0;
}
