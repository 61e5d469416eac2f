// The row LayerNorm shared by the SECC->plane / img2plane token paths (r3dp_sp_layernorm) and HuBERT (r3dp_hb_layernorm).
#pragma once
#include <cuda_fp16.h>
#include <math.h>

namespace r3dp {

// One warp per row; lane holds channels lane + 32 i, i < NV (8: C <= 256, 32: C <= 1024).  Two-pass statistics in fp32 (nn.LayerNorm:
// biased variance).  u = (v - mean) * rstd, then * g + b when g is given (g and b are given together), then exact GELU when `gelu`.
// Outputs (each may be null): xo [R][C] the pre-norm row v = x (+ t); yf rows of yfs floats; yh rows of yhs halves, fp16 of u, and with
// yhlo > 0 the split form: hi at column c, lo (u - hi) at column yhlo + c.  yf may be x itself (in place: each warp holds its whole row in
// registers before it writes), so it is not __restrict__.
template <int NV>
__global__ void __launch_bounds__(256) layernorm_rows_kernel(const float* x, const float* __restrict__ t, int R, int C, const float* __restrict__ g,
                                                             const float* __restrict__ b, float eps, float* xo, float* yf, int yfs,
                                                             __half* __restrict__ yh, int yhs, int yhlo, int gelu) {
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= R) return;
    const int nv = C / 32;
    float v[NV];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        if (i < nv) {
            const size_t o = (size_t)row * C + lane + 32 * i;
            v[i] = x[o] + (t ? t[o] : 0.f);
            s += v[i];
        }
    }
#pragma unroll
    for (int m = 16; m; m >>= 1) s += __shfl_xor_sync(0xffffffffu, s, m);
    const float mean = s / C;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i)
        if (i < nv) { const float d = v[i] - mean; q = fmaf(d, d, q); }
#pragma unroll
    for (int m = 16; m; m >>= 1) q += __shfl_xor_sync(0xffffffffu, q, m);
    const float rstd = rsqrtf(q / C + eps);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        if (i >= nv) break;
        const int c = lane + 32 * i;
        const size_t o = (size_t)row * C + c;
        if (xo) xo[o] = v[i];
        float u = g ? fmaf((v[i] - mean) * rstd, g[c], b[c]) : (v[i] - mean) * rstd;
        if (gelu) u = 0.5f * u * (1.f + erff(u * 0.70710678118654752f));
        if (yf) yf[(size_t)row * yfs + c] = u;
        if (yh) {
            const __half h = __float2half_rn(u);
            yh[(size_t)row * yhs + c] = h;
            if (yhlo) yh[(size_t)row * yhs + yhlo + c] = __float2half_rn(u - __half2float(h));
        }
    }
}

}  // namespace r3dp
