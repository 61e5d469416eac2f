// blink_eye_for_secc (inference/edit_secc.py) on sm_90a: closes the eye holes of SECC images in place.  The spec (DESIGN.md, "SECC blink"):
// quantise q = trunc(((x + 1) / 2) 255); face = every channel's q != 0; coarse = ~face inside the two prior eye regions; a box of the coarse rows
// and each eye's coarse columns, widened by 4 (half-open); er = face pixels of the box farther than 5 px from every coarse pixel; eye = box & ~er;
// per-column row statistics of eye give the thresholds p mean + (1 - p) min / max; eye pixels beyond them take the q of their nearest er pixel
// (ties to the lowest row-major index).  The output is q / 127.5 - 1 everywhere else.
//   blink_bounds_kernel   one CTA per image: the coarse row / column ranges over the prior rows, the fault test, and the per-call scratch reset
//   blink_classify_kernel 32 x 8 tiles of the widest possible box: er (compacted with its q) or eye (flagged, and counted into column stats)
//   blink_mark_kernel     one thread per pixel of the image: blinked eye pixels go to a list, every other pixel is written quantised
//   blink_fill_kernel     one warp per listed pixel: the exact nearest er pixel over the compacted list, its q written to all three channels
// Per image control: a double p, or (t, T) from an fp32 row (p = -4/T^2 t^2 + 4/T t in double, in Python's order).  Untouched images exit at
// the top of every CTA and are not written.  Images the reference would raise on are left as rendered and counted in *faults.
#include "common.cuh"

namespace r3dp {
namespace blink {

constexpr int kTileW = 32, kTileH = 8;       // classify tile
constexpr int kHalo = 5;                     // erosion radius: dy^2 + dx^2 <= 25
constexpr int kFillCtas = 32;                // fill CTAs per image (8 warps each, grid-stride over the blink list)
constexpr int kBig = 1 << 30;

// Per-image header (int32 words) at the start of each image's scratch.
enum { H_FAULT, H_MIN_H, H_MAX_H, H_LMIN, H_LMAX, H_RMIN, H_RMAX, H_NER, H_NBLINK, H_WORDS = 16 };

// Geometry of one call: the widest box is rows [S/4 - 4, S/2 + 4) x cols [S/4 - 4, (S/4) 3 + 4) (the "window").
struct Geo {
    int S, r0, c0, Hr, Wc;                  // window origin and extent
    size_t img_bytes;                       // scratch bytes per image
    size_t off_cols, off_eye, off_er, off_blink;
};

__host__ __device__ inline Geo geometry(int S) {
    Geo g;
    g.S = S;
    g.r0 = S / 4 - 4;
    g.c0 = S / 4 - 4;
    g.Hr = S / 2 - S / 4 + 8;
    g.Wc = (S / 4) * 3 - S / 4 + 8;
    const size_t area = (size_t)g.Hr * g.Wc;
    g.off_cols = H_WORDS * 4;                                       // n, sum, min, max per window column (int32)
    g.off_eye = g.off_cols + (size_t)16 * g.Wc;                     // eye flag per window pixel (uint8)
    g.off_er = (g.off_eye + area + 7) & ~(size_t)7;                 // er list: (r << 10 | c) << 24 | q (uint64)
    g.off_blink = g.off_er + 8 * area;                              // blink list: pixel index (uint32)
    g.img_bytes = (g.off_blink + 4 * area + 255) & ~(size_t)255;
    return g;
}

// The image's control: false when untouched; else p in double.
__device__ __forceinline__ bool control(const double* pv, const float* rows, int row_stride, int b, double& p) {
    if (pv) {
        p = pv[b];
        return p >= 0.0 && p <= 1.0;                                // negative (or NaN) = untouched
    }
    const float ft = rows[(size_t)b * row_stride], fT = rows[(size_t)b * row_stride + 1];
    if (!(fT > 0.f) || !(ft >= 0.f) || !(ft < fT) || fT > 4096.f) return false;
    const int t = (int)ft, T = (int)fT;                             // truncated, as int() does
    if (t >= T) return false;                                       // fractional rows: 0 < T < 1 (T = 0 after truncation), or int(t) = int(T)
    // real3d_infer.py's -4/T**2 * t**2 + 4/T * t: ((-4 / T^2) t^2) + ((4 / T) t), each step rounded once
    p = __dadd_rn(__dmul_rn(__ddiv_rn(-4.0, (double)(T * T)), (double)(t * t)), __dmul_rn(__ddiv_rn(4.0, (double)T), (double)t));
    return true;
}

__device__ __forceinline__ int quant(float x) {                    // ((x + 1) / 2) * 255 in fp32, truncated
    const float v = __fmul_rn(__fdiv_rn(__fadd_rn(x, 1.f), 2.f), 255.f);
    return (int)fminf(fmaxf(v, 0.f), 255.f);
}

__device__ __forceinline__ float dequant(int q) { return __fsub_rn(__fdiv_rn((float)q, 127.5f), 1.f); }

__device__ __forceinline__ bool is_face(const float* img, size_t SS, int i) {
    return quant(img[i]) != 0 && quant(img[SS + i]) != 0 && quant(img[2 * SS + i]) != 0;
}

__device__ __forceinline__ int* header(unsigned char* scratch, const Geo& g, int b) {
    return reinterpret_cast<int*>(scratch + (size_t)b * g.img_bytes);
}

__global__ void __launch_bounds__(512) blink_bounds_kernel(const float* __restrict__ secc, int S, const double* __restrict__ pv,
                                                           const float* __restrict__ rows, int row_stride, unsigned char* __restrict__ scratch,
                                                           int* __restrict__ faults) {
    const int b = blockIdx.x;
    double p;
    if (!control(pv, rows, row_stride, b, p) || p == 0.0) return;
    const Geo g = geometry(S);
    int* h = header(scratch, g, b);
    int* cols = reinterpret_cast<int*>(reinterpret_cast<unsigned char*>(h) + g.off_cols);
    for (int c = threadIdx.x; c < g.Wc; c += blockDim.x) {
        cols[4 * c] = 0; cols[4 * c + 1] = 0; cols[4 * c + 2] = kBig; cols[4 * c + 3] = -kBig;
    }
    const size_t SS = (size_t)S * S;
    const float* img = secc + (size_t)b * 3 * SS;
    const int ra = S / 4, rb = S / 2, ca = S / 4, cm = S / 2, cb = (S / 4) * 3, w = cb - ca;
    int mnh = kBig, mxh = -kBig, lmn = kBig, lmx = -kBig, rmn = kBig, rmx = -kBig;
    const int n = (rb - ra) * w;
#pragma unroll 4
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int r = ra + i / w, c = ca + i % w;
        if (!is_face(img, SS, r * S + c)) {
            mnh = min(mnh, r); mxh = max(mxh, r);
            if (c < cm) { lmn = min(lmn, c); lmx = max(lmx, c); }
            else { rmn = min(rmn, c); rmx = max(rmx, c); }
        }
    }
    __shared__ int s[6];
    if (threadIdx.x == 0) { s[0] = kBig; s[1] = -kBig; s[2] = kBig; s[3] = -kBig; s[4] = kBig; s[5] = -kBig; }
    __syncthreads();
    atomicMin(s + 0, mnh); atomicMax(s + 1, mxh); atomicMin(s + 2, lmn); atomicMax(s + 3, lmx); atomicMin(s + 4, rmn); atomicMax(s + 5, rmx);
    __syncthreads();
    if (threadIdx.x == 0) {
        // coarse empty, or either eye's half of it empty: the reference's min() of an empty array raises
        const bool fault = s[2] == kBig || s[4] == kBig;
        h[H_FAULT] = fault;
        h[H_MIN_H] = s[0]; h[H_MAX_H] = s[1]; h[H_LMIN] = s[2]; h[H_LMAX] = s[3]; h[H_RMIN] = s[4]; h[H_RMAX] = s[5];
        h[H_NER] = 0; h[H_NBLINK] = 0;
        if (fault) atomicAdd(faults, 1);
    }
}

// box: rows [min_h - 4, max_h + 4), columns [lmin - 4, lmax + 4) or [rmin - 4, rmax + 4)
__device__ __forceinline__ bool in_box(const int* h, int r, int c) {
    return r >= h[H_MIN_H] - 4 && r < h[H_MAX_H] + 4 &&
           ((c >= h[H_LMIN] - 4 && c < h[H_LMAX] + 4) || (c >= h[H_RMIN] - 4 && c < h[H_RMAX] + 4));
}

__global__ void __launch_bounds__(kTileW * kTileH) blink_classify_kernel(const float* __restrict__ secc, int S, const double* __restrict__ pv,
                                                                         const float* __restrict__ rows, int row_stride,
                                                                         unsigned char* __restrict__ scratch) {
    const int b = blockIdx.z;
    double p;
    if (!control(pv, rows, row_stride, b, p) || p == 0.0) return;
    const Geo g = geometry(S);
    int* h = header(scratch, g, b);
    if (h[H_FAULT]) return;
    const int tr0 = g.r0 + blockIdx.y * kTileH, tc0 = g.c0 + blockIdx.x * kTileW;
    // the tile against the box's bounding rectangle
    if (tr0 >= h[H_MAX_H] + 4 || tr0 + kTileH <= h[H_MIN_H] - 4 || tc0 >= h[H_RMAX] + 4 || tc0 + kTileW <= h[H_LMIN] - 4) return;
    const size_t SS = (size_t)S * S;
    const float* img = secc + (size_t)b * 3 * SS;
    // coarse flags of the tile and its 5-pixel halo (coarse lies in rows [S/4, S/2), columns [S/4, (S/4) 3))
    constexpr int TH = kTileH + 2 * kHalo, TW = kTileW + 2 * kHalo;
    __shared__ unsigned char s_coarse[TH][TW];
    const int ra = S / 4, rb = S / 2, ca = S / 4, cb = (S / 4) * 3;
    const int tid = threadIdx.y * kTileW + threadIdx.x;
    for (int i = tid; i < TH * TW; i += kTileW * kTileH) {
        const int r = tr0 - kHalo + i / TW, c = tc0 - kHalo + i % TW;
        s_coarse[i / TW][i % TW] = (r >= ra && r < rb && c >= ca && c < cb) ? !is_face(img, SS, r * S + c) : 0;
    }
    __syncthreads();
    const int r = tr0 + threadIdx.y, c = tc0 + threadIdx.x;
    if (r >= g.r0 + g.Hr || c >= g.c0 + g.Wc || !in_box(h, r, c)) return;
    const int i = r * S + c;
    const int q0 = quant(img[i]), q1 = quant(img[SS + i]), q2 = quant(img[2 * SS + i]);
    bool er = q0 != 0 && q1 != 0 && q2 != 0;                        // af = face & box
    if (er) {
        for (int dy = -kHalo; dy <= kHalo && er; ++dy)
            for (int dx = -kHalo; dx <= kHalo; ++dx)
                if (dy * dy + dx * dx <= kHalo * kHalo && s_coarse[threadIdx.y + kHalo + dy][threadIdx.x + kHalo + dx]) {
                    er = false;
                    break;
                }
    }
    unsigned char* base = reinterpret_cast<unsigned char*>(h);
    base[g.off_eye + (size_t)(r - g.r0) * g.Wc + (c - g.c0)] = !er;
    if (er) {
        const int k = atomicAdd(h + H_NER, 1);
        reinterpret_cast<unsigned long long*>(base + g.off_er)[k] =
            ((unsigned long long)((r << 10) | c) << 24) | (unsigned)((q0 << 16) | (q1 << 8) | q2);
    } else {
        int* col = reinterpret_cast<int*>(base + g.off_cols) + 4 * (c - g.c0);
        atomicAdd(col, 1);
        atomicAdd(col + 1, r);
        atomicMin(col + 2, r);
        atomicMax(col + 3, r);
    }
}

__global__ void __launch_bounds__(256) blink_mark_kernel(float* __restrict__ secc, int S, const double* __restrict__ pv,
                                                         const float* __restrict__ rows, int row_stride, unsigned char* __restrict__ scratch,
                                                         int* __restrict__ faults) {
    const int b = blockIdx.y;
    double p;
    if (!control(pv, rows, row_stride, b, p)) return;
    const Geo g = geometry(S);
    int* h = header(scratch, g, b);
    if (p != 0.0) {
        if (h[H_FAULT]) return;
        if (h[H_NER] == 0) {                                        // nothing left of the face around the eyes: the reference's fit() raises
            if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(faults, 1);
            return;
        }
    }
    const int SS = S * S;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= SS) return;
    float* img = secc + (size_t)b * 3 * SS;
    const int r = i / S, c = i % S;
    if (p != 0.0 && r >= g.r0 && r < g.r0 + g.Hr && in_box(h, r, c)) {
        const unsigned char* base = reinterpret_cast<const unsigned char*>(h);
        if (base[g.off_eye + (size_t)(r - g.r0) * g.Wc + (c - g.c0)]) {
            const int* col = reinterpret_cast<const int*>(base + g.off_cols) + 4 * (c - g.c0);
            const int n = col[0];                                   // >= 1: this pixel is an eye pixel of the column
            const double mean = __ddiv_rn((double)col[1], (double)n);
            // p mean + (1 - p) min and p mean + (1 - p) max: two products and an add, never fused
            const double pm = __dmul_rn(p, mean), q = __dsub_rn(1.0, p);
            const double lo = __dadd_rn(pm, __dmul_rn(q, (double)col[2]));
            const double hi = __dadd_rn(pm, __dmul_rn(q, (double)col[3]));
            if ((double)r <= lo || (double)r >= hi) {
                const int k = atomicAdd(h + H_NBLINK, 1);
                reinterpret_cast<unsigned*>(reinterpret_cast<unsigned char*>(h) + g.off_blink)[k] = (unsigned)i;
                return;                                             // written by blink_fill_kernel
            }
        }
    }
    img[i] = dequant(quant(img[i]));
    img[SS + i] = dequant(quant(img[SS + i]));
    img[2 * SS + i] = dequant(quant(img[2 * SS + i]));
}

__global__ void __launch_bounds__(256) blink_fill_kernel(float* __restrict__ secc, int S, const double* __restrict__ pv,
                                                         const float* __restrict__ rows, int row_stride,
                                                         const unsigned char* __restrict__ scratch) {
    const int b = blockIdx.y;
    double p;
    if (!control(pv, rows, row_stride, b, p) || p == 0.0) return;
    const Geo g = geometry(S);
    const int* h = reinterpret_cast<const int*>(scratch + (size_t)b * g.img_bytes);
    if (h[H_FAULT]) return;
    const int n_er = h[H_NER], n_blink = h[H_NBLINK];
    if (n_er == 0) return;
    const unsigned long long* er = reinterpret_cast<const unsigned long long*>(scratch + (size_t)b * g.img_bytes + g.off_er);
    const unsigned* bl = reinterpret_cast<const unsigned*>(scratch + (size_t)b * g.img_bytes + g.off_blink);
    const int lane = threadIdx.x & 31, warps = blockDim.x / 32;
    const int SS = S * S;
    float* img = secc + (size_t)b * 3 * SS;
    for (int k = blockIdx.x * warps + (threadIdx.x >> 5); k < n_blink; k += gridDim.x * warps) {
        const int i = (int)bl[k], r = i / S, c = i % S;
        // key = d^2 << 44 | (row << 10 | col) << 24 | q: the minimum is the nearest er pixel, ties to the lowest row-major index
        // (d^2 < 2^19 inside the window)
        unsigned long long best = ~0ull;
        for (int j = lane; j < n_er; j += 32) {
            const unsigned long long e = er[j];
            const int rc = (int)(e >> 24), dy = (rc >> 10) - r, dx = (rc & 1023) - c;
            const unsigned long long key = ((unsigned long long)(dy * dy + dx * dx) << 44) | e;
            best = key < best ? key : best;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
            best = other < best ? other : best;
        }
        if (lane == 0) {
            const unsigned q = (unsigned)(best & 0xffffffu);
            img[i] = dequant((int)(q >> 16));
            img[SS + i] = dequant((int)((q >> 8) & 255));
            img[2 * SS + i] = dequant((int)(q & 255));
        }
    }
}

}  // namespace blink
}  // namespace r3dp

using namespace r3dp;
using namespace r3dp::blink;

extern "C" size_t r3dp_secc_blink_scratch_bytes(int B, int S) {
    if (B <= 0 || S < 64 || S > 1024) return 0;
    return (size_t)B * geometry(S).img_bytes;
}

extern "C" int r3dp_secc_blink(float* secc, int B, int S, const double* p, const float* rows, int row_stride, void* scratch, int* faults,
                               r3dp_stream_t stream) {
    R3DP_REQUIRE(secc && scratch && faults, "secc_blink: null pointer");
    R3DP_REQUIRE((p != nullptr) != (rows != nullptr), "secc_blink: give exactly one of p and rows");
    R3DP_REQUIRE(B > 0 && B <= 65535 && S >= 64 && S <= 1024, "secc_blink: bad shape (64 <= S <= 1024)");
    R3DP_REQUIRE(!rows || row_stride >= 2, "secc_blink: bad row stride");
    R3DP_REQUIRE(((uintptr_t)scratch & 255) == 0, "secc_blink: scratch must be 256-byte aligned");
    const Geo g = geometry(S);
    cudaStream_t st = as_stream(stream);
    unsigned char* sc = reinterpret_cast<unsigned char*>(scratch);
    blink_bounds_kernel<<<B, 512, 0, st>>>(secc, S, p, rows, row_stride, sc, faults);
    R3DP_LAUNCH_CHECK();
    blink_classify_kernel<<<dim3((g.Wc + kTileW - 1) / kTileW, (g.Hr + kTileH - 1) / kTileH, B), dim3(kTileW, kTileH), 0, st>>>(
        secc, S, p, rows, row_stride, sc);
    R3DP_LAUNCH_CHECK();
    blink_mark_kernel<<<dim3((S * S + 255) / 256, B), 256, 0, st>>>(secc, S, p, rows, row_stride, sc, faults);
    R3DP_LAUNCH_CHECK();
    blink_fill_kernel<<<dim3(kFillCtas, B), 256, 0, st>>>(secc, S, p, rows, row_stride, sc);
    R3DP_LAUNCH_CHECK();
    count_launches(4);
    return 0;
}
