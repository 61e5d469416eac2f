"""Float64 references and element-wise error bounds for the torso head's fusion, gating and resampling kernels (csrc/sr_tc.cu), for
tests/test_gpu_torso_fusion_conformance.py.  Test infrastructure: it does not import the library, so it also runs on a machine without a
GPU (tests/test_cpu_torso_fusion_reference.py shows there that each bar passes a float32 simulation of its kernel and fails its mutants).

Every reference is computed from the operands the kernel reads, converted exactly to float64 (hi + lo for split [hi | lo] tensors), and
every bound is sr_conv_reference.check_bound's  |got - ref| <= alpha |ref| + extra + beta S,  S the same operation on absolute values.
Here no alpha, extra or beta is measured: the kernels are short chains of fp32 operations, so each term is derived from the arithmetic.
u = 2^-24 is the unit roundoff of fp32; the library is built without --use_fast_math, so divisions are correctly rounded, expf is the
libdevice one (at most 2 ulp = 4u relative, CUDA C Programming Guide, table of single-precision functions) and subnormals are kept.

  * alpha_cat, fp16 (`tc`):  fp16(x * m), m = alpha or fl(1 - alpha).  fl(1 - alpha) is within u, the product rounds once (u), the fp16
    store rounds once (2^-11, or 2^-25 absolute for subnormal results).  There is no add, so the result is (x.float() * m).half() of torch
    fp32 bit for bit, and against float64:  alpha = 2^-11 + 2^-22 (>= (1 + u)^2 (1 + 2^-11) - 1), extra = FLOOR_F16.
  * alpha_cat, split (`tcx`):  fl(hi + lo) (u), fl(1 - alpha) (u), the product (u), then the [hi | lo] store (2^-22, sr_conv_reference):
    alpha = 2^-22 + 4u = 2^-21 (>= (1 + u)^3 (1 + 2^-22) - 1), extra = FLOOR_F16.
  * alpha_mix / blend:  a * alpha + b * fl(1 - alpha) with S = |a| alpha + |b| (1 - alpha), alpha in [0, 1].  Whether nvcc contracts
    either product into an fma or not, the b term carries at most two roundings (1 - alpha and its product), the a term one, the sum one:
    <= 3u S in fp32.  The fp32 blend stores that value: beta = 4u, alpha = 0.  alpha_mix `tc` adds the fp16 store of a value within 3u S of
    ref: 2^-11 |ref| + 3u (1 + 2^-11) S, so alpha = ALPHA_F16, beta = 4u, extra = FLOOR_F16.  Split operands add fl(hi + lo) to each term
    (<= 4u S in fp32) and the split store: alpha = ALPHA_SPLIT, beta = 5u, extra = FLOOR_F16.
  * alpha_gate:  s' = fl(1 / fl(1 + expf(-v'))), v' = fl(hi + lo) (v' = hi when lo_off = 0).  With E = exp(-v) and r = E / (1 + E) = 1 - s,
    expf's 4u relative error moves 1 + E by at most 4u r (1 + E), the add and the division round once each: s' = s(v') (1 + d) with
    |d| <= (2 + 4r) u + O(u^2) <= 6u: beta = 7u on S = sigmoid(v) (three ulps of the result).  The rounding of hi + lo moves v by at most
    u |v|, and sigmoid' = s (1 - s) changes by a factor <= exp(u |v|) < 1.01 over that step: extra = 1.01 u |v| s (1 - s) when lo_off > 0.
    Results below 2^-126 (v < -87.3) are fp32 subnormals or flush to 0 when expf overflows: extra also holds 2^-126 absolute.  The cap is
    a min: |min(a, c) - min(b, c)| <= |a - b|, so the same bound holds for the capped value.
  * person_occlusion:  clamp(torso + (w > thr ? 1 : w), 0, 1): one comparison, one add, a clamp, all in fp32 - bit equality with the
    torch fp32 restatement (person_occlusion_f32).  thr is the fp32 value the C ABI receives, and torch compares an fp32 tensor with a
    Python float in fp32 as well (the reference's alpha > thr), so both sides decide on the same fp32 threshold.
  * resize_aa_down2:  the separable filter matrix of aa_down2_matrix ([1,3,3,1] / 8 inside, [3,3,1] / 7 and [1,3,3] / 7 at the borders,
    [1,1] / 2 when the output side is 1).  Each of the <= 16 products of an output passes through at most 10 fp32 roundings: its column
    weight wx / sx (1), the 4-fma row chain (<= 4), its row weight wy / sy (1), the 4-fma column chain (<= 4): beta = gamma_10, alpha = 0.
  * warp_input:  bilinear resizes (align_corners=False) at sizes whose source coordinates are exact in fp32 (power-of-two targets: the
    scale n / size, the coordinate (o + 0.5) n / size - 0.5 and 1 - t are exact).  bilinear_mix = fma(r0, 1 - tx, fl(r1 tx)) with
    r0 = fma(a00, 1 - ty, fl(a10 ty)) and r1 likewise: a11 passes through 4 roundings (its product, r1's fma, r1 tx, the last fma), every
    other value through fewer, so rgb0 and w_256 are within gamma_4 S.  x0 is the fp16 (split) store of the same fp32 value: alpha_store,
    extra FLOOR_F16, beta = gamma_5 (>= gamma_4 (1 + 2^-11)).  rgb_256 = B2(rgb0'), rgb0' the computed rgb0 (|rgb0' - B1 x| <= gamma_4 B1|x|):
    |B2 rgb0' - B2 B1 x| <= B2(gamma_4 B1|x|) + gamma_4 B2|rgb0'| <= (2 gamma_4 + gamma_4^2) S2 with S2 = B2 B1 |x|."""
import torch
import torch.nn.functional as F

import sr_conv_reference as scr
from sr_conv_reference import ALPHA_F16, ALPHA_SPLIT, FLOOR_F16, U_F32, gamma, join, nhwc  # noqa: F401  (re-exported for the tests)

U = U_F32
#: derived bounds (module docstring); mode 'tc' = fp16 operands, 'tcx' = split [hi | lo] operands
ALPHA_CAT = {'tc': ALPHA_F16 + 2.0 ** -22, 'tcx': 2.0 ** -21}
BETA_MIX = {'tc': 4 * U, 'tcx': 5 * U}
ALPHA_MIX = {'tc': ALPHA_F16, 'tcx': ALPHA_SPLIT}
BETA_BLEND = 4 * U
BETA_GATE = 7 * U
FLOOR_GATE = 2.0 ** -126
BETA_AA = gamma(10)
BETA_BILINEAR = gamma(4)
BETA_BILINEAR_STORE = gamma(5)
BETA_BILINEAR_TWICE = 2 * gamma(4) + gamma(4) ** 2


def alpha_store(split: bool) -> float:
    return scr.alpha_store(split)


# ---- fusion --------------------------------------------------------------------------------------------------------------------------
def alpha_cat(xa: torch.Tensor, xb: torch.Tensor, alpha: torch.Tensor) -> torch.Tensor:
    """cat[xa * alpha, xb * (1 - alpha)] on NHWC float64; xb may hold one frame shared by the batch; alpha [N,H,W].  S = |ref|."""
    a = alpha.double()[..., None]
    return torch.cat([xa.double() * a, xb.double().expand(xa.shape[0], -1, -1, -1) * (1 - a)], dim=-1)


def cat3(xa: torch.Tensor, xb: torch.Tensor, xc: torch.Tensor) -> torch.Tensor:
    """cat[xa, xb, xc] on NHWC; xc may hold one frame shared by the batch."""
    return torch.cat([xa, xb, xc.expand(xa.shape[0], -1, -1, -1)], dim=-1)


def alpha_mix(xa: torch.Tensor, xb: torch.Tensor, alpha: torch.Tensor):
    """(ref, S) of xa * alpha + xb * (1 - alpha) on NHWC float64, alpha [N,H,W] in [0, 1]."""
    a = alpha.double()[..., None]
    xa, xb = xa.double(), xb.double()
    return xa * a + xb * (1 - a), xa.abs() * a + xb.abs() * (1 - a)


def blend(a: torch.Tensor, b: torch.Tensor, alpha: torch.Tensor):
    """(ref, S) of a * alpha + b * (1 - alpha) on NCHW float64, alpha [N,1,H,W] in [0, 1]."""
    al = alpha.double()
    a, b = a.double(), b.double()
    return a * al + b * (1 - al), a.abs() * al + b.abs() * (1 - al)


# ---- gating ----------------------------------------------------------------------------------------------------------------------------
def alpha_gate(logit: torch.Tensor, cap: torch.Tensor, summed: bool):
    """(ref, S, extra) of min(sigmoid(logit), cap), logit the float64 value the kernel reads (hi, or hi + lo when summed = lo_off > 0)."""
    v = logit.double()
    s = torch.sigmoid(v)
    extra = torch.full_like(s, FLOOR_GATE)
    if summed:
        extra = extra + 1.01 * U * v.abs() * s * (1 - s)
    return torch.minimum(s, cap.double()), s, extra


def person_occlusion_f32(alpha: torch.Tensor, torso: torch.Tensor, thr: float) -> torch.Tensor:
    """The kernel restated in torch fp32 (sr_with_ref.py's torso_occlusion + where(alpha > thr, 1, alpha), clamped)."""
    alpha, torso = alpha.float(), torso.float()
    return (torso + torch.where(alpha > thr, torch.ones_like(alpha), alpha)).clamp(0, 1)


def person_occlusion(alpha: torch.Tensor, torso: torch.Tensor, thr: float) -> torch.Tensor:
    """The same decision in float64 (thr as given)."""
    alpha, torso = alpha.double(), torso.double()
    return (torso + torch.where(alpha > thr, torch.ones_like(alpha), alpha)).clamp(0, 1)


# ---- resampling ------------------------------------------------------------------------------------------------------------------------
def aa_down2_matrix(n_out: int, dtype=torch.float64, device=None) -> torch.Tensor:
    """[n_out, 2 n_out] rows of F.interpolate(scale 1/2, bilinear, antialias=True) along one axis: the triangle of support 2 samples the
    taps [1,3,3,1] / 8 at inputs 2o - 1 .. 2o + 2; taps outside the input are dropped and the rest renormalised ([3,3,1] / 7 at o = 0,
    [1,3,3] / 7 at o = n_out - 1, [1,1] / 2 when n_out = 1)."""
    M = torch.zeros(n_out, 2 * n_out, dtype=dtype, device=device)
    k = (1.0, 3.0, 3.0, 1.0)
    for o in range(n_out):
        for t in range(4):
            i = 2 * o - 1 + t
            if 0 <= i < 2 * n_out:
                M[o, i] = k[t]
    return M / M.sum(dim=1, keepdim=True)


def aa_down2(x: torch.Tensor) -> torch.Tensor:
    """[N,C,2h,2w] -> [N,C,h,w] through the filter matrices, in x's dtype (float64 for the reference; S = aa_down2(|x|))."""
    h, w = x.shape[-2] // 2, x.shape[-1] // 2
    My, Mx = aa_down2_matrix(h, x.dtype, x.device), aa_down2_matrix(w, x.dtype, x.device)
    return torch.einsum('ai,ncij,bj->ncab', My, x, Mx)


def bilinear(x: torch.Tensor, size) -> torch.Tensor:
    """F.interpolate(bilinear, align_corners=False) of NCHW x in float64 (upsampling only: no antialias difference)."""
    return F.interpolate(x.double(), size=size, mode='bilinear', align_corners=False)


def warp_input(x_nhwc: torch.Tensor, wsum: torch.Tensor, h: int, w: int, size: int, res: int = 256):
    """{name: (ref, S)} of r3dp_sr_warp_input: x0 (float64 NCHW of all C channels), rgb0, rgb_256 and w_256."""
    N = x_nhwc.shape[0]
    x = x_nhwc.double().reshape(N, h, w, -1).permute(0, 3, 1, 2)
    ws = wsum.double().reshape(N, 1, h, w)
    x0, S0 = bilinear(x, (size, size)), bilinear(x.abs(), (size, size))
    return {'x0': (x0, S0), 'rgb0': (x0[:, :3], S0[:, :3]),
            'rgb_256': (bilinear(x0[:, :3], (res, res)), bilinear(S0[:, :3], (res, res))),
            'w_256': (bilinear(ws, (res, res)), bilinear(ws.abs(), (res, res)))}
