"""Float64 references and error bounds for the fused render (csrc/render.cu, csrc/render_stream.cu) and its stand-alone ops, for
tests/test_gpu_render_conformance.py and tests/test_cpu_render_reference.py.  Test infrastructure: it does not import the library, so it
also runs on a machine without a GPU.

Operands.  Every reference takes the fp32 inputs exactly (planes, rays, jitter, decoder weights) and computes in float64, reusing
oracle/real3d_oracle.py's dtype-generic functions.  Two pieces are kept in fp32 on purpose because the kernels compute them with correctly
rounded fp32 operations in a fixed order, and the reference reproduces those bits instead of bounding them: the ray limits and the coarse
sample depths (math_utils.py / renderer.py order, as the oracle writes it, and the stratified steps k / (S - 1) are the oracle's fp32
constants), and the sample positions o + d t.  Fine (importance) depths are computed in float64 and rounded to fp32, the precision the
kernel stores them in.

Grid coordinates.  The kernels unnormalise g = (2 / box_warp) x to pixel units p = ((g + 1) size - 1) / 2 in fp32, and nvcc contracts
those products and sums into FMAs, so p is reproducible only to about one ulp.  At 256 texels one ulp of p moves a tap weight by 2^-16,
which is far more than the decoder's own error; the per-element tests therefore place samples where every one of those operations is
exact (dyadic coordinates: `dyadic`), and the whole-render tolerance below bounds the coordinate term statistically, not per sample.

Decoder bound (`decoder_bound`).  For features f the kernel decodes (each with an absolute input error ef, from the gather), every output
obeys |got - ref| <= the bound built as follows, with u = 2^-24 (fp32), S1 = |f| |W1'|^T + |b1|, S2 = |h| |W2'|^T + |b2|, W1' = W1 / sqrt(32)
and W2' = W2 / 8 rounded to fp32 (2^-24 relative more on W1'):

  * split operands (the wgmma decoders): v = hi + lo with hi = fp16(v), lo = fp16(v - hi).  |v - hi| <= 2^-11 |v| and lo rounds that again,
    so |v - (hi + lo)| <= 2^-22 |v| while lo is a normal fp16 number; below 2^-14 fp16 is subnormal with spacing 2^-24, so every split also
    carries an absolute floor of 2^-25.  The decoder weights are NOT scaled (unlike the SR convolutions' x 2^10): with W1' ~ 0.01 the lo
    halves of the weights are subnormal and the floor is the larger term.  Per layer: 2^-22 S + 2^-25 (sum|w| + sum|v|) for the two
    representations, and the dropped lo x lo product <= (2^-11 |v| + 2^-25)(2^-11 |w| + 2^-25) summed, i.e. 2^-22 S + small floors;
  * accumulation: the worst case BETA S per layer (wgmma: one fp32 rounding per k-step of 16 exact fp16 x fp16 products, 6 k-steps in
    layer 1 and 12 in layer 2; the CUDA-core decoder: sequential fp32 FMAs, n u S for n products) plus u |a| for the bias add;
  * softplus: 1-Lipschitz, so layer-1 errors pass to h unchanged; the kernels' approximations (ex2/lg2.approx in softplus2, exp2f/__log2f
    in softplus_fast: <= 2 ulp each on arguments in [1, 2] / [-inf, 0]) add <= SP_ABS + SP_REL |h|;
  * layer 2 sees the layer-1 error through sum_j |W2'_oj| e_j;
  * sigma = y_0; colours c = 1.002 sigmoid(y) - 0.001 with sigmoid 1/4-Lipschitz: e_c = 1.002 / 4 e_y + SIG_ABS (ex2.approx + rcp.approx,
    or __expf + __fdividef).

Gather bound (`gather_bound`): at exact pixel coordinates the fp32 tap weights are products of exact fractional parts, rounded once (u);
the 4 (8) taps of 3 planes are summed with FMAs (12 (24) terms: 12 (24) u of sum w |t|) and scaled by fp32(1/3) (2 u).  Off dyadic
coordinates add DELTA_PX per axis (two ulp of the pixel coordinate, the FMA contraction) times the quad's sum |t|.

Whole-render tolerances (TAU_*).  With the decoder within its bound and the march in fp32, rgb = 2 sum_k v_k c_k - 1 moves by at most
2 sum_k v_k e_c,k + the march term.  Over the cases of the conformance suite the colour bound is <= 1.5e-6 where the weights sit (opaque
decoders: a few samples carry all the weight) and the march adds (S + 2) u relative per sum; TAU_RGB = 5e-6 keeps a factor two over the sum
of both and stays below 1/3 of the smallest defect error on the same inputs (test_cpu_render_reference.py asserts >= 3x for each defect).
The same TAU_RGB holds for the transparent decoder, where it claims nothing about defects (they move rgb by only 2.5e-6 there).
Two terms are outside this budget:
  * the pixel-coordinate ulp (above).  It moves single samples, and a render averages it over the samples that carry weight: at
    BASELINE config 1 (256^2 planes, 48 samples) single-pass renders stay within 1e-6 of float64 on an H100;
  * importance resampling.  The kernels build the importance CDF from fp32 weights; where the pdf is flat (den ~ 1e-5) an fp32 rounding
    of the CDF moves a fine sample by up to (u / den) of its bin, and on 256^2 planes that moves its features by far more than the decoder's
    error.  The fp32 oracle itself is 9.5e-6 from float64 at BASELINE config 1 with 48 + 48 samples and an opaque decoder (the kernel:
    9.4e-6), so TAU_RGB cannot hold there for any fp32 implementation.  The smallest decoder defect on those inputs moves rgb by 3.1e-5
    (x_lo), so a bar with 3x teeth must be <= 1.03e-5: a window of less than 10 % over the resampling term alone, too narrow to derive a
    bar in.  That case is kept as a strict expected failure at TAU_RGB carrying these numbers.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

from oracle import real3d_oracle as orc
from real3dportrait_b200 import synthetic as syn

U = 2.0 ** -24
SPLIT = 2.0 ** -22
FLOOR = 2.0 ** -25
#: accumulation term per decoder and layer, worst cases: wgmma adds the 16 exact fp16 x fp16 products of each k-step to its fp32 accumulator
#: with one rounding (<= 2^-23 of the result, <= 2^-23 S), over 6 (layer 1: 3 partial products x 2) and 12 (layer 2: 3 x 4) k-steps; the
#: CUDA-core decoder's sequential fp32 FMAs, bias first, over 32 and 64 products: gamma_n <= n u of S
BETA = {True: (6 * 2.0 ** -23, 12 * 2.0 ** -23), False: (32 * 2.0 ** -24, 64 * 2.0 ** -24)}
SP_ABS, SP_REL = 2.0 ** -21, 2.0 ** -21
SIG_ABS = 2.0 ** -20
#: whole-render tolerances (see the module docstring)
TAU_RGB = 5e-6
TAU_WSUM = 5e-6
TAU_DEPTH = 5e-6
G1, G2 = 1.0 / math.sqrt(32.0), 0.125


# ---- decoders -----------------------------------------------------------------------------------------------------------------------------
def transparent_decoder(seed: int = 4) -> Dict[str, torch.Tensor]:
    """The suite's usual decoder (synthetic.make_decoder_params): sum w <= 0.2 on most rays."""
    return syn.make_decoder_params(seed=seed)


def opaque_decoder(seed: int = 4, scale: float = 1.0, density_bias: float = 30.0) -> Dict[str, torch.Tensor]:
    """A decoder whose density saturates (sum w ~ 1), as a trained head's does on the face: the transparent decoder of `seed` with every
    weight scaled by `scale` and net.2.bias[0] = density_bias."""
    p = {k: v.clone() for k, v in syn.make_decoder_params(seed=seed).items()}
    p['net.0.weight'] *= scale
    p['net.2.weight'] *= scale
    p['net.2.bias'][0] = density_bias
    return p


def decoder_set():
    """(name, params): the opaque decoders of the conformance suite."""
    return [('opaque_s4', opaque_decoder(4)), ('opaque_s11', opaque_decoder(11)), ('opaque_s23_x0.05', opaque_decoder(23, 0.05)),
            ('opaque_s5_x4', opaque_decoder(5, 4.0, 60.0))]


def scaled_weights(mlp, dtype=torch.float64):
    """W1' = fp32(W1 * fp32(1/sqrt 32)) and W2' = W2 / 8 as the kernels form them, and the biases, in `dtype`."""
    w1 = (mlp['net.0.weight'].float() * torch.tensor(G1, dtype=torch.float32)).to(dtype)
    w2 = (mlp['net.2.weight'].float() * G2).to(dtype)
    return w1, mlp['net.0.bias'].to(dtype), w2, mlp['net.2.bias'].to(dtype)


def decode64(f: torch.Tensor, mlp):
    """f[..., 32] (any dtype) -> (colours [..., 32], sigma [..., 1]) in float64 from the exact weights."""
    m = {k: v.double() for k, v in mlp.items()}
    h = orc.softplus(f.double() @ (m['net.0.weight'] * G1).t() + m['net.0.bias'])
    y = h @ (m['net.2.weight'] * G2).t() + m['net.2.bias']
    return torch.sigmoid(y[..., 1:]) * 1.002 - 0.001, y[..., :1]


def _split(v: torch.Tensor):
    hi = v.half().float()
    return hi, (v - hi).half().float()


def decode_split(f: torch.Tensor, mlp, drop: Optional[str] = None):
    """CPU simulation of the wgmma decoders on fp32 features f[..., 32]: hi / lo halves by torch.half, the three partial products
    hi hi + lo hi + hi lo (lo lo dropped) accumulated in fp32.  `drop` removes one more partial product, as a defective kernel would:
    'x_lo' (x_lo w1_hi: the gather's lo half lost), 'w1_lo' (x_hi w1_lo), 'h_lo' (h_lo w2_hi), 'w2_lo' (h_hi w2_lo), 'all_lo' (plain fp16)."""
    w1, b1, w2, b2 = scaled_weights(mlp, torch.float32)
    xh, xl = _split(f.float())
    w1h, w1l = _split(w1)
    a = xh @ w1h.t()
    if drop not in ('x_lo', 'all_lo'):
        a = a + xl @ w1h.t()
    if drop not in ('w1_lo', 'all_lo'):
        a = a + xh @ w1l.t()
    h = orc.softplus(a + b1)
    hh, hl = _split(h)
    w2h, w2l = _split(w2)
    y = hh @ w2h.t()
    if drop not in ('h_lo', 'all_lo'):
        y = y + hl @ w2h.t()
    if drop not in ('w2_lo', 'all_lo'):
        y = y + hh @ w2l.t()
    y = y + b2
    return torch.sigmoid(y[..., 1:]) * 1.002 - 0.001, y[..., :1]


def decode_fp32(f: torch.Tensor, mlp):
    """The fp32 oracle's decoder on fp32 features."""
    return orc.decode(f.float().unsqueeze(-3), {k: v.float() for k, v in mlp.items()})


def decoder_bound(f: torch.Tensor, mlp, ef, split: bool):
    """Element-wise bound (colours [..., 32], sigma [..., 1]) on |decoder(f) - decode64(f_true)| for features f (float64 of what the kernel
    holds) that are within ef (tensor or scalar) of f_true.  split = True: the wgmma decoders; False: the CUDA-core decoder (fp32)."""
    w1, b1, w2, b2 = scaled_weights(mlp)
    f = f.double()
    af = f.abs()
    ef = torch.as_tensor(ef, dtype=torch.float64).expand_as(f)
    aw1, aw2 = w1.abs(), w2.abs()
    s1 = af @ aw1.t() + b1.abs()
    a = f @ w1.t() + b1
    h = orc.softplus(a)
    s2 = h.abs() @ aw2.t() + b2.abs()
    y = h @ w2.t() + b2
    rep = 3 * SPLIT if split else 0.0                         # x and w representations, the dropped lo x lo
    b1_acc, b2_acc = BETA[split]
    e1 = ef @ aw1.t() + (rep + U + b1_acc) * s1 + U * a.abs()
    if split:
        e1 = e1 + FLOOR * (aw1.sum(1) + af.sum(-1, keepdim=True)) * 1.5
    eh = e1 + SP_ABS + SP_REL * h.abs()
    ey = eh @ aw2.t() + (rep + b2_acc) * s2 + U * y.abs()
    if split:
        ey = ey + FLOOR * (aw2.sum(1) + h.abs().sum(-1, keepdim=True)) * 1.5
    ec = 1.002 / 4 * ey[..., 1:] + SIG_ABS + U
    return ec, ey[..., :1]


# ---- gather --------------------------------------------------------------------------------------------------------------------------------
def dyadic(t: torch.Tensor, bits: int = 12) -> torch.Tensor:
    """Round coordinates to multiples of 2^-bits: with box_warp a power of two and plane sizes below 2^(23 - bits) the kernels' pixel
    coordinates ((2 / box_warp) x + 1) size - 1) / 2 are then exact whatever FMA contraction nvcc picks."""
    return torch.round(t * 2.0 ** bits) / 2.0 ** bits


def _pix(g: torch.Tensor, size: int) -> torch.Tensor:
    """fp32 unnormalisation as the oracle writes it (((g + 1) size - 1) / 2), returned in float64."""
    return (((g.float() + 1) * size - 1) / 2).double()


def gather64(planes: torch.Tensor, xyz: torch.Tensor, box_warp: float, depth: int = 0):
    """planes [N,3,C,H,W] (tri-grids: [N,3,C*D,H,W]), fp32 points xyz [N,P,3] -> (f [N,P,C] float64 mean over the planes, Q [N,P]
    = sum over the planes of the tap quads' largest |texel|, Sg [N,P,C] = sum of w |t|)."""
    N, _, CD, H, W = planes.shape
    D = depth if depth > 0 else 1
    C = CD // D
    g = xyz.float() * torch.tensor(2.0 / box_warp, dtype=torch.float32)
    pl = planes.double().reshape(N, 3, C, D, H * W)
    P = xyz.shape[1]
    f = torch.zeros(N, C, P, dtype=torch.float64)
    sg = torch.zeros_like(f)
    q = torch.zeros(N, P, dtype=torch.float64)
    for p, ((au, av), aw) in enumerate(zip(orc.PLANE_UV, orc.PLANE_W)):
        px, py = _pix(g[..., au], W), _pix(g[..., av], H)
        pz = _pix(g[..., aw], D) if depth > 0 else torch.zeros_like(px)
        x0, y0, z0 = torch.floor(px), torch.floor(py), torch.floor(pz)
        wx, wy = ((x0 + 1) - px, px - x0), ((y0 + 1) - py, py - y0)
        wz = ((z0 + 1) - pz, pz - z0) if depth > 0 else (torch.ones_like(pz), torch.zeros_like(pz))
        gp = pl[:, p].reshape(N, C, D * H * W)
        qm = torch.zeros(N, P, dtype=torch.float64)
        for dz in ((0, 1) if depth > 0 else (0,)):
            for dy in (0, 1):
                for dx in (0, 1):
                    xi, yi, zi = (x0 + dx).long(), (y0 + dy).long(), (z0 + dz).long()
                    inb = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H) & (zi >= 0) & (zi < D)
                    lin = (zi.clamp(0, D - 1) * H + yi.clamp(0, H - 1)) * W + xi.clamp(0, W - 1)
                    tex = torch.gather(gp, 2, lin[:, None, :].expand(-1, C, -1)) * inb[:, None, :]
                    w = wx[dx] * wy[dy] * wz[dz]
                    f += tex * w[:, None, :]
                    sg += tex.abs() * w[:, None, :]
                    qm = torch.maximum(qm, tex.abs().amax(1))
        q += qm
    return (f / 3).permute(0, 2, 1), q, (sg / 3).permute(0, 2, 1)


def gather_bound(q: torch.Tensor, sg: torch.Tensor, depth: int = 0, exact_px: bool = True, sizes=(1, 1, 1)):
    """Bound on the fp32 mean features of gather64's points: [N,P,C].  exact_px = False adds two ulp of each pixel coordinate (sizes =
    the largest H, W, D) times 2 x the quad's largest |texel| per axis and plane (q sums the planes)."""
    terms = 24 if depth > 0 else 12
    e = (terms + 3) * U * sg
    if not exact_px:
        delta = sum(2 * U * 2 * s for s in sizes)
        e = e + (delta * 2 * q / 3)[..., None]
    return e


# ---- whole render ------------------------------------------------------------------------------------------------------------------------
def render64(planes, mlp, ray_o, ray_d, *, S, S_imp=0, box_warp=1.0, white_back=False, u_coarse, u_fine=None, trigrid_depth=0,
             planes2=None, decode=None):
    """ImportanceRenderer.forward with 'auto' limits in float64 from fp32 inputs (see the module docstring for the fp32 parts kept).
    planes2: a second plane set added to the first (frame count 1 or N).  decode(f32 features) replaces the float64 decoder (CPU
    simulations of the kernels' decoders).  Returns rgb [N,M,32], depth [N,M,1], weights_sum [N,M,1], is_ray_valid [N,M,1]."""
    N, M, _ = ray_o.shape
    if planes2 is not None:                                                        # sampling is linear: sample the float64 sum
        planes = planes.double() + planes2.double()
    t0, t1, valid = orc.auto_limits(ray_o.float(), ray_d.float(), box_warp)
    d_c = orc.stratified_depths(t0, t1, S, u_coarse.float())                       # fp32, bit-exact with the kernels

    def model(d32):
        xyz = (ray_o.float().unsqueeze(-2) + d32 * ray_d.float().unsqueeze(-2)).reshape(N, -1, 3)
        f, _, _ = gather64(planes, xyz, box_warp, trigrid_depth)
        if decode is not None:
            c, s = decode(f.float())
            c, s = c.double(), s.double()
        else:
            c, s = decode64(f, mlp)
        return c.reshape(N, M, d32.shape[2], -1), s.reshape(N, M, d32.shape[2], 1)

    col, sig = model(d_c)
    d_c64 = d_c.double()
    if S_imp > 0:
        _, _, w = orc.ray_march(col, sig, d_c64, white_back)
        d_f = orc.importance_depths(d_c64, w, u_fine.double()).float()
        col_f, sig_f = model(d_f)
        d_a, c_a, s_a = orc.unify(d_c64, col, sig, d_f.double(), col_f, sig_f)
        rgb, depth, w = orc.ray_march(c_a, s_a, d_a, white_back)
    else:
        rgb, depth, w = orc.ray_march(col, sig, d_c64, white_back)
    return rgb, depth, w.sum(2), valid


# ---- inputs --------------------------------------------------------------------------------------------------------------------------------
def probe_rays(N: int, M: int, seed: int, box: float = 1.0):
    """Rays along exactly (0, 0, -1) from dyadic (x, y) inside the box: every sample of a ray has the same plane-0 features."""
    g = torch.Generator().manual_seed(seed)
    xy = dyadic((torch.rand(N, M, 2, generator=g) - 0.5) * 0.98 * box)
    o = torch.cat([xy, torch.full((N, M, 1), 1.6 * box)], -1)
    d = torch.zeros(N, M, 3)
    d[..., 2] = -1.0
    return o, d


def probe_planes(N: int, H: int, W: int, scale: float, seed: int):
    """Plane 0 random, planes 1 and 2 zero: features depend on (x, y) only."""
    g = torch.Generator().manual_seed(seed)
    p = torch.zeros(N, 3, 32, H, W)
    p[:, 0] = torch.randn(N, 32, H, W, generator=g) * scale
    return p


def scatter_rays(N: int, M: int, seed: int, spread: float = 0.45, miss: bool = True):
    """Explicit rays from z = 1.6 towards the box with random directions (some miss it when `miss`)."""
    g = torch.Generator().manual_seed(seed)
    o = torch.tensor([0.0, 0.0, 1.6]).expand(N, M, 3).contiguous() + 0.05 * torch.randn(N, M, 3, generator=g)
    d = torch.nn.functional.normalize(torch.tensor([0.0, 0.0, -1.0]) + spread * torch.randn(N, M, 3, generator=g), dim=-1)
    if not miss:
        d = torch.nn.functional.normalize(torch.tensor([0.0, 0.0, -1.0]) + 0.12 * torch.randn(N, M, 3, generator=g), dim=-1)
    return o, d
