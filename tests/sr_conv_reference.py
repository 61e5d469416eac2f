"""Float64 references and element-wise error bounds for the tensor-core SR convolutions (csrc/sr_tc.cu), for
tests/test_gpu_sr_conv_conformance.py, and for the exact-fp32 SR path (csrc/sr_fp32.cu, last section below), for
tests/test_gpu_sr_fp32_conformance.py.  Test infrastructure: it does not import the library, so it also runs on a machine without a GPU.

Operands.  Every reference is computed from the operands the kernel actually reads, converted exactly to float64: the fp16 activations
(hi + lo for split [hi | lo] tensors), the packed weights read back and unpacked ((hi + lo) / 2^10 for split weights), and the fp32
bias, ToRGB weights and skip images as given.  The operations reuse oracle/real3d_oracle.py's dtype-generic mod_conv, fir_pad,
upsample2x and lrelu_gain; they run on the operands' device (cuDNN float64 on the GPU is independent of this library).

Error bound.  Each output element must satisfy

    |got - ref| <= alpha |ref| + extra + beta S

where S is the same operation applied to |x|, |w| and |bias| (and |residual|, |skip|, |wrgb|) in float64.  S bounds every partial sum of
the element, so beta S bounds the accumulation error whatever the summation order.  alpha is the rounding of the stored value:

  * fp16 store (`tc`):  the kernel stores fp16(y), y the fp32 result.  Round to nearest gives |fp16(y) - y| <= 2^-11 |y|, so alpha = 2^-11.
  * split store (`tcx`):  hi = fp16(y), lo = fp16(y - hi).  |y - hi| <= 2^-11 |y| and lo rounds that remainder again, so
    |y - (hi + lo)| <= 2^-11 |y - hi| <= 2^-22 |y|: alpha = 2^-22 on the reconstructed hi + lo.
  * Both hold for normal fp16 results only.  Below 2^-14 fp16 numbers are subnormal with a spacing of 2^-24, so every fp16 rounding
    also carries an absolute FLOOR = 2^-25.  For a split pair it is the lo half that turns subnormal, as soon as |y - hi| < 2^-14, i.e.
    for |y| below about 2^-3: the pair then reconstructs y to 2^-25 absolute, not 2^-22 relative (small resized input values show
    it).  Split weights are stored x 2^10 to keep their lo halves normal; in weight units the floor is 2^-35.
  * fp32 image (ToRGB outputs):  the result is the fp32 accumulator itself; its last rounding is 2^-24 |y|, alpha = 2^-24.
  * `tc` up path (transposed conv + FIR):  the kernel rounds the (2H+1) x (2W+1) transposed-conv grid to fp16 before the FIR, so each
    grid value carries up to 2^-11 |grid| + FLOOR more.  The FIR has positive taps summing to 4 and the activation is gain-Lipschitz,
    which adds extra = gain * (FIR(2^-11 |grid|) + 4 FLOOR).  The split path stores the grid as a split pair: the same term with 2^-22.
  * `tc` residual:  the kernel rounds twice, fp16(fp16(act) + res): extra = 2^-11 |act| + FLOOR for the inner rounding, alpha = 2^-11
    for the outer.
  * uint8 frames are compared bit for bit with torch's conversion of the kernel's own fp32 image; the conversion itself is exact.

beta is the accumulation term: fp32 sums of fp16 x fp16 products (exact in fp32) in the tensor cores' order, plus for split operands
the dropped lo x lo product (<= 2^-22 |x| |w| per term).  It is set from the worst (|got - ref| - alpha |ref| - extra) / S measured over
every case of the conformance suite, with headroom (see BETA).  The split mode's worst ratio is eight to ten times the fp16 mode's: its K
loop is three times longer (hi x hi + lo x hi + hi x lo) and the worst case has 512 input channels, 3 x 4608 = 13824 products per output.

The exact-fp32 path (csrc/sr_fp32.cu, sr_mode='fp32'; tests/test_gpu_sr_fp32_conformance.py).  Operands are fp32 and NCHW, and every
product is an fma on fp32 operands, so the conv output is an fp32 sum whose roundings all lie in beta S.  What remains, with
u = 2^-24 and the library built without --use_fast_math (sqrtf and divisions correctly rounded):

  * SR layer epilogue (bias + lrelu(0.2) * sqrt2):  three roundings, the bias add, the x 0.2f of negative values and the
    x 1.4142135623730951f, each <= u relative and multiplicative, so they compose to a relative error of the stored value.  The
    constants are not the reference's: 0.2f = 0.2 (1 + 1.5e-8) and the fp32 sqrt2 = sqrt2 (1 - 1.7e-8).  3u + 3.2e-8 = 2.1e-7 <= 2^-22:
    ALPHA_FP32_LAYER = 2^-22, against the float64 reference with the exact 0.2 and sqrt2.
  * up=2: the kernel writes the (2H+1) x (2W+1) transposed-conv grid to fp32 scratch and runs the FIR over it.  Each grid value carries
    its final rounding 2^-24 |grid|; the FIR's positive taps and the gain-Lipschitz activation carry it to the output as
    extra = gain * FIR(2^-24 |grid|), the fp32 analogue of the `tc` up-path term.  The FIR's own partial sums are bounded by S.
  * ToRGB: bias and the upsampled skip image are summands of the same fp32 sum: alpha = 2^-24 on the result, as for the fp32 images above.
  * styles = (w . fl(A fl(1 / sqrtf(w_dim))) + a) * post, post the fp32 value the kernel is given: every term's relative error (the fp32
    gain and the scaled affine weight, <= 2.5u) and the partial sums lie in beta S with S = post (|w| @ |A|^T / sqrt(w_dim) + |a|); the
    final x post rounds once: alpha = 2^-24.
  * fold:  v = fl(W s) (u), q = sum of the len = k^2 I squares v^2 (positive terms: <= gamma_len relative in any order, plus 2u from the
    rounding of v), fl(q + 1e-8f) (u), d = 1 / sqrtf (2u), out = fl(v d) (u).  rsqrt halves the relative error of q, so
    |out - ref| <= (5.5u + gamma_len / 2) |ref|; fold_alpha rounds 5.5u up to 6u to cover the second-order terms.  1e-8f differs from
    1e-8 by 6e-17, far below u q.  Without demodulation only fl(W s) remains: u.  fold_error carries an error of the styles on.

BETA['fp32'] covers the accumulation of the conv and ToRGB sums and of the styles.  It is measured like the others and is also no larger
than the deterministic bound gamma_K = K u / (1 - K u) of recursive summation at the suite's largest K = 9 * 256, so the bar is never
looser than what can be proved."""
import math

import torch
import torch.nn.functional as F

from oracle import real3d_oracle as orc

SQRT2 = math.sqrt(2.0)
ALPHA_F16 = 2.0 ** -11
ALPHA_SPLIT = 2.0 ** -22
ALPHA_F32 = 2.0 ** -24
ALPHA_FP32_LAYER = 2.0 ** -22                # the fp32 SR layer epilogue: bias add, x 0.2f, x fp32 sqrt2 (module docstring)
U_F32 = 2.0 ** -24                           # unit roundoff of fp32
FLOOR_F16 = 2.0 ** -25                       # half the spacing of fp16 subnormals
SPLIT_WEIGHT_SCALE = 1024.0                  # split weights are stored x 2^10 so that their lo halves stay normal fp16 numbers
#: accumulation term per mode.  Worst ratio measured over the conformance suite on one H100 80GB HBM3 (SXM, 700 W power limit):
#: tc 4.25e-7 and tcx 3.45e-6, both the torso head's fuse_head_torso_convs[0] (3x3, 512 -> 256 at 256^2, N = 4): K = 9 x 512 = 4608
#: products per output, twice the longest K of any other row, and 1.3x to 1.5x the ratios of the 256-channel launches at the same shape
#: (tc 2.90e-7, tcx 2.62e-6).  The small-shape rows alone: tc 1.75e-7 (layer_torgb 128 -> 256), tcx 2.27e-6 (layer up=1, 256 -> 128);
#: the rows with I <= 33 input channels 7.2e-8 and 1.0e-6.  beta = 2^-21 = 4.77e-7 (1.12x) and 2^-18 = 3.81e-6 (1.10x), far below the
#: deterministic bound of fp32 summation, gamma_K = 2.7e-4 at K = 4608.  The kernels are deterministic and every H100 runs the same SASS
#: in the same summation order, so the headroom only has to cover new cases, not run-to-run noise.
#: fp32 (tests/test_gpu_sr_fp32_conformance.py), on one H100 80GB HBM3 (SXM, 400 W power limit): 4.27e-7 (the up=2 scratch grid,
#: 256 -> 128 at 256^2; the worst layer output 3.57e-7, up=1 128 -> 128 at 512^2; ToRGB 2.50e-7; styles 3.42e-8).  beta = 2^-20 =
#: 9.54e-7 (2.2x), far below gamma_K = 1.37e-4 at K = 9 * 256.
BETA = {'tc': 2.0 ** -21, 'tcx': 2.0 ** -18, 'fp32': 2.0 ** -20}
#: epilogue activations of conv_tc3_kernel: code -> (slope, gain).  0 linear, 1 bias_act lrelu * sqrt2, 2 nn.LeakyReLU(0.01), 3 ReLU
ACT = {0: (1.0, 1.0), 1: (0.2, SQRT2), 2: (0.01, 1.0), 3: (0.0, 1.0)}
#: the FIR [1,3,3,1] x gain 4 per axis, as composed into the up weights
G4 = (0.25, 0.75, 0.75, 0.25)


def alpha_store(split: bool) -> float:
    return ALPHA_SPLIT if split else ALPHA_F16


# ---- operands as the kernel reads them ---------------------------------------------------------------------------------------------------
def join(t: torch.Tensor) -> torch.Tensor:
    """[hi | lo] fp16 [..., 2C] -> float64 [..., C] = hi + lo."""
    C = t.shape[-1] // 2
    return t[..., :C].double() + t[..., C:].double()


def activations(x: torch.Tensor, C: int, split: bool) -> torch.Tensor:
    """NHWC fp16 [N,H,W,Cp] ([N,H,W,2Cp] split) -> float64 NCHW [N,C,H,W] of the first C channels."""
    v = join(x) if split else x.double()
    return v[..., :C].permute(0, 3, 1, 2).contiguous()


def nhwc(y: torch.Tensor, split: bool) -> torch.Tensor:
    """A kernel's NHWC fp16 output -> float64 NCHW (hi + lo when split)."""
    return (join(y) if split else y.double()).permute(0, 3, 1, 2)


def packed_weights(wp: torch.Tensor, I: int, split: bool) -> torch.Tensor:
    """Packed weights [Nw,T,O,Ip] ([Nw,T,O,2Ip] split, x 2^10) -> float64 [Nw,T,O,I]."""
    w = join(wp) / SPLIT_WEIGHT_SCALE if split else wp.double()
    return w[..., :I]


def taps3x3(w: torch.Tensor) -> torch.Tensor:
    """[Nw,9,O,I] (tap = ky * 3 + kx) -> [Nw,O,I,3,3]."""
    Nw, _, O, I = w.shape
    return w.permute(0, 2, 3, 1).reshape(Nw, O, I, 3, 3)


def taps_composed(w: torch.Tensor) -> torch.Tensor:
    """[Nw,36,O,I] (tap = (p * 2 + q) * 9 + (dy + 1) * 3 + dx + 1) -> [Nw,4,O,I,3,3]."""
    Nw, _, O, I = w.shape
    return w.reshape(Nw, 4, 9, O, I).permute(0, 1, 3, 4, 2).reshape(Nw, 4, O, I, 3, 3)


def per_sample(w: torch.Tensor, N: int) -> torch.Tensor:
    """Weights of Nw = 1 (shared) or N sets -> N sets."""
    return w.expand(N, *w.shape[1:]) if w.shape[0] == 1 else w


# ---- operations in float64 ---------------------------------------------------------------------------------------------------------------
def bias_act(v: torch.Tensor, bias: torch.Tensor, code: int) -> torch.Tensor:
    """bias + activation of the conv epilogue on NCHW v."""
    if code == 1:
        return orc.lrelu_gain(v, bias)
    v = v + bias.view(1, -1, 1, 1)
    if code == 2:
        return F.leaky_relu(v, 0.01)                                       # nn.LeakyReLU()
    if code == 3:
        return torch.relu(v)
    return v


def act_gain(code: int) -> float:
    return ACT[code][1]


def conv_same(x: torch.Tensor, w: torch.Tensor, ksize: int = 3) -> torch.Tensor:
    """Per-sample 'same' correlation, x [N,I,H,W], w [N,O,I,3,3]; ksize 1 uses the centre tap only (the one the kernel reads)."""
    if ksize == 1:
        w = w[..., 1:2, 1:2]
    with torch.device(x.device):
        return orc.mod_conv(x, w, 1)


def conv_transposed(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """The (2H+1) x (2W+1) grid of the stride-2 transposed conv with the unflipped weight (the first step of mod_conv(up=2))."""
    return torch.cat([F.conv_transpose2d(x[n:n + 1], w[n].transpose(0, 1), stride=2) for n in range(x.shape[0])], 0)


def fir_up(grid: torch.Tensor) -> torch.Tensor:
    """The second step of mod_conv(up=2): FIR pad 1, gain 4."""
    with torch.device(grid.device):
        return orc.fir_pad(grid, (1, 1, 1, 1), 4.0)


def upsample2x(img: torch.Tensor) -> torch.Tensor:
    with torch.device(img.device):
        return orc.upsample2x(img)


def compose_matrix(dtype=torch.float64, device=None) -> torch.Tensor:
    """A[p][dy + 1][ky] = g[u] with p + u - 1 - ky == 2 dy (zero where no u in 0..3 exists)."""
    A = torch.zeros(2, 3, 3, dtype=dtype, device=device)
    for p in range(2):
        for dy in (-1, 0, 1):
            for ky in range(3):
                u = 2 * dy + 1 + ky - p
                if 0 <= u <= 3:
                    A[p, dy + 1, ky] = G4[u]
    return A


def compose_up_weights(w: torch.Tensor) -> torch.Tensor:
    """FIR(conv_transpose(x, w)) as four 3x3 correlations on x, one per output parity (p, q):
    G[p * 2 + q][dy][dx] = sum_{ky,kx} A[p][dy][ky] A[q][dx][kx] w[ky][kx].  w [..., 3, 3] -> [..., 4, 3, 3] (parity axis before the taps)."""
    A = compose_matrix(w.dtype, w.device)
    G = torch.einsum('pak,qbl,...kl->...pqab', A, A, w)
    return G.reshape(*w.shape[:-2], 4, 3, 3)


def conv_up_composed(x: torch.Tensor, G: torch.Tensor) -> torch.Tensor:
    """x [N,I,H,W], G [N,4,O,I,3,3] -> [N,O,2H,2W]: output pixel (2i + p, 2j + q) is the correlation with G[p * 2 + q]."""
    N, _, H, W = x.shape
    out = x.new_zeros(N, G.shape[2], 2 * H, 2 * W)
    for ph in range(4):
        out[:, :, ph >> 1::2, ph & 1::2] = conv_same(x, G[:, ph])
    return out


def torgb(a: torch.Tensor, wrgb: torch.Tensor) -> torch.Tensor:
    """Per-sample 1x1 ToRGB without bias: a [N,C,H,W], wrgb [N,3,C] -> [N,3,H,W]."""
    return torch.einsum('nchw,nkc->nkhw', a, wrgb)


def styles(w: torch.Tensor, A: torch.Tensor, a: torch.Tensor, post: float = 1.0) -> torch.Tensor:
    """affine(w) * post: w [N,w_dim], A [Cin,w_dim], a [Cin] -> [N,Cin]."""
    return orc.affine_styles(w, A, a) * post


def styles_abs(w: torch.Tensor, A: torch.Tensor, a: torch.Tensor, post: float = 1.0) -> torch.Tensor:
    """S of styles(): |post| (|w| @ |A|^T / sqrt(w_dim) + |a|)."""
    return orc.affine_styles(w.abs(), A.abs(), a.abs()) * abs(post)


def fold(W: torch.Tensor, s: torch.Tensor, demod: bool) -> torch.Tensor:
    """Modulated (+ demodulated) weights: W [O,I,k,k], s [N,I] -> [N,O,I,k,k]."""
    return orc.fold_weight(W, s, demod)


def fold_abs(W: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """|W| |s|, the magnitude of every modulated weight before demodulation."""
    return orc.fold_weight(W.abs(), s.abs(), False)


def gamma(k: int) -> float:
    """gamma_k = k u / (1 - k u): the relative bound of k fp32 roundings, e.g. of a recursive sum of k terms."""
    return k * U_F32 / (1 - k * U_F32)


def fold_alpha(length: int, demod: bool) -> float:
    """Relative error of r3dp_sr_fold_weights for exact styles; length = k^2 I (module docstring)."""
    return 6 * U_F32 + gamma(length) / 2 if demod else U_F32


def fold_error(W: torch.Tensor, s: torch.Tensor, ds: torch.Tensor, demod: bool):
    """(ref, E): ref = fold(W, s) and an element-wise bound E on |fold_kernel(W, s') - ref| for any styles s' with |s' - s| <= ds.
    W [O,I,k,k], s and ds [N,I], float64.  With v = W s, D = |W| ds and eta = fold_alpha: the kernel's result is W s' d' (1 + eta') with
    |eta'| <= eta and d' = rsqrt(||W s'||^2 + 1e-8) per output channel.  sqrt(||W s'||^2 + 1e-8) lies within ||D|| of
    sqrt(||W s||^2 + 1e-8) = 1 / d (triangle inequality), so d / (1 + r) <= d' <= d / (1 - r) with r = ||D|| d, and
        |W s' d' (1 + eta') - W s d| <= D d g + |ref| (g - 1),   g = (1 + eta) / (1 - r).
    Without demodulation: |fl(W s') - W s| <= D (1 + eta) + eta |ref|.  ds = 0 gives eta |ref|."""
    ref = fold(W, s, demod)
    D = fold_abs(W, ds)
    eta = fold_alpha(W[0].numel(), demod)
    if not demod:
        return ref, D * (1 + eta) + eta * ref.abs()
    dims = [2, 3, 4]
    q = fold(W, s, False).square().sum(dim=dims, keepdim=True) + 1e-8
    r = D.square().sum(dim=dims, keepdim=True).sqrt() / q.sqrt()
    assert float(r.max()) < 0.5, 'styles error too large for the first-order fold bound'
    g = (1 + eta) / (1 - r)
    return ref, D * q.rsqrt() * g + ref.abs() * (g - 1)


def to_uint8(img: torch.Tensor) -> torch.Tensor:
    """The caller's frame conversion ((x + 1) / 2 * 255).int() of a clamped fp32 NCHW image -> uint8 HWC frames."""
    return ((img + 1) / 2 * 255.).int().permute(0, 2, 3, 1).to(torch.uint8)


# ---- the bound ---------------------------------------------------------------------------------------------------------------------------
def excess_ratio(got, ref, S, alpha, extra=None) -> float:
    """max over elements of (|got - ref| - alpha |ref| - extra) / S: what beta has to cover."""
    d = (got.double() - ref).abs() - alpha * ref.abs()
    if extra is not None:
        d = d - extra
    return float((d / S.clamp_min(1e-300)).max())


def check_bound(got, ref, S, alpha, beta, extra=None, tag=''):
    """Assert |got - ref| <= alpha |ref| + extra + beta S element-wise (non-finite values fail); returns the excess ratio.
    extra: a tensor or a number (the rounding floors)."""
    got = got.double()
    assert got.shape == ref.shape == S.shape, (tag, got.shape, ref.shape, S.shape)
    allow = alpha * ref.abs() + beta * S
    if extra is not None:
        allow = allow + extra
    d = (got - ref).abs()
    bad = ~(d <= allow)
    r = excess_ratio(got, ref, S, alpha, extra)
    print(f'{tag}: worst excess / S = {r:.3e} (beta {beta:.3e}), max |err| {float(d.max()):.3e}, max |ref| {float(ref.abs().max()):.3e}')
    if bool(bad.any()):
        i = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError(f'{tag}: {int(bad.sum())} of {bad.numel()} elements outside the bound; first at {i}: got {float(got[i]):.9g}, '
                             f'ref {float(ref[i]):.9g}, allowed {float(allow[i]):.3e}')
    return r
