"""Float64 references and element-wise error bounds for the tensor-core SR convolutions (csrc/sr_tc.cu), for
tests/test_gpu_sr_conv_conformance.py.  Test infrastructure: it does not import the library, so it also runs on a machine without a GPU.

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
every case of the conformance suite, with headroom (see BETA).  The split mode's worst ratio is ten times the fp16 mode's: its K loop is
three times longer (hi x hi + lo x hi + hi x lo) and the worst case has 256 input channels, 6912 products per output."""
import math

import torch
import torch.nn.functional as F

from oracle import real3d_oracle as orc

SQRT2 = math.sqrt(2.0)
ALPHA_F16 = 2.0 ** -11
ALPHA_SPLIT = 2.0 ** -22
ALPHA_F32 = 2.0 ** -24
FLOOR_F16 = 2.0 ** -25                       # half the spacing of fp16 subnormals
SPLIT_WEIGHT_SCALE = 1024.0                  # split weights are stored x 2^10 so that their lo halves stay normal fp16 numbers
#: accumulation term per mode.  Worst ratio measured over the conformance suite on one H100 80GB HBM3 (SXM, 700 W power limit):
#: tc 2.12e-7 (torgb_ex, 256 channels; the worst conv output 1.76e-7, layer_torgb 128 -> 256), tcx 2.27e-6 (layer up=1, 256 -> 128).
#: beta = 2^-21 = 4.77e-7 (2.2x) and 2^-18 = 3.81e-6 (1.7x).  The kernels are deterministic and every H100 runs the same SASS in the
#: same summation order, so the headroom only has to cover new cases, not run-to-run noise.
BETA = {'tc': 2.0 ** -21, 'tcx': 2.0 ** -18}
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
