"""Conformance of the exact-fp32 SR path (csrc/sr_fp32.cu, sr_mode='fp32') against float64.

* Every entry point through the C API (r3dp_sr_styles, r3dp_sr_fold_weights, r3dp_sr_layer_fp32 up 1 and 2, r3dp_sr_torgb_fp32) against a
  float64 reference built on the GPU from the fp32 operands the kernel reads, with the element-wise bounds of tests/sr_conv_reference.py
  (its docstring derives the fp32 alpha, extra and the fold bound; BETA['fp32'] is measured).  The layer cases cover the production
  shapes and the edges of conv_taps_kernel: partial and single 8-channel ci chunks, partial 32-wide co blocks, exact, partial and
  non-square 16 x 32 tiles, and up=2 phase grids of (H+1) x (W+1) that spill one tile in each axis.
* Per call: canaries around the output (and the up=2 scratch grid), every output element and every scratch grid element written, image
  k of an N = 3 launch bit for bit equal to the N = 1 launch of image k, and a repeated launch giving the same bits.
* The chain from latent to weights: SynthesisLayer / ToRGBLayer.folded_weight and the tensor-core packers sr_tc._pack /
  _pack_up_composed against float64 fold(styles(w)) from the module parameters.
* The whole SuperresolutionHybrid8XDC(sr_mode='fp32') against oracle.superres in float64, at a bar that float64 on fp16-rounded folded
  weights does not meet, and frame independence bit for bit."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import real3dportrait_b200 as r3
from real3dportrait_b200 import _capi as capi
from real3dportrait_b200 import sr_tc
from real3dportrait_b200 import synthetic as syn
from oracle import real3d_oracle as orc
import sr_conv_reference as scr

pytestmark = pytest.mark.gpu
DEV = 'cuda'
GUARD = 4096
SENTINEL = 0x7FC01234                       # an fp32 NaN no kernel produces
#: whole-image bar of the fp32 SR against float64, max |err| <= TAU * range.  Measured on one H100 80GB HBM3 (SXM, 400 W power limit):
#: 6.03e-7 (64^2 input, resized) and 6.19e-7 (128^2) x range, so TAU = 2e-6 (3.2x).  float64 on fp16-rounded folded weights lands at
#: 2.0e-4 and 2.5e-4 x range, a hundred times outside.
TAU = 2e-6


def _randn(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator(device=DEV).manual_seed(seed), device=DEV)


def _canary(shape):
    """(buffer, view): a float32 view of `shape` inside a sentinel-filled buffer with GUARD elements on each side."""
    n = math.prod(shape)
    buf = torch.empty(n + 2 * GUARD, device=DEV)
    buf.view(torch.int32).fill_(SENTINEL)
    return buf, buf[GUARD:GUARD + n].view(shape)


def _check_canary(buf, what):
    b = buf.view(torch.int32)
    assert bool((b[:GUARD] == SENTINEL).all()) and bool((b[-GUARD:] == SENTINEL).all()), f'{what}: written outside its bounds'
    assert not bool((b[GUARD:-GUARD] == SENTINEL).any()), f'{what}: elements left unwritten'


def _bits(t):
    return t.contiguous().view(torch.int32)


def _check(got, ref, E, tag):
    """|got - ref| <= E element-wise; prints the share of the bound used."""
    return scr.check_bound(got, ref, E, 0.0, 1.0, tag=tag + ' (ratio = share of the bound)')


# ---- (a) styles --------------------------------------------------------------------------------------------------------------------------
def _styles(w, A, a, post):
    N, w_dim = w.shape
    Cin = A.shape[0]
    buf, s = _canary((N, Cin))
    capi.check(capi.lib().r3dp_sr_styles(capi.ptr(w), capi.ptr(A), capi.ptr(a), N, w_dim, Cin, C.c_float(post), capi.ptr(s), capi.stream()))
    torch.cuda.synchronize()
    _check_canary(buf, 'styles')
    return s


# N, w_dim, Cin, post (1 / sqrt(Cin): the ToRGB use)
STYLE_CASES = [(1, 512, 3, 1.0), (3, 512, 32, 1.0), (3, 512, 256, 1.0), (1, 512, 256, 1 / 16), (3, 512, 128, 1 / math.sqrt(128)),
               (3, 512, 3, 1 / math.sqrt(3)), (3, 100, 33, 1.0), (1, 77, 256, 1 / 16)]


@pytest.mark.parametrize('case', STYLE_CASES, ids=[f'N{c[0]}-wd{c[1]}-C{c[2]}-post{c[3]:.3f}' for c in STYLE_CASES])
def test_styles_vs_float64(case):
    N, w_dim, Cin, post = case
    seed = 100 + STYLE_CASES.index(case)
    w, A, a = _randn(seed, N, w_dim), _randn(seed + 1000, Cin, w_dim), 1 + 0.1 * _randn(seed + 2000, Cin)
    s = _styles(w, A, a, post)
    post32 = float(np.float32(post))                                        # the value the kernel multiplies by
    ref, S = scr.styles(w.double(), A.double(), a.double(), post32), scr.styles_abs(w.double(), A.double(), a.double(), post32)
    scr.check_bound(s, ref, S, scr.ALPHA_F32, scr.BETA['fp32'], tag=f'styles N={N} w_dim={w_dim} Cin={Cin} post={post:.4f}')
    if N > 1:
        for k in range(N):
            assert torch.equal(_bits(_styles(w[k:k + 1].contiguous(), A, a, post)), _bits(s[k:k + 1])), f'styles: sample {k} of N={N} vs N=1'


# ---- (b) fold ----------------------------------------------------------------------------------------------------------------------------
def _fold(W, s, demod):
    O, I, k, _ = W.shape
    N = s.shape[0]
    buf, wf = _canary((N, O, I, k, k))
    capi.check(capi.lib().r3dp_sr_fold_weights(capi.ptr(W), capi.ptr(s), N, O, I, k, int(demod), capi.ptr(wf), capi.stream()))
    torch.cuda.synchronize()
    _check_canary(buf, 'folded weights')
    return wf


# N, O, I, k, demod, weight scale.  The production sizes of the SR layers (k = 3) and ToRGB (k = 1); O, I that are multiples of neither
# 8 nor 32; and small weights, where the demodulation epsilon 1e-8 is 2e-4 of the sum of squares.
FOLD_CASES = [(3, 256, 32, 3, True, 1.0), (3, 256, 256, 3, True, 1.0), (3, 128, 256, 3, True, 1.0), (3, 128, 128, 3, True, 1.0),
              (3, 37, 13, 3, True, 1.0), (2, 5, 3, 3, True, 1e-3), (3, 3, 256, 1, False, 1.0), (3, 3, 128, 1, False, 1.0),
              (2, 3, 37, 1, False, 1.0)]


@pytest.mark.parametrize('case', FOLD_CASES, ids=[f'N{c[0]}-O{c[1]}-I{c[2]}-k{c[3]}-demod{int(c[4])}-scale{c[5]:g}' for c in FOLD_CASES])
def test_fold_weights_vs_float64(case):
    N, O, I, k, demod, scale = case
    seed = 200 + FOLD_CASES.index(case)
    W, s = scale * _randn(seed, O, I, k, k), 1 + _randn(seed + 1000, N, I)        # N different styles
    wf = _fold(W, s, demod)
    ref, E = scr.fold_error(W.double(), s.double(), torch.zeros(N, I, device=DEV, dtype=torch.float64), demod)
    _check(wf, ref, E, f'fold N={N} O={O} I={I} k={k} demod={int(demod)} scale={scale:g}')
    assert torch.equal(_bits(_fold(W, s[N - 1:].contiguous(), demod)), _bits(wf[N - 1:])), 'fold: last sample of N vs N=1'


# ---- (c) SR layer ------------------------------------------------------------------------------------------------------------------------
def _layer(x, wf, bias, up):
    """r3dp_sr_layer_fp32 with canaries around the output and the up=2 scratch grid -> (y, grid or None)."""
    L = capi.lib()
    N, I, H, W = x.shape
    O = wf.shape[1]
    ybuf, y = _canary((N, O, H * up, W * up))
    gbuf = grid = None
    if up == 2:
        nbytes = L.r3dp_sr_layer_scratch_bytes(N, O, H, W)
        assert nbytes == N * O * (2 * H + 1) * (2 * W + 1) * 4
        gbuf, grid = _canary((N, O, 2 * H + 1, 2 * W + 1))
    capi.check(L.r3dp_sr_layer_fp32(capi.ptr(x), capi.ptr(wf), capi.ptr(bias), N, I, O, H, W, up, capi.ptr(y), capi.ptr(grid), capi.stream()))
    torch.cuda.synchronize()
    _check_canary(ybuf, 'layer output')
    if up == 2:
        _check_canary(gbuf, 'up=2 scratch grid')          # the four phase launches tile the (2H+1) x (2W+1) grid
    return y, grid


def _layer_reference(x, wf, bias, up):
    """[(name, ref, S, alpha, extra)] of the output and, for up=2, of the transposed-conv grid the kernel leaves in scratch."""
    x64, w64, b64 = x.double(), wf.double(), bias.double()
    gain = scr.act_gain(1)
    terms = []
    if up == 1:
        v, s, extra = scr.conv_same(x64, w64), scr.conv_same(x64.abs(), w64.abs()), None
    else:
        grid, sgrid = scr.conv_transposed(x64, w64), scr.conv_transposed(x64.abs(), w64.abs())
        terms.append(('grid', grid, sgrid, 0.0, None))
        v, s = scr.fir_up(grid), scr.fir_up(sgrid)
        extra = gain * scr.fir_up(scr.ALPHA_F32 * grid.abs())
    terms.insert(0, ('y', scr.bias_act(v, b64, 1), gain * (s + b64.abs().view(1, -1, 1, 1)), scr.ALPHA_FP32_LAYER, extra))
    return terms


# N, I, O, H, W, up.  Production shapes at N = 1, then edge shapes at N = 3 with per-sample weights.
LAYER_CASES = [
    (1, 32, 256, 128, 128, 2), (1, 256, 256, 256, 256, 1), (1, 256, 128, 256, 256, 2), (1, 128, 128, 512, 512, 1),
    (3, 1, 33, 1, 1, 1),          # one partial ci chunk, 1 x 1
    (3, 3, 40, 15, 31, 1),        # partial ci chunk, two co blocks (8 of the second used), a partial tile
    (3, 12, 1, 16, 32, 1),        # one full and one partial ci chunk, one output channel, exactly one tile
    (3, 40, 33, 17, 33, 1),       # five chunks, co block spill of 1, tiles spilling by one row and one column
    (3, 12, 40, 9, 70, 1),        # three tiles across, one down
    (3, 8, 32, 9, 70, 1),         # exactly one ci chunk and one co block
    (3, 3, 33, 16, 32, 2),        # phase grids 17 x 33: one tile + one row / column in each axis
    (3, 40, 40, 1, 1, 2),         # phase grids of 2 x 2, 1 x 2, 2 x 1, 1 x 1
    (3, 12, 1, 17, 33, 2),
    (3, 1, 40, 9, 70, 2),
    (3, 40, 33, 15, 31, 2),
]


def _layer_id(c):
    return f'N{c[0]}-I{c[1]}-O{c[2]}-{c[3]}x{c[4]}-up{c[5]}'


@pytest.mark.parametrize('case', LAYER_CASES, ids=[_layer_id(c) for c in LAYER_CASES])
def test_sr_layer_fp32_vs_float64(case):
    N, I, O, H, W, up = case
    seed = 300 + LAYER_CASES.index(case)
    x = _randn(seed, N, I, H, W)
    wf = _randn(seed + 1000, N, O, I, 3, 3) / math.sqrt(9 * I)         # per-sample folded weights
    bias = 0.5 * _randn(seed + 2000, O)
    y, grid = _layer(x, wf, bias, up)
    got = {'y': y, 'grid': grid}
    for name, ref, S, alpha, extra in _layer_reference(x, wf, bias, up):
        scr.check_bound(got[name], ref, S, alpha, scr.BETA['fp32'], extra, tag=f'layer {_layer_id(case)} {name}')
    y2, grid2 = _layer(x, wf, bias, up)
    assert torch.equal(_bits(y2), _bits(y)) and (up == 1 or torch.equal(_bits(grid2), _bits(grid))), 'repeated launch differs'
    if N > 1:
        for k in range(N):
            yk, gk = _layer(x[k:k + 1].contiguous(), wf[k:k + 1].contiguous(), bias, up)
            assert torch.equal(_bits(yk), _bits(y[k:k + 1])), f'image {k} of the N={N} launch vs its N=1 launch'
            assert up == 1 or torch.equal(_bits(gk), _bits(grid[k:k + 1])), f'grid of image {k} of the N={N} launch vs its N=1 launch'


# ---- (d) ToRGB ---------------------------------------------------------------------------------------------------------------------------
def _torgb(x, wrgb, bias, skip):
    N, I, H, W = x.shape
    buf, img = _canary((N, 3, H, W))
    capi.check(capi.lib().r3dp_sr_torgb_fp32(capi.ptr(x), capi.ptr(wrgb), capi.ptr(bias), capi.ptr(skip), N, I, H, W, capi.ptr(img),
                                             capi.stream()))
    torch.cuda.synchronize()
    _check_canary(buf, 'ToRGB image')
    return img


# N, I, H, W, skip image
TORGB_CASES = [(3, I, H, W, True) for I in (3, 128, 256) for H, W in ((2, 2), (18, 34))] + [
    (1, 256, 256, 256, True), (1, 128, 512, 512, True), (3, 128, 15, 31, False), (3, 3, 1, 1, False)]


def _torgb_id(c):
    return f'N{c[0]}-I{c[1]}-{c[2]}x{c[3]}-skip{int(c[4])}'


@pytest.mark.parametrize('case', TORGB_CASES, ids=[_torgb_id(c) for c in TORGB_CASES])
def test_torgb_fp32_vs_float64(case):
    N, I, H, W, with_skip = case
    seed = 400 + TORGB_CASES.index(case)
    x, wrgb, bias = _randn(seed, N, I, H, W), _randn(seed + 1000, N, 3, I) / math.sqrt(I), 1.5 * _randn(seed + 2000, 3)
    skip = _randn(seed + 3000, N, 3, H // 2, W // 2) if with_skip else None
    img = _torgb(x, wrgb, bias, skip)
    x64, w64, b64 = x.double(), wrgb.double(), bias.double().view(1, 3, 1, 1)
    ref, S = scr.torgb(x64, w64) + b64, scr.torgb(x64.abs(), w64.abs()) + b64.abs()
    if with_skip:
        ref, S = ref + scr.upsample2x(skip.double()), S + scr.upsample2x(skip.double().abs())
    scr.check_bound(img, ref, S, scr.ALPHA_F32, scr.BETA['fp32'], tag=f'torgb {_torgb_id(case)}')
    assert torch.equal(_bits(_torgb(x, wrgb, bias, skip)), _bits(img)), 'repeated launch differs'
    if N > 1:
        for k in range(N):
            one = _torgb(x[k:k + 1].contiguous(), wrgb[k:k + 1].contiguous(), bias, None if skip is None else skip[k:k + 1].contiguous())
            assert torch.equal(_bits(one), _bits(img[k:k + 1])), f'image {k} of the N={N} launch vs its N=1 launch'


# ---- (e) the chain from latent to weights ------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def sr_fp32():
    sr = r3.SuperresolutionHybrid8XDC(channels=32, img_resolution=512, sr_num_fp16_res=0, sr_antialias=True, sr_mode='fp32')
    sr.load_state_dict(syn.make_sr_params(seed=5), strict=True)
    return sr.to(DEV).eval()


def _chain_reference(lay, w, torgb):
    """(ref, E) of lay.folded_weight(w) in float64 from the module's parameters: styles (with 1 / sqrt(Cin) for ToRGB) within their bound
    2^-24 |s| + BETA['fp32'] S, plus 2^-24 |s| for the fp32 rounding of 1 / sqrt(Cin), carried through the fold by scr.fold_error."""
    A, a, W = (t.detach().double() for t in (lay.affine.weight, lay.affine.bias, lay.weight))
    post = 1 / math.sqrt(lay.in_channels) if torgb else 1.0
    s, S = scr.styles(w.double(), A, a, post), scr.styles_abs(w.double(), A, a, post)
    return scr.fold_error(W, s, 2 * scr.ALPHA_F32 * s.abs() + scr.BETA['fp32'] * S, not torgb)


CHAIN = ['block0.conv0', 'block0.conv1', 'block1.conv0', 'block1.conv1', 'block0.torgb', 'block1.torgb']


@pytest.mark.parametrize('name', CHAIN)
def test_folded_weight_from_latent_vs_float64(sr_fp32, name):
    lay = sr_fp32.get_submodule(name)
    torgb = name.endswith('torgb')
    w = _randn(500 + CHAIN.index(name), 3, 512)
    got = lay.folded_weight(w)
    ref, E = _chain_reference(lay, w, torgb)
    if torgb:
        ref, E = ref.reshape(got.shape), E.reshape(got.shape)
    _check(got, ref, E, f'{name}.folded_weight')


def _to_packed(t):
    """[Nw,O,I,3,3] -> the packed order [Nw,9,O,I]."""
    Nw, O, I = t.shape[:3]
    return t.reshape(Nw, O, I, 9).permute(0, 3, 1, 2)


def _to_packed_composed(G):
    """[Nw,O,I,4,3,3] -> the packed order [Nw,36,O,I]."""
    Nw, O, I = G.shape[:3]
    return G.permute(0, 3, 4, 5, 1, 2).reshape(Nw, 36, O, I)


@pytest.mark.parametrize('split', [False, True], ids=['tc', 'tcx'])
@pytest.mark.parametrize('name,composed', [('block0.conv0', True), ('block0.conv0', False), ('block1.conv0', False), ('block1.conv1', False)])
def test_packed_weights_from_latent_vs_float64(sr_fp32, name, composed, split):
    """sr_tc._pack / _pack_up_composed from a latent, read back, against the float64 chain plus the packing: with wf the kernel's folded
    weights (|wf - ref| <= E), the store rounds to alpha_store |wf| + floor; the composition adds <= 2^-21 compose(|wf|) (four fp32 fmas
    of exact products, see test_gpu_sr_conv_conformance) and carries E as compose(E)."""
    lay = sr_fp32.get_submodule(name)
    w = _randn(600 + CHAIN.index(name), 2, 512)
    wp = (sr_tc._pack_up_composed if composed else sr_tc._pack)(lay, w, split)
    torch.cuda.synchronize()
    ref, E = _chain_reference(lay, w, False)
    if composed:
        ref, X = scr.compose_up_weights(ref), 2.0 ** -21 * scr.compose_up_weights(ref.abs() + E) + scr.compose_up_weights(E)
        ref, X = _to_packed_composed(ref), _to_packed_composed(X)
    else:
        ref, X = _to_packed(ref), _to_packed(E)
    floor = scr.FLOOR_F16 / (scr.SPLIT_WEIGHT_SCALE if split else 1.0)
    bound = scr.alpha_store(split) * (ref.abs() + X) + floor + X
    _check(scr.packed_weights(wp, lay.in_channels, split), ref, bound, f'{"tcx" if split else "tc"} {name} packed{" composed" if composed else ""}')


# ---- (f) the whole SR --------------------------------------------------------------------------------------------------------------------
def _superres64(rgb, x, ws):
    p = {k: v.double().to(DEV) for k, v in syn.make_sr_params(seed=5).items()}
    with torch.device(DEV):
        return orc.superres(rgb.double(), x.double(), ws.double(), p)


@pytest.mark.parametrize('size', [64, 128], ids=['resized-64', 'direct-128'])
def test_sr_fp32_vs_float64(sr_fp32, size, monkeypatch):
    """N = 2 with different ws: the fp32 SR image within TAU * range of float64; the float64 SR on fp16-rounded folded weights is not;
    image k of the N = 2 run equals the N = 1 run of image k bit for bit."""
    g = torch.Generator(device=DEV).manual_seed(700 + size)
    x = torch.rand(2, 32, size, size, generator=g, device=DEV) * 2 - 1
    rgb = x[:, :3].contiguous()
    ws = 1 + 0.3 * torch.randn(2, 14, 512, generator=g, device=DEV)
    with torch.no_grad():
        img = sr_fp32(rgb, x, ws, noise_mode='none')
        ref = _superres64(rgb, x, ws)
        rng = float(ref.max() - ref.min())
        err = float((img.double() - ref).abs().max())
        fold64 = orc.fold_weight
        monkeypatch.setattr(orc, 'fold_weight', lambda W, s, demod: fold64(W, s, demod).half().double())
        err16 = float((_superres64(rgb, x, ws) - ref).abs().max())
        monkeypatch.undo()
        print(f'fp32 SR {size}->512 vs float64: max |err| {err:.3e} = {err / rng:.3e} x range {rng:.3f} (tau {TAU:.1e}); '
              f'float64 on fp16 folded weights: {err16 / rng:.3e} x range')
        assert err <= TAU * rng, (err, rng)
        assert err16 > TAU * rng, (err16, rng)
        for k in range(2):
            one = sr_fp32(rgb[k:k + 1].contiguous(), x[k:k + 1].contiguous(), ws[k:k + 1].contiguous(), noise_mode='none')
            assert torch.equal(_bits(one), _bits(img[k:k + 1])), f'image {k} of the N=2 run vs its N=1 run'
