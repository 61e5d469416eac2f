"""conv3d.pack_conv3d, the one packer of r3dp_mf_conv3d's weights, against a restatement of the format the kernel reads (include/r3dp_b200.h,
csrc/conv3d_tc.cu): wp[phase][tap][co][ci] with tap = (z * kh + y) * kw + x, output channels padded with zero filters to the cout tile
(16, 32, 64, then multiples of 128), the I logical input channels at their cin_map positions of the cin the kernel reads and zero
elsewhere; split: [hi | lo] with hi = fp16(w * 2^10), lo = fp16(w * 2^10 - hi).  Also the GEMM ([O, K] on 1x1x1 taps) and 3x3 forms the
plane backbones pack (pack_gemm, pack_taps), read back as the kernel reads them and applied against float64 of the fp16 weights."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from real3dportrait_b200 import conv3d

#: cout -> cop as the kernel tiles it
COP = [(1, 16), (5, 16), (16, 16), (17, 32), (32, 32), (33, 64), (64, 64), (65, 128), (96, 128), (128, 128), (130, 256), (512, 512),
       (1000, 1024)]


def _w(*shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


def _restated(w, cin, cop, cin_map, split):
    """float64 [nph,O,I,kd,kh,kw] -> the packed array, element by element (numpy float16; torch rounds float64 to fp16 through fp32)."""
    nph, O, I, kd, kh, kw = w.shape
    cmap = list(range(I)) if cin_map is None else cin_map
    s = w.numpy() * (1024.0 if split else 1.0)
    out = np.zeros((nph, kd * kh * kw, cop, cin * (2 if split else 1)), dtype=np.float16)
    for p in range(nph):
        for z in range(kd):
            for y in range(kh):
                for x in range(kw):
                    t = (z * kh + y) * kw + x
                    for o in range(O):
                        for i in range(I):
                            v = s[p, o, i, z, y, x]
                            hi = np.float16(np.float32(v))
                            out[p, t, o, cmap[i]] = hi
                            if split:
                                out[p, t, o, cin + cmap[i]] = np.float16(np.float32(v - np.float64(hi)))
    return out


@pytest.mark.parametrize('cout,cop', COP)
def test_cop(cout, cop):
    assert conv3d.cout_pad(cout) == cop
    pk = conv3d.pack_conv3d(_w(1, cout, 3, 1, 1, 1, seed=cout), None, 32, False)
    assert (pk.cout, pk.cop) == (cout, cop) and tuple(pk.w.shape) == (1, 1, cop, 32)


def test_ceil32():
    assert [conv3d.ceil32(n) for n in (1, 13, 25, 32, 33, 50, 89, 1024)] == [32, 32, 32, 32, 64, 64, 96, 1024]


# (nph, O, I, taps, cin, cin_map): the estimator's 3x3x3 down conv, the 4 nearest-up phases of (3, 2, 2), the fuser's channel map (K = 4),
# a 1x7x7 head conv, the VAE's k3 taps along W, and a ragged cout tile
CASES = [(1, 20, 25, (3, 3, 3), 32, None), (4, 9, 40, (3, 2, 2), 64, None), (1, 7, 29, (2, 3, 3), 96, list(range(25)) + [32, 33, 34, 35]),
         (1, 33, 4, (1, 7, 7), 32, None), (1, 70, 60, (1, 1, 3), 64, None), (1, 130, 32, (1, 1, 1), 32, None)]


@pytest.mark.parametrize('split', [False, True])
@pytest.mark.parametrize('case', range(len(CASES)))
def test_layout(case, split):
    nph, O, I, taps, cin, cin_map = CASES[case]
    w = _w(nph, O, I, *taps, seed=case) * 3.0
    b = _w(O, seed=100 + case)
    pk = conv3d.pack_conv3d(w, b, cin, split, cin_map=cin_map)
    cop = conv3d.cout_pad(O)
    assert (pk.cout, pk.cop) == (O, cop)
    assert pk.w.dtype == torch.float16 and pk.w.is_contiguous()
    want = _restated(w, cin, cop, cin_map, split)
    assert tuple(pk.w.shape) == want.shape
    assert np.array_equal(pk.w.numpy().view(np.int16), want.view(np.int16))            # bit for bit: tap order, zero rows, channel map
    assert pk.bias.dtype == torch.float32 and tuple(pk.bias.shape) == (cop,)
    assert torch.equal(pk.bias[:O], b.float()) and not bool(pk.bias[O:].any())
    if split:
        hi, lo = pk.w[..., :cin].double(), pk.w[..., cin:].double()
        s = torch.zeros_like(hi)                                                         # w * 2^10 where packed, else 0
        cmap = list(range(I)) if cin_map is None else cin_map
        s[..., :O, cmap] = w.permute(0, 3, 4, 5, 1, 2).reshape(nph, -1, O, I) * 1024.0
        assert bool((hi - s).abs().le(2.0 ** -11 * s.abs() + 2.0 ** -25).all())         # hi: w * 2^10 to fp16 rounding
        assert torch.equal(lo, (s - hi).half().double())                                 # lo: the fp16 of the residual
        assert bool(((hi + lo) / 1024.0 - s / 1024.0).abs().le(2.0 ** -22 * s.abs() / 1024.0 + 2.0 ** -35).all())


def test_zero_bias():
    pk = conv3d.pack_conv3d(_w(1, 20, 32, 1, 1, 1, seed=3), None, 32, True)
    assert tuple(pk.bias.shape) == (32,) and not bool(pk.bias.any())


def test_gemm_form():
    """[O, K] weights on 1x1x1 taps (the backbones' token GEMMs): rows x @ W^T as the kernel reads wp."""
    O, K, R = 40, 96, 7
    w, b, x = _w(O, K, seed=4), _w(O, seed=5), _w(R, K, seed=6)
    pk = conv3d.pack_gemm(w, b, 'cpu')
    assert tuple(pk.w.shape) == (64, K) and (pk.cout, pk.cop) == (O, 64)
    got = x @ pk.w.double()[:O].T + pk.bias.double()[:O]
    assert torch.equal(got, x @ w.half().double().T + b.float().double())


def test_3x3_form():
    """[O, I, 3, 3] conv weights on 1x3x3 taps (the backbones' stride-1 3x3 convs): the sum over taps t = ky * 3 + kx of shifted inputs
    times wp[0, t] equals the padded conv of the fp16 weights."""
    O, I, H, W = 18, 32, 5, 6
    w, b, x = _w(O, I, 3, 3, seed=7), _w(O, seed=8), _w(1, I, H, W, seed=9)
    pk = conv3d.pack_taps(w, b, 'cpu')
    assert tuple(pk.w.shape) == (9, 32, I) and torch.equal(pk.bias[:O], b.float())
    xp = F.pad(x, (1, 1, 1, 1))
    got = torch.zeros(1, O, H, W, dtype=torch.float64)
    for ky in range(3):
        for kx in range(3):
            got += torch.einsum('oi,nihw->nohw', pk.w[ky * 3 + kx, :O].double(), xp[..., ky:ky + H, kx:kx + W])
    want = F.conv2d(x, w.half().double(), padding=1)
    assert float((got - want).abs().max()) < 1e-12
