"""The float64 references of tests/sr_conv_reference.py on the CPU, so that the GPU conformance suites are not their first run: they agree
with the fp32 oracle, the composed up weights reproduce the two-step up convolution, and the error bound with the chosen beta accepts a
simulation of the `tc` arithmetic and rejects the same simulation with one weight tap dropped.  For the exact-fp32 path: the styles and
fold helpers agree with the oracle, the fold bound carries a styles error through the demodulation, and at the largest K BETA['fp32']
accepts a float32 simulation of the layer and rejects fp16 or TF32 weights, a dropped tap and a permuted FIR."""
import math

import pytest
import torch
import torch.nn.functional as F

import sr_conv_reference as scr
from oracle import real3d_oracle as orc


def _rand(*shape, seed, dtype=torch.float32):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=dtype)


def _close(a, b, rel):
    err, mag = float((a.double() - b.double()).abs().max()), float(b.double().abs().max())
    assert err <= rel * mag, (err, mag)


def test_float64_helpers_match_the_fp32_oracle():
    N, I, O, H, W = 2, 8, 16, 5, 6
    x, w, b = _rand(N, I, H, W, seed=1), _rand(N, O, I, 3, 3, seed=2) / 8, _rand(O, seed=3)
    x64, w64, b64 = x.double(), w.double(), b.double()
    _close(scr.conv_same(x64, w64), orc.mod_conv(x, w, 1), 1e-5)
    _close(scr.conv_same(x64, w64, ksize=1), torch.cat([F.conv2d(x[n:n + 1], w[n][..., 1:2, 1:2]) for n in range(N)]), 1e-5)
    _close(scr.fir_up(scr.conv_transposed(x64, w64)), orc.mod_conv(x, w, 2), 1e-5)
    v, v64 = orc.mod_conv(x, w, 1), orc.mod_conv(x, w, 1).double()
    _close(scr.bias_act(v64, b64, 1), orc.lrelu_gain(v, b), 1e-6)
    _close(scr.bias_act(v64, b64, 2), F.leaky_relu(v + b.view(1, -1, 1, 1), 0.01), 1e-6)
    _close(scr.bias_act(v64, b64, 3), torch.relu(v + b.view(1, -1, 1, 1)), 1e-6)
    _close(scr.bias_act(v64, b64, 0), v + b.view(1, -1, 1, 1), 1e-6)
    wr = _rand(N, 3, O, seed=4)
    _close(scr.torgb(v64, wr.double()), torch.cat([F.conv2d(v[n:n + 1], wr[n][..., None, None]) for n in range(N)]), 1e-5)
    img = _rand(N, 3, H, W, seed=5)
    _close(scr.upsample2x(img.double()), orc.upsample2x(img), 1e-6)
    frames = scr.to_uint8(torch.tensor([-1.0, -0.5, 0.0, 0.999, 1.0]).view(1, 1, 1, 5).expand(1, 3, 1, 5))   # truncation, HWC
    assert frames.shape == (1, 1, 5, 3) and frames[0, 0, :, 1].tolist() == [0, 63, 127, 254, 255]


def test_composed_up_weights_reproduce_the_two_step_up_conv():
    N, I, O, H, W = 2, 5, 7, 6, 9
    x, w = _rand(N, I, H, W, seed=6, dtype=torch.float64), _rand(N, O, I, 3, 3, seed=7, dtype=torch.float64)
    G = scr.compose_up_weights(w).permute(0, 3, 1, 2, 4, 5)                       # [N,O,I,4,3,3] -> [N,4,O,I,3,3]
    two_step = scr.fir_up(scr.conv_transposed(x, w))
    assert float((scr.conv_up_composed(x, G) - two_step).abs().max()) <= 1e-12 * float(two_step.abs().max())


def _tc_simulation(x16, w16, b):
    """The `tc` arithmetic on the CPU: fp16 operands, a float32 conv, bias and lrelu * sqrt2 in float32, fp16 output."""
    return orc.lrelu_gain(F.conv2d(x16.float(), w16.float(), padding=1), b).half()


def test_bound_accepts_tc_arithmetic_and_rejects_a_dropped_tap():
    N, I, O, H, W = 1, 64, 128, 6, 16
    x16 = _rand(N, I, H, W, seed=8).half()
    w16 = (_rand(O, I, 3, 3, seed=9) / math.sqrt(9 * I)).half()
    b = 0.5 * _rand(O, seed=10)
    x64, w64, b64 = x16.double(), w16.double()[None], b.double()
    ref = scr.bias_act(scr.conv_same(x64, w64), b64, 1)
    S = scr.act_gain(1) * (scr.conv_same(x64.abs(), w64.abs()) + b64.abs().view(1, -1, 1, 1))
    scr.check_bound(_tc_simulation(x16, w16, b), ref, S, scr.ALPHA_F16, scr.BETA['tc'], tag='tc simulation')
    w_drop = w16.clone()
    w_drop[..., 0, 0] = 0
    with pytest.raises(AssertionError, match='outside the bound'):
        scr.check_bound(_tc_simulation(x16, w_drop, b), ref, S, scr.ALPHA_F16, scr.BETA['tc'], tag='tc simulation, tap (0, 0) dropped')


# ---- the exact-fp32 path ---------------------------------------------------------------------------------------------------------------
def test_styles_and_fold_helpers_match_the_fp32_oracle():
    N, wd, I, O = 3, 100, 12, 7
    w, A, a = _rand(N, wd, seed=20), _rand(I, wd, seed=21), 1 + 0.1 * _rand(I, seed=22)
    post = 1 / math.sqrt(I)
    s64 = scr.styles(w.double(), A.double(), a.double(), post)
    _close(s64, orc.affine_styles(w, A, a) * post, 1e-6)
    assert torch.equal(scr.styles_abs(w.double(), A.double(), a.double(), post), scr.styles(w.double().abs(), A.double().abs(), a.double().abs(), post))
    W = _rand(O, I, 3, 3, seed=23)
    for demod in (True, False):
        _close(scr.fold(W.double(), s64, demod), orc.fold_weight(W, s64.float(), demod), 1e-6)
    assert torch.equal(scr.fold_abs(W.double(), -s64), scr.fold(W.double().abs(), s64.abs(), False))
    ref, E = scr.fold_error(W.double(), s64, torch.zeros_like(s64), True)
    assert torch.allclose(E, scr.fold_alpha(9 * I, True) * ref.abs(), rtol=1e-9, atol=0)


@pytest.mark.parametrize('demod', [True, False])
def test_fold_error_covers_perturbed_styles(demod):
    """fold_error's first-order propagation holds for styles moved by up to ds in float64, where the kernel's own roundings play no part."""
    N, I, O, k = 4, 24, 16, 3 if demod else 1
    W, s = _rand(O, I, k, k, seed=24, dtype=torch.float64), 1 + _rand(N, I, seed=25, dtype=torch.float64)
    ds = 1e-4 * (s.abs() + 1)
    ref, E = scr.fold_error(W, s, ds, demod)
    for seed in range(4):
        moved = s + ds * torch.sign(_rand(N, I, seed=26 + seed, dtype=torch.float64))
        assert bool(((scr.fold(W, moved, demod) - ref).abs() <= E).all())
        assert float(((scr.fold(W, moved, demod) - ref).abs() / E).max()) > 0.05                  # and is not vacuous


def _fir_f32(grid, taps):
    """The fp32 FIR pass of the up path with per-axis taps (the kernel's are (0.25, 0.75, 0.75, 0.25)), pad 1."""
    gp = F.pad(grid, (1, 1, 1, 1))
    Ho, Wo = gp.shape[-2] - 3, gp.shape[-1] - 3
    out = torch.zeros(*grid.shape[:-2], Ho, Wo, dtype=grid.dtype)
    for u in range(4):
        for v in range(4):
            out = out + (taps[u] * taps[v]) * gp[..., u:u + Ho, v:v + Wo]
    return out


def _fp32_simulation(x, w, b, up, taps=scr.G4):
    """The fp32 path's arithmetic on the CPU: a float32 conv (up=2: transposed conv to an fp32 grid, then the FIR), bias and lrelu * sqrt2
    in float32."""
    v = F.conv2d(x, w, padding=1) if up == 1 else _fir_f32(F.conv_transpose2d(x, w.transpose(0, 1), stride=2), taps)
    return orc.lrelu_gain(v, b)


def _tf32(t):
    """Mantissa cut to 10 bits (TF32 operands)."""
    return (t.view(torch.int32) & ~0x1FFF).view(torch.float32)


@pytest.mark.parametrize('up', [1, 2])
def test_fp32_bound_accepts_fp32_arithmetic_and_rejects_lower_precision_and_wrong_taps(up):
    """At the suite's largest K (I = 256, 9 * 256 products per output), BETA['fp32'] accepts the fp32 layer and rejects fp16 or TF32
    weights, a dropped tap and (up=2) a permuted FIR."""
    assert scr.BETA['fp32'] <= scr.gamma(9 * 256)
    N, I, O, H, W = 1, 256, 64, 8, 16
    x = _rand(N, I, H, W, seed=30)
    w = _rand(O, I, 3, 3, seed=31) / math.sqrt(9 * I)
    b = 0.5 * _rand(O, seed=32)
    x64, w64, b64 = x.double(), w.double()[None], b.double()
    gain = scr.act_gain(1)
    if up == 1:
        v, s, extra = scr.conv_same(x64, w64), scr.conv_same(x64.abs(), w64.abs()), None
    else:
        grid = scr.conv_transposed(x64, w64)
        v, s = scr.fir_up(grid), scr.fir_up(scr.conv_transposed(x64.abs(), w64.abs()))
        extra = gain * scr.fir_up(scr.ALPHA_F32 * grid.abs())
    ref, S = scr.bias_act(v, b64, 1), gain * (s + b64.abs().view(1, -1, 1, 1))

    def check(got, tag):
        return scr.check_bound(got, ref, S, scr.ALPHA_FP32_LAYER, scr.BETA['fp32'], extra, tag=f'fp32 simulation up={up}{tag}')
    check(_fp32_simulation(x, w, b, up), '')
    w_drop = w.clone()
    w_drop[..., 1, 2] = 0
    bad = {'fp16 weights': _fp32_simulation(x, w.half().float(), b, up), 'TF32 weights': _fp32_simulation(x, _tf32(w), b, up),
           'tap (1, 2) dropped': _fp32_simulation(x, w_drop, b, up)}
    if up == 2:
        bad['FIR taps permuted'] = _fp32_simulation(x, w, b, up, taps=(0.75, 0.25, 0.25, 0.75))
    for tag, got in bad.items():
        with pytest.raises(AssertionError, match='outside the bound'):
            check(got, ', ' + tag)
