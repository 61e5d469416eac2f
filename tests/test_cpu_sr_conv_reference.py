"""The float64 references of tests/sr_conv_reference.py on the CPU, so that the GPU conformance suite is not their first run: they agree
with the fp32 oracle, the composed up weights reproduce the two-step up convolution, and the error bound with the chosen beta accepts a
simulation of the `tc` arithmetic and rejects the same simulation with one weight tap dropped."""
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
