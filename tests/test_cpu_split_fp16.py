"""The tensor-core OSG decoder (render.cu, MlpTcImage) feeds wgmma with fp16 operands and still claims fp32-grade results: every fp32
operand is split as v = hi + lo (two fp16 numbers) and the products hi*hi + lo*hi + hi*lo are accumulated in fp32.  This CPU test
restates that arithmetic with numpy on decoder-shaped data (SURVEY.md Appendix A: 32 -> 64 softplus -> 33, gains 1/sqrt(fan_in)) and
bounds its error against float64, next to plain fp32 and plain fp16 evaluations of the same layer."""
import numpy as np


def _split(v):
    hi = v.astype(np.float16)
    lo = (v - hi.astype(np.float32)).astype(np.float16)
    return hi.astype(np.float32), lo.astype(np.float32)


def _gemm_split(x, w):
    """x [M,K], w [N,K] fp32 -> the three significant partial products, summed in fp32 (tensor-core accumulation is fp32)."""
    xh, xl = _split(x)
    wh, wl = _split(w)
    return (xh @ wh.T + xl @ wh.T + xh @ wl.T).astype(np.float32)


def _softplus(v):
    return np.logaddexp(v, 0.0)


def test_split_reconstructs_fp32_operands_to_22_bits():
    rng = np.random.default_rng(0)
    v = (rng.standard_normal(1 << 16) * np.exp(rng.uniform(-6, 3, 1 << 16))).astype(np.float32)      # 2^-9 .. 2^4 magnitudes
    hi, lo = _split(v)
    err = np.abs((hi.astype(np.float64) + lo.astype(np.float64)) - v.astype(np.float64))
    assert np.all(err <= np.abs(v) * 2.0 ** -21 + 2.0 ** -25)                   # + the fp16 subnormal floor of the low half


def test_decoder_layers_match_float64_like_fp32_does():
    rng = np.random.default_rng(1)
    M = 4096
    x = (rng.standard_normal((M, 32)) * 0.6).astype(np.float32)                 # mean of three N(0,1) plane samples
    w1 = (rng.standard_normal((64, 32)) / np.sqrt(32)).astype(np.float32)
    b1 = (0.1 * rng.standard_normal(64)).astype(np.float32)
    w2 = (rng.standard_normal((33, 64)) / np.sqrt(64)).astype(np.float32)
    b2 = (0.1 * rng.standard_normal(33)).astype(np.float32)

    h64 = _softplus(x.astype(np.float64) @ w1.astype(np.float64).T + b1)
    y64 = h64 @ w2.astype(np.float64).T + b2

    h_split = _softplus(_gemm_split(x, w1) + b1).astype(np.float32)
    y_split = _gemm_split(h_split, w2) + b2
    h_f32 = _softplus(x @ w1.T + b1).astype(np.float32)
    y_f32 = h_f32 @ w2.T + b2
    h_f16 = _softplus((x.astype(np.float16).astype(np.float32) @ w1.astype(np.float16).astype(np.float32).T) + b1).astype(np.float32)
    y_f16 = h_f16.astype(np.float16).astype(np.float32) @ w2.astype(np.float16).astype(np.float32).T + b2

    e_split, e_f32, e_f16 = (float(np.abs(v - y64).max()) for v in (y_split, y_f32, y_f16))
    assert e_split < 5e-6                                                      # fp32-grade: outputs are O(1)
    assert e_split < 4.0 * e_f32 + 1e-6                                        # same league as evaluating in fp32
    assert e_f16 > 50.0 * e_split                                              # and far from what plain fp16 operands would give
    # the rendered colour is sigmoid(y) * 1.002 - 0.001: Lipschitz 0.25 -> well inside the 1e-4 the GPU tests assert
    assert 0.25 * 1.002 * e_split < 1e-5
