"""HuBERT on the GPU: r3dp_hb_gemm at every (N, K, epilogue) of the hubert-large forward and r3dp_hb_attention on mixed segment batches,
each against float64 of the split operands they read, with sentinel guards; the small config against the reference's extract_hubert
(fixture) and the float64 chunk loop at its edges up to T = 30 001; hubert-large with formula weights against the float64 restatement,
up to three launch groups; all within hubert_reference.E2E_BAR; out=, determinism and CUDA-graph capture, one group and three."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import hubert_reference as hr  # noqa: E402
from launch_harness import guarded, guards_intact  # noqa: E402
from real3dportrait_b200 import _capi as capi  # noqa: E402
from real3dportrait_b200 import hubert as hb  # noqa: E402
from real3dportrait_b200 import HubertModel, get_hubert_from_16k_speech, hubert_frames  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = 'cuda'
LARGE = dict(conv_dim=(512,) * 7, hidden_size=1024, num_attention_heads=16, intermediate_size=4096, num_hidden_layers=24,
             num_conv_pos_embeddings=128, num_conv_pos_embedding_groups=16, feat_extract_norm='layer', do_stable_layer_norm=True,
             conv_bias=True)


def split_rows(x):
    """fp32/64 [M, K] -> (split rows [M, hi K | lo K] fp16, the value they represent, float64)."""
    h = x.half()
    lo = (x - h.double() if x.dtype == torch.float64 else x - h.float()).half()
    return torch.cat([h, lo], 1).contiguous(), h.double() + lo.double()


def weights(N, K, seed):
    g = torch.Generator(device='cpu').manual_seed(seed)
    w = torch.randn(N, K, generator=g, dtype=torch.float64) / np.sqrt(K)
    return w


def packed_value(wp, K):
    return (wp[:, :K].double() + wp[:, K:].double()) / 1024.0


# (N, K, epi) of every r3dp_hb_gemm launch of the hubert-large forward: conv layers 1-6 (windows), projection, QKV, out_proj, FFN in / out
CONV = [(512, 3 * 512, 3, 3, 2), (512, 2 * 512, 3, 2, 2)]
DENSE = [(1024, 512, 3), (3072, 1024, 0), (1024, 1024, 2), (4096, 1024, 1), (1024, 4096, 2)]
MS = [1, 63, 64, 65, 127, 128, 129, 1000, 1031, 30000]


def run_gemm(A, M, width, stride, seg, wp, N, Kp, bias, epi, y, ldy, ylo):
    capi.check(capi.lib().r3dp_hb_gemm(ctypes.c_void_p(A.data_ptr()), M, width, stride, seg, capi.ptr(wp, torch.float16), N, Kp, capi.ptr(bias), epi,
                                       ctypes.c_void_p(y.data_ptr()), ldy, ylo, capi.stream()))


@pytest.mark.parametrize('M', MS)
@pytest.mark.parametrize('case', DENSE + CONV, ids=lambda c: '_'.join(map(str, c)))
def test_gemm(case, M):
    torch.manual_seed(M)
    if len(case) == 5:
        N, K, epi, k, s = case
        C = 512
        F = (M - 1) * s + k
        x = torch.randn(F, C, device=DEV).mul_(2.0)
        Arows, xv = split_rows(x)
        X = xv.unfold(0, k, s).permute(0, 2, 1).reshape(M, k * C)                # window rows, K channel j C + i
        width, stride, seg = k * 2 * C, s * 2 * C, C
    else:
        N, K, epi = case
        x = torch.randn(M, K, device=DEV).mul_(2.0)
        Arows, X = split_rows(x)
        width, stride, seg = 2 * K, 2 * K, K
    w = weights(N, K, 7 + N + K)
    wp = hb.pack_split(w).to(DEV)
    W = packed_value(wp, K)
    bias = torch.randn(N, device=DEV)
    ref = X @ W.t() + bias.double()
    mag = X.abs() @ W.abs().t()
    if epi in (0, 1):
        if epi == 1:
            ref = hr.gelu(ref)
        buf, y = guarded(M * 2 * N, torch.float16, fill=-7.0, device=DEV)
        run_gemm(Arows, M, width, stride, seg, wp, N, K, bias, epi, y, 2 * N, N)
        torch.cuda.synchronize()
        y = y.view(M, 2 * N)
        got = y[:, :N].double() + y[:, N:].double()
        assert guards_intact(buf, y.numel(), fill=-7.0)
    else:
        init = torch.randn(M, N, device=DEV) if epi == 2 else None
        buf, y = guarded(M * N, torch.float32, fill=float('nan') if epi == 3 else 0.0, device=DEV)
        if epi == 2:
            y.copy_(init.view(-1))
            ref = ref + init.double()
        run_gemm(Arows, M, width, stride, seg, wp, N, K, bias, epi, y, N, 0)
        torch.cuda.synchronize()
        got = y.view(M, N).double()
        assert guards_intact(buf, y.numel(), fill=float('nan') if epi == 3 else 0.0)
    bar = 2.0 ** -17 * mag * (1.8 if epi == 1 else 1.0) + 2.0 ** -20 * ref.abs() + 1e-30
    ratio = float(((got - ref).abs() / bar).max())
    print(f'gemm {case} M={M}: worst err/bar {ratio:.3f}')
    assert ratio <= 1.0, ratio


def test_gemm_residual_leaves_other_rows():
    M, N, K = 129, 1024, 1024
    x = torch.randn(M, K, device=DEV)
    A, _ = split_rows(x)
    wp = hb.pack_split(weights(N, K, 3)).to(DEV)
    y = torch.randn(M + 64, N, device=DEV)
    keep = y.clone()
    run_gemm(A, M, 2 * K, 2 * K, K, wp, N, K, torch.zeros(N, device=DEV), 2, y, N, 0)
    torch.cuda.synchronize()
    assert torch.equal(y[M:], keep[M:])


def attention_ref(qkv, segs, H):
    """float64 softmax(q k^T) v per segment from the split rows' values."""
    V = qkv[:, :3 * H].double() + qkv[:, 3 * H:].double()
    out, s0 = [], 0
    heads = H // 64
    for L in segs:
        o, mag = torch.empty(L, H, dtype=torch.float64, device=DEV), torch.empty(L, H, dtype=torch.float64, device=DEV)
        for hd in range(heads):                     # one head at a time: a 15000-frame segment's T x T scores fit in memory
            q, k, v = (V[s0:s0 + L, j * H + 64 * hd:j * H + 64 * hd + 64] for j in range(3))
            P = torch.softmax(q @ k.t(), -1)
            o[:, 64 * hd:64 * hd + 64] = P @ v
            mag[:, 64 * hd:64 * hd + 64] = (q.abs() @ k.abs().t()).amax(-1, keepdim=True) * v.abs().amax(0, keepdim=True) + P @ v.abs()
            del P
        out.append((o, mag))
        s0 += L
    return torch.cat([o for o, _ in out]), torch.cat([m for _, m in out])


@pytest.mark.parametrize('segs', [[1, 2, 63, 64, 65, 127, 128, 129, 999, 1000, 31], [1000] * 3 + [17], [15000]],
                         ids=['mixed', 'segments', 'long'])
def test_attention(segs):
    H = 1024
    R = sum(segs)
    torch.manual_seed(len(segs))
    x = torch.randn(R, 3 * H, device=DEV) * 2.0
    qkv, _ = split_rows(x)
    buf, o = guarded(R * 2 * H, torch.float16, fill=-7.0, device=DEV)
    lens = (ctypes.c_int * len(segs))(*segs)
    capi.check(capi.lib().r3dp_hb_attention(capi.ptr(qkv, torch.float16), R, 6 * H, 3 * H, 16, lens, len(segs), ctypes.c_void_p(o.data_ptr()),
                                            2 * H, H, capi.stream()))
    torch.cuda.synchronize()
    assert guards_intact(buf, o.numel(), fill=-7.0)
    o = o.view(R, 2 * H)
    got = o[:, :H].double() + o[:, H:].double()
    ref, mag = attention_ref(qkv, segs, H)
    bar = 2.0 ** -17 * mag + 2.0 ** -20 * ref.abs()
    ratio = float(((got - ref).abs() / bar).max())
    print(f'attention {segs[:4]}...: worst err/bar {ratio:.3f}')
    assert ratio <= 1.0, ratio


# ---- whole model --------------------------------------------------------------------------------------------------------------------
def load_fixture():
    z = np.load(os.path.join(ROOT, 'tests', 'golden', 'hubert_small.npz'))
    return z


def small_model():
    z = load_fixture()
    cfg = {k[7:]: (tuple(z[k].tolist()) if z[k].ndim else z[k].item()) for k in z.files if k.startswith('config.')}
    m = HubertModel(cfg)
    sd = hr.formula_params({k: tuple(v.shape) for k, v in m.state_dict().items()})
    m.load_state_dict({k: v.float() for k, v in sd.items()}, strict=True)
    return m.to(DEV), z


@pytest.mark.parametrize('L', [400, 4000, 330000])
def test_small_against_fixture(L):
    m, z = small_model()
    ref = torch.from_numpy(z[f'hubert_{L}']).double()
    got = get_hubert_from_16k_speech(hr.wave(L), m).double().cpu()
    assert got.shape == ref.shape
    err = float((got - ref).abs().max()) / float(ref.abs().max())
    print(f'small L={L}: max|err| / max|ref| = {err:.2e} (bar {hr.E2E_BAR:.0e})')
    assert err <= hr.E2E_BAR


@pytest.mark.parametrize('k', [1, 4, 30])
@pytest.mark.parametrize('r', [79, 80, 399, 400])
def test_small_chunk_edges(k, r):
    """L = 320 000 k + r: the reference's chunk loop drops a last chunk of fewer than 400 samples (r < 400) and cuts its last full chunk
    short when r < 80, so T = 1000 k - 1, 1000 k, 1000 k, 1000 k + 1; k = 4 ends a launch group, k = 30 runs eight groups."""
    m, _ = small_model()
    cfg = hr.small_config()
    sd = {key: v.to(DEV) for key, v in hr.formula_params({key: tuple(v.shape) for key, v in m.state_dict().items()}).items()}
    L = 320_000 * k + r
    T = hubert_frames(L)
    assert T == 1000 * k + (r - 80) // 320
    speech = torch.from_numpy(hr.wave(L))
    got = get_hubert_from_16k_speech(speech, m).double()
    ref = hr.get_hubert(sd, cfg, speech.to(DEV))
    assert got.shape == ref.shape == (T, 128)
    err = float((got - ref).abs().max()) / float(ref.abs().max())
    print(f'small L={L} (T={T}): max|err| / max|ref| = {err:.2e} (bar {hr.E2E_BAR:.0e})')
    assert err <= hr.E2E_BAR


@pytest.fixture(scope='module')
def large():
    m = HubertModel(LARGE)
    sd = hr.formula_params({k: tuple(v.shape) for k, v in m.state_dict().items()})
    m.load_state_dict({k: v.float() for k, v in sd.items()}, strict=True)
    return m.to(DEV), {k: v.to(DEV) for k, v in sd.items()}


@pytest.mark.parametrize('T', [1, 49, 999, 1000, 1031, 2500, 4000, 4001, 9000])
def test_large_against_restatement(large, T):
    """T = 4000 fills one launch group of four segments; 4001 adds a second group of one 1-frame segment; 9000 runs three groups, the last
    with one segment."""
    m, sd = large
    L = 320 * T + 80 + (T % 7) * 37
    assert hubert_frames(L) == T
    speech = torch.from_numpy(hr.wave(L))
    got = get_hubert_from_16k_speech(speech, m).double()
    ref = hr.get_hubert(sd, LARGE, speech.to(DEV))
    err = float((got - ref).abs().max()) / float(ref.abs().max())
    print(f'large T={T}: max|err| / max|ref| = {err:.2e} (bar {hr.E2E_BAR:.0e})')
    assert err <= hr.E2E_BAR


def test_out_padding_determinism_and_graph(large):
    m, _ = large
    T = 1031
    L = 320 * T + 80
    x = torch.from_numpy(hr.wave(L)).to(DEV)
    a = get_hubert_from_16k_speech(x, m)
    b = get_hubert_from_16k_speech(x, m)
    assert torch.equal(a, b)
    Tp = (T + 7) // 8 * 8
    audio = torch.full((2, Tp, 1024), float('nan'), device=DEV)
    r = get_hubert_from_16k_speech(x, m, out=audio[0])
    assert r.data_ptr() == audio[0].data_ptr() and torch.equal(audio[0, :T], a)
    assert bool((audio[0, T:] == 0).all()) and bool(audio[1].isnan().all())
    # CUDA graph at fixed L: replay is bit-identical to eager
    out = torch.empty(T, 1024, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        get_hubert_from_16k_speech(x, m, out=out)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        get_hubert_from_16k_speech(x, m, out=out)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, a)


@torch.no_grad()
def test_multi_group_out_and_graph(large):
    """A clip of three launch groups (T = 9000): out= into a wider row-strided buffer and a CUDA-graph replay, both bit-identical to eager."""
    m, _ = large
    T = 9000
    x = torch.from_numpy(hr.wave(320 * T + 80 + 211)).to(DEV)
    a = get_hubert_from_16k_speech(x, m)
    buf = torch.full((T + 13, 1024 + 64), float('nan'), device=DEV)
    r = get_hubert_from_16k_speech(x, m, out=buf[:, :1024])
    assert r.data_ptr() == buf.data_ptr() and torch.equal(buf[:T, :1024], a)
    assert bool((buf[T:, :1024] == 0).all()) and bool(buf[:, 1024:].isnan().all())
    out = torch.empty(T, 1024, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        get_hubert_from_16k_speech(x, m, out=out)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        get_hubert_from_16k_speech(x, m, out=out)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, a)
