"""HuBERT's front-end and positional-conv entry points on the GPU, each against float64 of the operands it reads, with sentinel guards around
every output: r3dp_hb_stats and r3dp_hb_conv0 (normalisation, k10 s5 conv, LayerNorm, GELU, split rows), r3dp_hb_layernorm in every output
form, r3dp_hb_pos_conv at segment edges; and the chain waveform -> HubertModel (out=batch['audio'][0]) -> PitchContourVAEModel (z= given)
against float64 HuBERT -> the VAE's float64 restatement (tests/audio2motion_reference.py), within the VAE's end-to-end bar E2E_BAR.

The LayerNorm inputs have a small variance (std ~0.05 around an offset), so an eps slip or an unbiased variance moves the output by
1e-3 or more of its scale, far above the bars (3e-5 of |gamma| (|z| + 1) + |beta|, times GELU's slope bound 1.13, plus 2^-21 of the output
for its rounding and the fp32 erf)."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import audio2motion_reference as a2m  # noqa: E402
import hubert_reference as hr  # noqa: E402
from launch_harness import guarded, guards_intact  # noqa: E402
from real3dportrait_b200 import _capi as capi  # noqa: E402
from real3dportrait_b200 import hubert as hb  # noqa: E402
from real3dportrait_b200 import HubertModel, PitchContourVAEModel, get_hubert_from_16k_speech, hubert_frames  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = 'cuda'
LN_REL = 3e-5


def split_value(y, C, lo):
    return y[:, :C].double() + y[:, lo:lo + C].double()


def ln64(x, g=None, b=None, eps=1e-5):
    mu = x.mean(-1, keepdim=True)
    z = (x - mu) / torch.sqrt(((x - mu) ** 2).mean(-1, keepdim=True) + eps)
    return z, (z if g is None else z * g + b)


def ln_bar(z, g, b, u, gelu):
    """Element-wise bar of a LayerNorm output u (before GELU) from its standardised value z."""
    a = z.abs() + 1 if g is None else g.abs() * (z.abs() + 1) + b.abs()
    return LN_REL * a * (1.13 if gelu else 1.0) + 2.0 ** -21 * (hr.gelu(u) if gelu else u).abs()


# ---- stats + conv0 ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('L', [400, 100003, 3000001])
def test_stats(L):
    x = (torch.from_numpy(hr.wave(L)) * 0.8 + 0.05).to(DEV)
    buf, st = guarded(2, torch.float64, fill=float('nan'), device=DEV)
    capi.check(capi.lib().r3dp_hb_stats(capi.ptr(x), L, ctypes.c_void_p(st.data_ptr()), capi.stream()))
    torch.cuda.synchronize()
    assert guards_intact(buf, st.numel(), fill=float('nan'))
    xd = x.double()
    mean, var = xd.mean(), xd.var(unbiased=False)
    assert abs(float(st[0] - mean)) <= 1e-13 * float(xd.abs().max())
    assert abs(float(st[1]) * float(torch.sqrt(var + 1e-7)) - 1.0) <= 1e-12


@pytest.mark.parametrize('C, F', [(512, 1), (512, 3001), (32, 777)])
def test_conv0(C, F):
    g = torch.Generator().manual_seed(C + F)
    L = 5 * (F - 1) + 10 + 3
    x = (torch.from_numpy(hr.wave(L)) * 1.3 - 0.2).to(DEV)
    stats = torch.empty(2, dtype=torch.float64, device=DEV)
    capi.check(capi.lib().r3dp_hb_stats(capi.ptr(x), L, capi.ptr(stats, torch.float64), capi.stream()))
    w = (0.03 * torch.randn(C, 10, generator=g)).to(DEV)
    bias = (0.05 * torch.randn(C, generator=g)).to(DEV)
    gam = (1 + 0.3 * torch.randn(C, generator=g)).to(DEV)
    bet = (0.2 * torch.randn(C, generator=g)).to(DEV)
    lo = C + 64
    buf, y = guarded(F * (2 * C + 128), torch.float16, fill=-7.0, device=DEV)
    capi.check(capi.lib().r3dp_hb_conv0(capi.ptr(x), capi.ptr(stats, torch.float64), F, C, capi.ptr(w), capi.ptr(bias), capi.ptr(gam),
                                        capi.ptr(bet), 1e-5, ctypes.c_void_p(y.data_ptr()), 2 * C + 128, lo, capi.stream()))
    torch.cuda.synchronize()
    assert guards_intact(buf, y.numel(), fill=-7.0)
    y = y.view(F, 2 * C + 128)
    assert bool((y[:, C:lo] == -7.0).all()) and bool((y[:, lo + C:] == -7.0).all())      # the columns between the halves are not written
    xd = x.double()
    xn = (xd - xd.mean()) / torch.sqrt(xd.var(unbiased=False) + 1e-7)
    win = xn[:5 * (F - 1) + 10].unfold(0, 10, 5)                                       # [F, 10]
    pre = win @ w.double().t() + bias.double()
    z, u = ln64(pre, gam.double(), bet.double())
    ref = hr.gelu(u)
    got = split_value(y, C, lo)
    ratio = float(((got - ref).abs() / ln_bar(z, gam.double(), bet.double(), u, True)).max())
    print(f'conv0 C={C} F={F}: worst err/bar {ratio:.3f}')
    assert ratio <= 1.0


# ---- LayerNorm -------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('C, R', [(32, 1), (512, 1000), (1024, 7), (1024, 4001)])
@pytest.mark.parametrize('mode', ['affine_gelu_split', 'affine_f32_strided', 'plain_split', 'affine_gelu_f32_inplace'])
def test_layernorm(mode, C, R):
    g = torch.Generator().manual_seed(C * 7 + R)
    x = (0.5 + 0.05 * torch.randn(R, C, generator=g)).to(DEV)
    affine = mode.startswith('affine')
    gelu = 'gelu' in mode
    gam = (1 + 0.3 * torch.randn(C, generator=g)).to(DEV) if affine else None
    bet = (0.2 * torch.randn(C, generator=g)).to(DEV) if affine else None
    z, u = ln64(x.double(), None if gam is None else gam.double(), None if bet is None else bet.double())
    ref = hr.gelu(u) if gelu else u
    L = capi.lib()
    if mode.endswith('split'):
        ys, lo = 2 * C + 64, C + 32
        buf, y = guarded(R * ys, torch.float16, fill=-7.0, device=DEV)
        capi.check(L.r3dp_hb_layernorm(capi.ptr(x), R, C, capi.ptr(gam), capi.ptr(bet), 1e-5, int(gelu), None, 0, ctypes.c_void_p(y.data_ptr()),
                                       ys, lo, capi.stream()))
        torch.cuda.synchronize()
        assert guards_intact(buf, y.numel(), fill=-7.0)
        y = y.view(R, ys)
        assert bool((y[:, C:lo] == -7.0).all()) and bool((y[:, lo + C:] == -7.0).all())
        got = split_value(y, C, lo)
    elif mode.endswith('strided'):
        ys = C + 40
        buf, y = guarded(R * ys, torch.float32, fill=float('nan'), device=DEV)
        capi.check(L.r3dp_hb_layernorm(capi.ptr(x), R, C, capi.ptr(gam), capi.ptr(bet), 1e-5, int(gelu), ctypes.c_void_p(y.data_ptr()), ys, None,
                                       0, 0, capi.stream()))
        torch.cuda.synchronize()
        assert guards_intact(buf, y.numel(), fill=float('nan'))
        y = y.view(R, ys)
        assert bool(y[:, C:].isnan().all())
        got = y[:, :C].double()
    else:                                                                              # in place, as the feature projection's input runs
        buf, y = guarded(R * C, torch.float32, fill=float('nan'), device=DEV)
        y.copy_(x.view(-1))
        capi.check(L.r3dp_hb_layernorm(ctypes.c_void_p(y.data_ptr()), R, C, capi.ptr(gam), capi.ptr(bet), 1e-5, int(gelu),
                                       ctypes.c_void_p(y.data_ptr()), C, None, 0, 0, capi.stream()))
        torch.cuda.synchronize()
        assert guards_intact(buf, y.numel(), fill=float('nan'))
        got = y.view(R, C).double()
    bar = ln_bar(z, None if gam is None else gam.double(), None if bet is None else bet.double(), u, gelu)
    ratio = float(((got - ref).abs() / bar).max())
    print(f'layernorm {mode} C={C} R={R}: worst err/bar {ratio:.3f}')
    assert ratio <= 1.0


# ---- positional conv -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('H, nseg, Lseg, M', [(1024, 1, 1, 1), (1024, 3, 1000, 2500), (128, 2, 130, 200), (1024, 4, 129, 4 * 129),
                                              (128, 1, 64, 63)])
def test_pos_conv(H, nseg, Lseg, M):
    g = torch.Generator().manual_seed(H + nseg + Lseg + M)
    G = H // 64
    xv = torch.randn(M, H, generator=g).to(DEV) * 1.5
    xs = torch.zeros(nseg * Lseg, 2 * H, device=DEV, dtype=torch.float16)
    capi.check(capi.lib().r3dp_a2m_split(capi.ptr(xv), M, H, capi.ptr(xs, torch.float16), None, capi.stream()))
    X = xs[:M, :H].double() + xs[:M, H:].double()
    w = torch.randn(H, 64, 128, generator=g, dtype=torch.float64) / np.sqrt(64 * 128)
    wp = hb.pack_split(hb.pos_gemm_weight(w)).to(DEV)
    W = (wp[:, :8192].double() + wp[:, 8192:].double()) / 1024.0                      # [H, 128 * 64], K = tap-major
    W3 = W.view(H, 128, 64).permute(0, 2, 1).contiguous()                              # back to [H, 64, 128]
    bias = (0.1 * torch.randn(H, generator=g)).to(DEV)
    buf, y = guarded(M * H + 3 * H, torch.float32, fill=0.0, device=DEV)
    init = torch.randn(M, H, generator=g).to(DEV)
    y[:M * H].copy_(init.view(-1))
    y[M * H:].fill_(-3.0)                                                              # rows past M: not written
    capi.check(capi.lib().r3dp_hb_pos_conv(capi.ptr(xs, torch.float16), nseg, Lseg, M, H, capi.ptr(wp, torch.float16), capi.ptr(bias),
                                           ctypes.c_void_p(y.data_ptr()), capi.stream()))
    torch.cuda.synchronize()
    assert guards_intact(buf, y.numel(), fill=0.0) and bool((y[M * H:] == -3.0).all())
    pre, mag = [], []
    for s in range(nseg):
        seg = X[s * Lseg:min((s + 1) * Lseg, M)]
        if seg.shape[0] == 0:
            continue
        pre.append(Fn.conv1d(seg.t()[None], W3, None, padding=64, groups=G)[0, :, :-1].t())
        mag.append(Fn.conv1d(seg.abs().t()[None], W3.abs(), None, padding=64, groups=G)[0, :, :-1].t())
    pre, mag = torch.cat(pre) + bias.double(), torch.cat(mag)
    ref = init.double() + hr.gelu(pre)
    got = y[:M * H].view(M, H).double()
    bar = 1.13 * (2.0 ** -17 * mag + 2.0 ** -22 * bias.double().abs()) + 2.0 ** -21 * hr.gelu(pre).abs() + 2.0 ** -22 * ref.abs()
    ratio = float(((got - ref).abs() / bar).max())
    print(f'pos_conv H={H} segs={nseg}x{Lseg} M={M}: worst err/bar {ratio:.3f}')
    assert ratio <= 1.0


# ---- waveform -> HuBERT -> VAE ---------------------------------------------------------------------------------------------------------
@torch.no_grad()
def test_hubert_into_vae():
    large = dict(conv_dim=(512,) * 7, hidden_size=1024, num_attention_heads=16, intermediate_size=4096, num_hidden_layers=24,
                 num_conv_pos_embeddings=128, num_conv_pos_embedding_groups=16, feat_extract_norm='layer', do_stable_layer_norm=True,
                 conv_bias=True)
    m = HubertModel(large)
    sd = hr.formula_params({k: tuple(v.shape) for k, v in m.state_dict().items()})
    m.load_state_dict({k: v.float() for k, v in sd.items()}, strict=True)
    m = m.to(DEV)
    vae = PitchContourVAEModel(a2m.HP_PITCH, audio_in_dim=1024)
    vsd = a2m.make_params({k: v.shape for k, v in vae.state_dict().items()}, 11)
    vae.load_state_dict(vsd, strict=True)
    vae = vae.to(DEV).eval()

    L = 320 * 1203 + 80 + 150                                                          # two segments, T = 1203 -> T_x = 1208
    T = hubert_frames(L)
    Tx = (T + 7) // 8 * 8
    speech = torch.from_numpy(hr.wave(L))
    batch = a2m.make_batch(1, Tx, 1024, seed=4, pitch=True, mouth_amp=0.45)
    v = a2m.f0_mel_scaled64(batch['f0']).clamp(1, 255) + 0.5                         # f0 clear of pitch-bin rounding edges
    fr = v - v.floor()
    batch['f0'][(fr < 1e-3) | (fr > 1 - 1e-3)] = 0.0
    z = torch.randn(1, 16, Tx // 8, generator=torch.Generator().manual_seed(2))

    audio = torch.full((1, Tx, 1024), float('nan'), device=DEV)
    get_hubert_from_16k_speech(speech, m, out=audio[0])
    lib_batch = {k: val.to(DEV) for k, val in batch.items()}
    lib_batch['audio'] = audio
    got = vae(lib_batch, {}, temperature=0.2, z=z.to(DEV))

    feats = torch.zeros(1, Tx, 1024, dtype=torch.float64, device=DEV)
    feats[0, :T] = hr.get_hubert({k: val.to(DEV) for k, val in sd.items()}, large, speech.to(DEV))
    ref_batch = {k: val.to(DEV) for k, val in batch.items()}
    ref_batch['audio'] = feats
    want = a2m.forward({k: val.to(DEV) for k, val in vsd.items()}, ref_batch, z.to(DEV), 0.2, pitch=True)
    err = float((got.double() - want).abs().max()) / float(want.abs().max())
    print(f'waveform -> HuBERT -> VAE: max|err| / max|ref| = {err:.2e} (bar {a2m.E2E_BAR:.0e})')
    assert err <= a2m.E2E_BAR
