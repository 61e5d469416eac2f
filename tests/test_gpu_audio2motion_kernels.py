"""r3dp_a2m_wn_layer against float64 at both WaveNet shapes of the audio2secc forward (hidden 64 / k 3 at T/4: the prior flow; hidden 256 /
k 5 at T: the decoder), at T = 1, around the 64-frame tile, and up to T = 7500 / 15000 (ten minutes of audio), B = 1 and 3, first / middle /
last layer; every output between sentinel guards.  The pitch bins of r3dp_a2m_input against float64 outside a margin around each bin edge.

Bar (per output element), from the split-fp16 operands: each operand is hi + lo to ~2^-22 relative, products accumulate in fp32 over
K = hidden * k terms, so a pre-activation a carries e_a = 2^-18 sum |w| |x| (+ 2^-23 |a|); the gate passes e_a + e_b / 4 (tanh' <= 1,
sigmoid' <= 1/4) plus 2^-22 |g| of its own split; res_skip adds sum |w_rs| e_g + 2^-18 sum |w_rs| |g|; the outputs are rounded once more."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import audio2motion_reference as ref
from launch_harness import guarded, guards_intact
from real3dportrait_b200 import _capi as capi
from real3dportrait_b200.audio2motion import F0_MEL_MAX, F0_MEL_MIN, gate_order, pack_wn_layer

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
SENT = -12345.0


def _layer64(H, k, NO, B, T, seed, first, last):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, H, generator=g, dtype=torch.float64)
    w_in = torch.randn(2 * H, H, k, generator=g, dtype=torch.float64) * (0.6 / (H * k) ** 0.5)
    w_rs = torch.randn(NO, H, generator=g, dtype=torch.float64) * (0.6 / H ** 0.5)
    b_rs = 0.05 * torch.randn(NO, generator=g, dtype=torch.float64)
    cond = torch.randn(B, T, 2 * H, generator=g, dtype=torch.float64) * 0.5         # paired rows, in_layer bias included
    skip = None if first else torch.randn(B, T, H, generator=g, dtype=torch.float64)
    return x, w_in, w_rs, b_rs, cond, skip


def _reference(x, w_in, w_rs, b_rs, cond, skip, H):
    """float64 outputs and bars: (x_out, skip_out) per the kernel's contract."""
    k = w_in.shape[2]
    wi = w_in[gate_order(H)]
    a = F.conv1d(x.transpose(1, 2), wi, padding=k // 2).transpose(1, 2) + cond
    mag = F.conv1d(x.abs().transpose(1, 2), wi.abs(), padding=k // 2).transpose(1, 2)
    e = 2.0 ** -18 * mag + 2.0 ** -23 * a.abs()
    gated = torch.tanh(a[..., 0::2]) * torch.sigmoid(a[..., 1::2])
    eg = e[..., 0::2] + 0.25 * e[..., 1::2] + 2.0 ** -22 * gated.abs()
    rs = gated @ w_rs.t() + b_rs
    ers = eg @ w_rs.abs().t() + 2.0 ** -18 * (gated.abs() @ w_rs.abs().t()) + 2.0 ** -22 * rs.abs()
    return rs, ers


CASES = [(64, 3, T, B) for T in (1, 63, 64, 65, 129, 7500) for B in (1, 3)] + [(256, 5, T, B) for T in (1, 63, 64, 65, 129, 15000) for B in (1, 3)]


@pytest.mark.parametrize('H,k,T,B', CASES)
@pytest.mark.parametrize('pos', ['first', 'middle', 'last'])
@torch.no_grad()
def test_wn_layer_matches_float64(H, k, T, B, pos):
    if T >= 7500 and B == 3 and pos == 'middle':
        pytest.skip('the long sequences run at B = 3 as first / last layers only')
    first, last = pos == 'first', pos == 'last'
    NO = H if last else 2 * H
    x, w_in, w_rs, b_rs, cond, skip = (None if t is None else t.to(DEV) for t in _layer64(H, k, NO, B, T, seed=H + 7 * T + B, first=first, last=last))
    rs, ers = _reference(x, w_in, w_rs, b_rs, cond, skip, H)
    n = B * T * H
    xb, xd = guarded(n, torch.float32, fill=SENT, device=DEV)
    xd.copy_(x.flatten().float())
    ob, od = guarded(n, torch.float32, fill=SENT, device=DEV)
    sb, sd = guarded(n, torch.float32, fill=SENT, device=DEV)
    if skip is not None:
        sd.copy_(skip.flatten().float())
    hb, hd = guarded(2 * n, torch.float16, fill=-3.0, device=DEV)
    cond_buf = torch.full((B * T, 2 * H + 6), SENT, device=DEV)                   # a row stride beyond the slice
    cond_buf[:, :2 * H] = cond.reshape(B * T, 2 * H).float()
    w = pack_wn_layer(w_in, w_rs)
    bias = b_rs.float()
    L = capi.lib()
    capi.check(L.r3dp_a2m_wn_layer(capi.ptr(xd), None if last else capi.ptr(od), capi.ptr(cond_buf), 2 * H + 6, capi.ptr(w, torch.float16),
                                   capi.ptr(bias), capi.ptr(sd), ctypes.c_void_p(hd.data_ptr()) if last else None, B, T, H, k,
                                   int(first), int(last), capi.stream()))
    torch.cuda.synchronize()
    assert guards_intact(xb, n, fill=SENT) and torch.equal(xd, x.flatten().float())          # the input is never written
    if last:
        want = skip + rs
        bar = ers + 2.0 ** -22 * want.abs()
        h = hd.view(B, T, 2 * H).double()
        got = h[..., :H] + h[..., H:]
        assert guards_intact(hb, 2 * n, fill=-3.0) and guards_intact(ob, n, fill=SENT) and bool((od == SENT).all())
    else:
        got_x = od.view(B, T, H).double()
        err_x = (got_x - (x + rs[..., :H])).abs()
        bar_x = ers[..., :H] + 2.0 ** -23 * (x + rs[..., :H]).abs()
        assert guards_intact(ob, n, fill=SENT)
        assert bool((err_x <= bar_x).all()), float((err_x / bar_x).max())
        want = rs[..., H:] if first else skip + rs[..., H:]
        bar = ers[..., H:] + 2.0 ** -23 * want.abs()
        got = sd.view(B, T, H).double()
        assert bool((hd == -3.0).all())
    assert guards_intact(sb, n, fill=SENT)
    err = (got - want).abs()
    # the ends of each sequence and the tile boundaries are where the halo and the zero padding act: report them on their own
    for t in sorted({0, T - 1} | {t for t in (63, 64, 127, 128) if t < T}):
        assert bool((err[:, t] <= bar[:, t]).all()), (t, float((err[:, t] / bar[:, t]).max()))
    assert bool((err <= bar).all()), float((err / bar).max())


@torch.no_grad()
def test_input_pitch_bins_match_float64():
    """Row i of a probe table holds i, so the pitch block of the packed rows reads back the bin.  Frames whose float64 value lies within
    1e-4 of a rounding edge are ambiguous (the fp32 log may fall either side); every other frame must match, and fewer than 1 % may be
    ambiguous."""
    g = torch.Generator().manual_seed(3)
    B, Tx = 2, 20000
    f0 = torch.cat([torch.linspace(-699.0, 1500.0, Tx // 2), 1200.0 * torch.rand(Tx // 2, generator=g)]).repeat(B, 1)
    f0[:, ::7] = 0.0
    audio = torch.randn(B, Tx, 13, generator=g)
    table = torch.arange(300, dtype=torch.float32)[:, None].repeat(1, 128).contiguous()
    T = Tx // 2
    C = 32 + 128
    y = torch.empty(B * T, 2 * C, device=DEV, dtype=torch.float16)
    yb = torch.empty(B * T, 64, device=DEV, dtype=torch.float16)
    audio_d, f0_d, table_d = audio.to(DEV), f0.to(DEV), table.to(DEV)                # alive until the kernel has run
    capi.check(capi.lib().r3dp_a2m_input(capi.ptr(audio_d), B, Tx, 13, 32, 0, capi.ptr(f0_d), None, None, None,
                                         capi.ptr(table_d), float(F0_MEL_MIN), float(F0_MEL_MAX - F0_MEL_MIN), capi.ptr(y, torch.float16),
                                         2 * C, C, capi.ptr(yb, torch.float16), 64, 32, capi.stream()))
    torch.cuda.synchronize()
    got = (y[:, 32:160].float() + y[:, C + 32:C + 160].float()).cpu()
    assert bool((got == got[:, :1]).all())
    got = got[:, 0].round().long().view(B, T)
    fd = f0[:, ::2]
    want = ref.f0_to_coarse_ref(fd.clone())
    v = ref.f0_mel_scaled64(fd).clamp(1, 255) + 0.5
    ambiguous = ((v - v.floor()) < 1e-4) | ((v - v.floor()) > 1 - 1e-4)
    assert bool((got == want)[~ambiguous].all())
    assert int(ambiguous.sum()) < 0.01 * B * T
    # the audio columns: frame 2i (nearest), zero padding to 32 channels; hi + lo holds a value to 2^-21 relative, or to the fp16
    # subnormal step 2^-24 where the remainder is that small
    a = (y[:, :32].double() + y[:, C:C + 32].double()).cpu().view(B, T, 32)
    assert torch.allclose(a[..., :13], audio[:, ::2].double(), rtol=2 ** -21, atol=2 ** -24) and bool((a[..., 13:] == 0).all())
    # the blink / amplitude block without blink or amplitudes: blink == 0 everywhere, zeros elsewhere
    assert bool((yb[:, 0] == 1).all()) and bool((yb[:, 1:] == 0).all())
