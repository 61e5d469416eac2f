"""Every launch of HuBERT (get_hubert_from_16k_speech, HubertModel.forward) at its exact arguments against float64, and a recorded-launch
check that keeps these tables equal to what the module launches.

* The tables hold one row per distinct launch of hubert_reference.launch_plan over hubert-large and the small fixture config at
  T = 1, 49, 1031, 4000 and 4001 (large) and T = 1, 49, 1031, 4001 (small).  The conv stack runs one launch group at a time, so T = 4000
  already has the largest M (256 015 conv0 rows); longer clips add groups, not launch shapes.
* r3dp_hb_gemm rows use the module's own _prepared() packing (the folded LayerNorms, the 1/8 in q, the Cp-padded conv K) against float64
  built from fold_weights, not from the packed halves, under tests/test_gpu_hubert.py's element-wise bar 2^-17 sum|w||x| (GELU: x 1.8)
  + 2^-20 |y|.  Inputs are random fp32 split by the test; the Cp pad channels are zero (the module zero-fills them) and the rows past the
  last one the launch reads are NaN.  Sentinels surround every output and fill the columns outside its halves; the residual epilogue leaves
  the rows past M untouched.  Each row asserts that the float64 result of hi-only activations, and of hi-only weights, breaks its bar.
  A one-row launch runs on ONE_ROW_DRAWS inputs: on one row of K = 4096 products a lost lo half moves the outputs by about the bar itself.
* r3dp_hb_attention rows at the module's H, heads and segment lengths (a one-frame segment's bar has no score term: its output is v): the
  first and last frame of each segment and the 64-row tile edges are checked on their own, hi-only q / k / v break the bar, and the last
  segment equals a launch on it alone bit for bit.
* r3dp_hb_layernorm (the module's gamma / beta or none, every output form including conv6's in place), r3dp_hb_conv0, r3dp_hb_pos_conv
  (the module's weight-normed weights against fold_weights') and r3dp_a2m_split at their real arguments.
* test_launches_have_rows records get_hubert_from_16k_speech at every plan's clip and HubertModel.forward on two items: the calls equal
  launch_plan (186 per group for hubert-large), every launch has a row and every row is still launched, and every split operand a GEMM,
  attention or positional-conv launch reads carries its lo halves (a module that wrote one of them hi-only would pass every row)."""
import ctypes

import pytest
import torch
import torch.nn.functional as Fn

import hubert_reference as hr
import test_gpu_hubert as tgh
import test_gpu_hubert_kernels as kern
from launch_harness import (Recorder, assert_plan, assert_rows, assert_written, at, call_signature, guarded, guards_intact, hi_w, inside, split,
                            untouched)
from real3dportrait_b200 import _capi as capi
from real3dportrait_b200 import hubert as hb
from real3dportrait_b200 import get_hubert_from_16k_speech

pytestmark = pytest.mark.gpu
DEV = 'cuda'
F16, F32, F64 = torch.float16, torch.float32, torch.float64
CFG = {'large': hr.LARGE, 'small': hr.small_config()}
PLANS = [('large', T) for T in (1, 49, 1031, 4000, 4001)] + [('small', T) for T in (1, 49, 1031, 4001)]
FORWARD_LX = 320 * 48 + 400 + 11                        # HubertModel.forward input length: T = 49, the rows of the T = 49 plans
GELU_LIP = 1.13
ONE_ROW_DRAWS = 32


def clip(T):
    return 320 * T + 80 + (T % 7) * 37


def _rows(fn):
    """{signature: (config, tag, plan label)} of one entry point over PLANS, the first of each distinct launch."""
    out = {}
    for name, T in PLANS:
        for tag, f, a in hr.launch_plan(CFG[name], clip(T)):
            if f == fn:
                out.setdefault(hr.launch_signature(f, a), (name, tag, f'{name}-T{T}'))
    return out


GEMM, ATTN, LNORM = _rows('r3dp_hb_gemm'), _rows('r3dp_hb_attention'), _rows('r3dp_hb_layernorm')
CONV0, POS, SPLIT = _rows('r3dp_hb_conv0'), _rows('r3dp_hb_pos_conv'), _rows('r3dp_a2m_split')
TABLES = {'r3dp_hb_gemm': GEMM, 'r3dp_hb_attention': ATTN, 'r3dp_hb_layernorm': LNORM, 'r3dp_hb_conv0': CONV0, 'r3dp_hb_pos_conv': POS,
          'r3dp_a2m_split': SPLIT}


def _ids(table):
    return [f'{v[2]}-{v[1].split(".", 1)[1]}-' + 'x'.join(str(a) for a in k[1] if not isinstance(a, (tuple, float))) for k, v in table.items()]


def randn(shape, seed, scale=1.0):
    return (torch.randn(shape, generator=torch.Generator().manual_seed(seed)) * scale).to(DEV)


# ---- the models: module packing and float64 folds ------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def models():
    out = {}
    for name, cfg in CFG.items():
        m, _ = hr.formula_model(cfg)
        m = m.to(DEV)
        with torch.no_grad():
            out[name] = (m, m._prepared(), hb.fold_weights(m))
    return out


def gemm_weights(Q, P, site, Cp):
    """(packed fp16 [N, 2 Kp], fp32 bias) of the module and (W [N, Kp], b) float64 of fold_weights (K zero-padded to Kp) for one GEMM."""
    if site.startswith('conv'):
        i = int(site[4])
        w, b, _ = P['conv'][i]
        return Q['conv'][i][0], Q['conv'][i][1], hb.conv_gemm_weight(w, Cp), b
    if site == 'proj':
        w, b = P['proj']
        wz = torch.zeros(w.shape[0], Cp, dtype=F64, device=DEV)
        wz[:, :w.shape[1]] = w
        return Q['proj'][0], Q['proj'][1], wz, b
    j, part = site[1:].split('.')
    n = ('qkv', 'out', 'ffn1', 'ffn2').index(part)
    q, p = Q['layers'][int(j)], P['layers'][int(j)]
    return q[2 * n], q[2 * n + 1], p[2 * n], p[2 * n + 1]


@torch.no_grad()
@pytest.mark.parametrize('key', list(GEMM), ids=_ids(GEMM))
def test_gemm_launch(models, key):
    """An encoder layer's row runs with every layer's weights.  A one-row launch (T = 1) runs on ONE_ROW_DRAWS independent inputs, so its
    hi-only check sees about as many outputs as a 49-row one: on a single row of K = 4096 products a lost lo half moves the outputs by
    about the bar itself."""
    name, tag, label = GEMM[key]
    M, N, Kp = key[1][0], key[1][4], key[1][5]
    seed = 1000 * list(GEMM).index(key)
    site = tag.split('.', 1)[1]
    layers = [f'l{j}.{site.split(".")[1]}' for j in range(CFG[name]['num_hidden_layers'])] if site.startswith('l') else [site]
    draws = ONE_ROW_DRAWS if M == 1 else 1
    res = [[_gemm_draw(models, key, ly, seed + 100 * j + d) for d in range(draws)] for j, ly in enumerate(layers)]
    ratio = max(r[0] for per in res for r in per)
    mx, mw = (min(max(r[i] for r in per) for per in res) for i in (1, 2))   # the weakest layer's hi-only margins
    what = f'{label} {tag.split(".", 1)[1]}'
    print(f'gemm {what} M={M} N={N} K={Kp} ({len(layers)} layers x {draws} draws): worst err/bar {ratio:.3f}; hi-only activations '
          f'x{mx:.2f}, hi-only weights x{mw:.2f}')
    assert ratio <= 1.0, f'{what}: err/bar {ratio:.3f}'
    assert mx > 1.0 and mw > 1.0, f'{what}: the bar does not see hi-only operands ({mx:.2f}, {mw:.2f})'


def _gemm_draw(models, key, site, seed):
    """One launch of a GEMM row with the weights of `site` on random inputs -> (worst err/bar, worst hi-only activations / bar, worst
    hi-only weights / bar)."""
    name, tag, label = GEMM[key]
    M, width, stride, seg, N, Kp, epi, ldy, ylo = key[1]
    what = f'{label} {site}'
    cfg = CFG[name]
    _, Q, P = models[name]
    C = cfg['conv_dim'][0]
    conv = site.startswith('conv')
    wp, bias, W64, b64 = gemm_weights(Q, P, site, seg)
    assert wp.shape == (N, 2 * Kp) and W64.shape == (N, Kp), what           # the module packs the launch's K and N
    k, s = (hr.KERNELS[int(site[4])], hr.STRIDES[int(site[4])]) if conv else (1, 1)
    K = C if conv or site == 'proj' else seg                                 # the real channels of an input row; [K, seg) is zero padding
    F = (M - 1) * s + k                                                      # the input rows the launch reads
    xv = randn((F, K), seed, 2.0)
    A = torch.full((F + 64, 2 * seg), float('nan'), device=DEV, dtype=F16)  # NaN rows past the last one read
    A[:F] = 0.0
    A[:F, :K], A[:F, seg:seg + K] = split(xv)
    X = torch.zeros(F, seg, dtype=F64, device=DEV)
    X[:, :K] = A[:F, :K].double() + A[:F, seg:seg + K].double()
    X = X.unfold(0, k, s).permute(0, 2, 1).reshape(M, k * seg)             # window rows, K channel j seg + i
    Xh = torch.zeros(F, seg, dtype=F64, device=DEV)
    Xh[:, :K] = A[:F, :K].double()
    Xh = Xh.unfold(0, k, s).permute(0, 2, 1).reshape(M, k * seg)
    pre = X @ W64.t() + b64
    mag = X.abs() @ W64.abs().t()
    pre_hx, pre_hw = Xh @ W64.t() + b64, X @ hi_w(W64).t() + b64
    if epi in (0, 1):
        buf, y = guarded(M * ldy, F16, device=DEV)
    else:
        buf, y = guarded(M * ldy + 64 * ldy, F32, device=DEV)                 # + 64 rows past M
    yv = y[:M * ldy].view(M, ldy)
    init = None
    if epi == 2:
        init = randn((M, ldy), seed + 1)
        yv.copy_(init)
    capi.check(capi.lib().r3dp_hb_gemm(at(A), M, width, stride, seg, capi.ptr(wp, F16), N, Kp, capi.ptr(bias), epi, at(y), ldy, ylo,
                                       capi.stream()))
    torch.cuda.synchronize()
    assert guards_intact(buf, y.numel()), f'{what}: written outside the output'
    mask = inside(ldy, 0, N, ylo, epi in (0, 1), device=DEV)
    if epi in (0, 1):
        got = yv[:, :N].double() + yv[:, ylo:ylo + N].double()
    else:
        got = yv[:, :N].double()
        assert bool(untouched(y[M * ldy:]).all()), f'{what}: rows past M written'
    if epi != 2:
        assert not bool(untouched(yv[:, mask]).any()), f'{what}: an output element was not written'
        assert bool(untouched(yv[:, ~mask]).all()), f'{what}: written outside the output halves'
    else:
        assert torch.equal(yv[:, N:], init[:, N:]), f'{what}: residual columns past N changed'
    if epi == 1:
        want, want_hx, want_hw = hr.gelu(pre), hr.gelu(pre_hx), hr.gelu(pre_hw)
    elif epi == 2:
        r = init[:, :N].double()
        want, want_hx, want_hw = pre + r, pre_hx + r, pre_hw + r
    else:
        want, want_hx, want_hw = pre, pre_hx, pre_hw
    bar = 2.0 ** -17 * mag * (1.8 if epi == 1 else 1.0) + 2.0 ** -20 * want.abs() + 1e-30
    return tuple(float(((w - want).abs() / bar).max()) for w in (got, want_hx, want_hw))


# ---- attention -----------------------------------------------------------------------------------------------------------------------------
def attention64(qkv, lens, H):
    """test_gpu_hubert.attention_ref's float64 output and magnitude, except that a segment of one frame has no score term: its softmax is
    1 whatever the score, so its output is v and the magnitude |v|."""
    want, mag = tgh.attention_ref(qkv, list(lens), H)
    r0 = 0
    for n in lens:
        if n == 1:
            mag[r0] = (qkv[r0, 2 * H:3 * H].double() + qkv[r0, 5 * H:].double()).abs()
        r0 += n
    return want, mag


def attention(qkv, rows, H, heads, lens, o, os_, olo):
    arr = (ctypes.c_int * len(lens))(*lens)
    capi.check(capi.lib().r3dp_hb_attention(qkv, rows, 6 * H, 3 * H, heads, arr, len(lens), o, os_, olo, capi.stream()))


@torch.no_grad()
@pytest.mark.parametrize('key', list(ATTN), ids=_ids(ATTN))
def test_attention_launch(key):
    name, tag, label = ATTN[key]
    rows, ld, lo, heads, lens, nseg, os_, olo = key[1]
    H = 64 * heads
    what = f'{label} {tag} lens {lens[:4]}'
    x = randn((rows, 3 * H), list(ATTN).index(key) + 50, 2.0)
    qkv = torch.cat(split(x), 1).contiguous()
    buf, o = guarded(rows * os_, F16, device=DEV)
    attention(at(qkv), rows, H, heads, lens, at(o), os_, olo)
    assert_written(buf, o, os_, inside(os_, 0, H, olo, True, device=DEV), what)
    ov = o.view(rows, os_)
    got = ov[:, :H].double() + ov[:, olo:olo + H].double()
    want, mag = attention64(qkv, lens, H)
    bar = 2.0 ** -17 * mag + 2.0 ** -20 * want.abs()
    bad = ~((got - want).abs() <= bar)
    r0 = 0
    for n in lens:                                              # each segment's ends and its 64-row tile edges, so a leak is named
        assert not bool(bad[r0].any()) and not bool(bad[r0 + n - 1].any()), f'{what}: segment at row {r0} (length {n}): an end frame'
        t = torch.arange(n, device=DEV)
        assert not bool(bad[r0:r0 + n][(t % 64 == 0) | (t % 64 == 63)].any()), f'{what}: segment at row {r0}: a 64-row tile edge'
        r0 += n
    ratio = float(((got - want).abs() / bar).max())
    hi_qkv = torch.cat([qkv[:, :3 * H], torch.zeros_like(qkv[:, 3 * H:])], 1)
    want_h, _ = attention64(hi_qkv, lens, H)
    mh = float(((want_h - want).abs() / bar).max())
    print(f'attention {what}: worst err/bar {ratio:.3f}; hi-only q, k, v x{mh:.1f}')
    assert ratio <= 1.0, f'{what}: err/bar {ratio:.3f}'
    assert mh > 1.0, f'{what}: the bar does not see hi-only q, k, v'
    last = lens[-1]
    obuf, one = guarded(last * os_, F16, device=DEV)
    attention(at(qkv, (rows - last) * 6 * H), last, H, heads, (last,), at(one), os_, olo)
    torch.cuda.synchronize()
    assert guards_intact(obuf, one.numel())
    assert torch.equal(one.view(torch.int16), o[(rows - last) * os_:].view(torch.int16)), f'{what}: the last segment vs a launch on it alone'


# ---- LayerNorm, conv0, positional conv, split -------------------------------------------------------------------------------------------
def ln_params(Q, site):
    if site.startswith('conv'):
        return Q['conv'][int(site[4])][2:4]
    return Q['ln_f'][:2] if site == 'ln_f' else (None, None)


@torch.no_grad()
@pytest.mark.parametrize('key', list(LNORM), ids=_ids(LNORM))
def test_layernorm_launch(models, key):
    name, tag, label = LNORM[key]
    site = tag.split('.', 1)[1]
    R, C, eps, gelu, yfs, yhs, yhlo = key[1]
    what = f'{label} {site}'
    _, Q, _ = models[name]
    g, b = ln_params(Q, site)
    x = 0.5 + randn((R, C), list(LNORM).index(key) + 300, 0.05)
    z, u = kern.ln64(x.double(), None if g is None else g.double(), None if b is None else b.double(), eps)
    want = hr.gelu(u) if gelu else u
    inplace = yfs and site.startswith('conv')
    if yhs:
        buf, y = guarded(R * yhs, F16, device=DEV)
        capi.check(capi.lib().r3dp_hb_layernorm(capi.ptr(x), R, C, capi.ptr(g), capi.ptr(b), eps, gelu, None, 0, at(y), yhs, yhlo,
                                                capi.stream()))
        mask = inside(yhs, 0, C, yhlo, True, device=DEV)
    else:
        buf, y = guarded(R * yfs, F32, device=DEV)
        if inplace:
            y.view(R, yfs)[:, :C].copy_(x)
        src = at(y) if inplace else capi.ptr(x)
        capi.check(capi.lib().r3dp_hb_layernorm(src, R, C, capi.ptr(g), capi.ptr(b), eps, gelu, at(y), yfs, None, 0, 0, capi.stream()))
        mask = inside(yfs, 0, C, device=DEV)
    torch.cuda.synchronize()
    assert guards_intact(buf, y.numel()), f'{what}: written outside the output'
    yv = y.view(R, -1)
    assert bool(untouched(yv[:, ~mask]).all()), f'{what}: written between or past the output halves'
    got = yv[:, :C].double() + (yv[:, yhlo:yhlo + C].double() if yhs else 0.0)
    ratio = float(((got - want).abs() / kern.ln_bar(z, None if g is None else g.double(), None if b is None else b.double(), u, gelu)).max())
    print(f'layernorm {what} R={R} C={C}: worst err/bar {ratio:.3f}')
    assert ratio <= 1.0, f'{what}: err/bar {ratio:.3f}'


@torch.no_grad()
@pytest.mark.parametrize('key', list(CONV0), ids=_ids(CONV0))
def test_conv0_launch(models, key):
    name, tag, label = CONV0[key]
    F, C, eps, ys, ylo = key[1]
    _, Q, _ = models[name]
    w0, b0, g0, be0, e0 = Q['conv'][0]
    assert ctypes.c_float(e0).value == eps
    n = 5 * (F - 1) + 10
    x = (torch.from_numpy(hr.wave(n + 7)) * 1.3 - 0.2).to(DEV)[:n]
    xd = x.double()
    stats = torch.stack([xd.mean(), 1.0 / torch.sqrt(xd.var(unbiased=False) + 1e-7)])
    buf, y = guarded(F * ys, F16, device=DEV)
    capi.check(capi.lib().r3dp_hb_conv0(capi.ptr(x), capi.ptr(stats, F64), F, C, capi.ptr(w0), capi.ptr(b0), capi.ptr(g0), capi.ptr(be0), eps,
                                        at(y), ys, ylo, capi.stream()))
    torch.cuda.synchronize()
    assert guards_intact(buf, y.numel())
    yv = y.view(F, ys)
    assert bool(untouched(yv[:, ~inside(ys, 0, C, ylo, True, device=DEV)]).all()), f'{label}: written between or past the halves'
    win = ((xd - stats[0]) * stats[1]).unfold(0, 10, 5)
    pre = win @ w0.double().t() + b0.double()
    z, u = kern.ln64(pre, g0.double(), be0.double(), eps)
    got = yv[:, :C].double() + yv[:, ylo:ylo + C].double()
    ratio = float(((got - hr.gelu(u)).abs() / kern.ln_bar(z, g0.double(), be0.double(), u, True)).max())
    print(f'conv0 {label} F={F} C={C}: worst err/bar {ratio:.3f}')
    assert ratio <= 1.0


def _pos64(X, W3, H, nseg, Ls, M):
    out = []
    for s in range(nseg):
        seg = X[s * Ls:min((s + 1) * Ls, M)]
        out.append(Fn.conv1d(seg.t()[None], W3, None, padding=64, groups=H // 64)[0, :, :-1].t())
    return torch.cat(out)


@torch.no_grad()
@pytest.mark.parametrize('key', list(POS), ids=_ids(POS))
def test_pos_conv_launch(models, key):
    name, tag, label = POS[key]
    nseg, Ls, M, H = key[1]
    _, Q, P = models[name]
    wp, bias = Q['pos']
    W3, b64 = P['pos']
    seed = list(POS).index(key) + 700
    xv = randn((M, H), seed, 1.5)
    xs = torch.zeros(nseg * Ls, 2 * H, device=DEV, dtype=F16)              # rows past M: zero, as the module allocates them
    xs[:M, :H], xs[:M, H:] = split(xv)
    X = xs[:M, :H].double() + xs[:M, H:].double()
    buf, y = guarded(M * H + 64 * H, F32, device=DEV)
    init = randn((M, H), seed + 1)
    y[:M * H].copy_(init.view(-1))
    capi.check(capi.lib().r3dp_hb_pos_conv(capi.ptr(xs, F16), nseg, Ls, M, H, capi.ptr(wp, F16), capi.ptr(bias), at(y), capi.stream()))
    torch.cuda.synchronize()
    assert guards_intact(buf, y.numel()) and bool(untouched(y[M * H:]).all()), f'{label}: written past row M'
    pre = _pos64(X, W3, H, nseg, Ls, M) + b64
    mag = _pos64(X.abs(), W3.abs(), H, nseg, Ls, M)
    want = init.double() + hr.gelu(pre)
    got = y[:M * H].view(M, H).double()
    bar = GELU_LIP * (2.0 ** -17 * mag + 2.0 ** -22 * b64.abs()) + 2.0 ** -21 * hr.gelu(pre).abs() + 2.0 ** -22 * want.abs()
    ratio = float(((got - want).abs() / bar).max())
    hx = init.double() + hr.gelu(_pos64(xs[:M, :H].double(), W3, H, nseg, Ls, M) + b64)
    hw = init.double() + hr.gelu(_pos64(X, hi_w(W3), H, nseg, Ls, M) + b64)
    mx, mw = (float(((h - want).abs() / bar).max()) for h in (hx, hw))
    print(f'pos_conv {label} {nseg}x{Ls} M={M}: worst err/bar {ratio:.3f}; hi-only activations x{mx:.1f}, hi-only weights x{mw:.1f}')
    assert ratio <= 1.0
    assert mx > 1.0 and mw > 1.0, f'{label}: the bar does not see hi-only operands'


@torch.no_grad()
@pytest.mark.parametrize('key', list(SPLIT), ids=_ids(SPLIT))
def test_split_launch(key):
    R, H = key[1]
    x = randn((R, H), R + H, 3.0)
    rows = (R + 999) // 1000 * 1000
    buf, y = guarded(rows * 2 * H, F16, device=DEV)
    y.zero_()
    capi.check(capi.lib().r3dp_a2m_split(capi.ptr(x), R, H, at(y), None, capi.stream()))
    torch.cuda.synchronize()
    assert guards_intact(buf, y.numel())
    yv = y.view(rows, 2 * H)
    assert torch.equal(yv[:R], torch.cat(split(x), 1)) and bool((yv[R:] == 0).all())


# ---- the recorded launches -----------------------------------------------------------------------------------------------------------------
def _has_row(fn, a):
    """Whether a launch has a float64 row here, or (the clip statistics, whose arguments are the clip length alone) in
    test_gpu_hubert_kernels.py::test_stats, which runs clips of up to 3 000 001 samples."""
    if fn == 'r3dp_hb_stats':
        return a[0] <= 3_000_001
    return (fn, a) in TABLES.get(fn, {})


class _HubertCalls(Recorder):
    """Records every r3dp_hb_* and r3dp_a2m_split call as its signature (attention's segment lengths copied out of their ctypes array), with
    capi.ptr wrapped so that the split operands they read can be looked at."""

    def __init__(self, lib):
        super().__init__(lib, lambda n: n.startswith('r3dp_hb_') or n == 'r3dp_a2m_split', ptrs=True)
        self.dead = []

    def check_lo(self, name, args):
        """A split operand [rows, hi | lo] that a GEMM, attention or positional-conv launch reads: where |hi| >= 1/4 the lo half is a normal
        fp16 and zero only when the fp32 value is fp16-exact (about 2^-13 of values), so an operand written without its lo halves shows as
        zeros.  (Smaller values, e.g. GELU's tails, have lo halves that underflow to zero.)"""
        half = {'r3dp_hb_gemm': 4, 'r3dp_hb_attention': 3, 'r3dp_hb_pos_conv': 4}.get(name)
        if half is None:
            return
        t, half = self.tensor(args[0].value), args[half]
        torch.cuda.synchronize()
        t = t.view(t.shape[0], -1)
        hi, lo = t[:, :half], t[:, half:2 * half]
        live = hi.abs() >= 0.25
        frac = float(((lo == 0) & live).sum()) / max(1, int(live.sum()))
        if frac > 0.01:
            self.dead.append(f'{name}: {frac:.1%} of the operand\'s lo halves are zero')

    def record(self, name, args):
        self.check_lo(name, args)
        fn, a = call_signature(name, args)
        if name == 'r3dp_hb_attention':
            a = a[:4] + (tuple(a[4][i] for i in range(a[5])),) + a[5:]
        return fn, a


@torch.no_grad()
def test_launches_have_rows(models):
    launched, missing = set(), []
    runs = [(name, T, None) for name, T in PLANS] + [(name, None, 2) for name in CFG]
    with _HubertCalls(capi.lib()) as rec:
        for name, T, B in runs:
            m = models[name][0]
            rec.clear()
            if B is None:
                get_hubert_from_16k_speech(hr.wave(clip(T)), m)
                want = hr.launch_plan(CFG[name], clip(T))
                label = f'{name}-T{T}'
            else:
                m(randn((B, FORWARD_LX), 5))
                want = hr.launch_plan(CFG[name], FORWARD_LX, B=B)
                label = f'{name}-forward-B{B}'
            got = rec.calls[:]
            assert_plan(got, [hr.launch_signature(f, a) for _, f, a in want], label)
            if name == 'large' and B is None:
                print(f'{label}: {len(got)} launches = 1 + 186 x {(len(got) - 1) // 186} groups')
                assert (len(got) - 1) % 186 == 0
            for fn, a in got:
                launched.add((fn, a))
                if not _has_row(fn, a):
                    missing.append(f'{label}: {fn}{a}')
        torch.cuda.synchronize()
    assert not rec.dead, 'split operands without their lo halves:\n' + '\n'.join(rec.dead[:20])
    stale = [f'{fn}: {v[1]} {k}' for fn, table in TABLES.items() for k, v in table.items() if k not in launched]
    assert_rows(missing, stale, 'the forwards')
