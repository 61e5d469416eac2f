"""Every launch of the audio2secc VAE's forward (PitchContourVAEModel, VAEModel) at its exact arguments against float64, and a recorded-launch
check that keeps these tables equal to what the module launches.

* CONV3D holds one row per distinct r3dp_mf_conv3d launch of audio2motion_reference.launch_plan over (pitch, 1024) at (B, T_x) = (1, 8),
  (2, 400), (3, 1032), (1, 30000) and over (vae, 13) and (vae, 1024) at (2, 400): the encoders' k3 convs (GELU epilogue on enc1 / penc1;
  enc2 / penc2 into column slices of gcat), cond_proj, g_pre (k3 over groups of four frames, T/4 = 1 included), flow_cond, every flow's
  pre and post (post added in place into zb, res == y, as the module runs it), dec_cond, dec_pre (4 frames per row) and out_proj.
  - The weights are a seeded model's own _prepared() packing, so the padded couts and the Flip reversal are the module's; the float64
    reference is built from fold_weights' float64 weights, not from the packed halves, so a packing that drops a lo half or misorders a
    channel fails.  Inputs are random fp32, split by the test; channels the launch must not read are NaN.
  - Bound: sr_conv_reference.check_bound, |got - ref| <= alpha |ref| + extra + beta S, alpha of the stored form (ALPHA_F32, ALPHA_SPLIT
    with the fp16 subnormal floor), S the same conv on |x|, |w|, |b| (x 1.13, GELU's Lipschitz constant, on the GELU rows; + |res| on
    post), beta per K below.  Each row also asserts that the float64 result of its hi-only operands, and of its hi-only weights alone,
    breaks its own bar: the bar sees a lost lo half at every launch.
  - Sentinels around and between every output: the columns outside the slice stay untouched; post leaves zb's other channels and lo
    halves bit-identical.  The first and last frame of each batch item and the 128-row tile edges are checked on their own, so a leak
    across items is named; the last item equals its N = 1 launch (the last rows of a GEMM a launch on those rows alone) bit for bit.
* r3dp_a2m_input (frame mean at A = 13 and 1024 with zero pad columns; blink runs and the mouth / eye amplitudes given and absent),
  r3dp_a2m_split, r3dp_a2m_latent and r3dp_a2m_store: exact against torch between guards, at B*T up to 15000.
* test_forward_launches_have_rows records both classes' forward at several sizes: the calls equal launch_plan (42 for the released
  config), every launch has a row here or in test_gpu_audio2motion_kernels.py, and every conv row of the largest size is still launched."""
import pytest
import torch
import torch.nn.functional as F

import audio2motion_reference as ref
import sr_conv_reference as scr
from launch_harness import (Recorder, assert_plan, assert_rows, at, bits, call_signature, conv3d, guarded, guards_intact, hi_w, inside, join, split,
                            untouched)
from real3dportrait_b200 import PitchContourVAEModel, VAEModel, _capi as capi
from real3dportrait_b200.audio2motion import F0_MEL_MAX, F0_MEL_MIN, fold_weights

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
F16, F32 = torch.float16, torch.float32
#: (kind, A, B, T_x) of the plans the tables cover and the forward calls the recorded-launch test makes
PLANS = [('pitch', 1024, 1, 8), ('pitch', 1024, 2, 400), ('pitch', 1024, 3, 1032), ('pitch', 1024, 1, 30000), ('vae', 13, 2, 400),
         ('vae', 1024, 2, 400)]
LARGEST = PLANS[3]
GELU_LIP = 1.13                               # max |GELU'(x)| = 1.1289
#: beta per K = taps x cin (the products of one output; split runs three MMAs per product).  Worst excess / S over the rows on an H100
#: 80GB HBM3 (700 W power limit): 1.59e-6 at K = 3072 (enc1), 1.00e-6 at K = 1536 (g_pre), 6.6e-7 at K <= 384; every row's hi-only
#: weights break its beta by 4x or more (enc1: 1.58e-5 against 2^-19)
def beta_of(K):
    return 2.0 ** -19 if K > 384 else 2.0 ** -20


def _label(kind, A, B, Tx):
    return f'{kind}{A}-B{B}-Tx{Tx}'


def _rows(fn):
    """{signature: (kind, A, tag, plan label)} of one entry point over PLANS, the first of each distinct launch."""
    out = {}
    for kind, A, B, Tx in PLANS:
        for tag, f, a in ref.launch_plan(kind, A, B, Tx):
            if f == fn:
                out.setdefault(ref.launch_signature(f, a), (kind, A, tag, _label(kind, A, B, Tx)))
    return out


CONV3D = _rows('r3dp_mf_conv3d')
CONV3D_KEYS = list(CONV3D)


def _id(key):
    kind, A, tag, label = CONV3D[key]
    a = key[1]
    return f'{label}-{tag}-K{a[9] * a[2]}-N{a[3]}xW{a[6]}-O{a[11]}'


# ---- the models' packed and float64 weights ------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def models():
    out = {}
    for kind, A in (('pitch', 1024), ('vae', 13), ('vae', 1024)):
        m = PitchContourVAEModel(ref.HP_PITCH, audio_in_dim=A) if kind == 'pitch' else VAEModel(audio_in_dim=A)
        m.load_state_dict(ref.make_params({k: v.shape for k, v in m.state_dict().items()}, 11), strict=True)
        m = m.to(DEV).eval()
        with torch.no_grad():
            out[(kind, A)] = (m, m._prepared(), fold_weights(m))
    return out


def _weights(Q, P, tag):
    """(packed fp16, fp32 bias, O, cop) of the module and (W [O, I, k], b) float64 of fold_weights for one launch."""
    if tag.startswith('flow') and '.' in tag:
        n, part = int(tag[4]), tag.split('.')[1]
        q, p = Q['flows'][n][part], P['flows'][n][part]
    else:
        q, p = Q[tag], P[tag]
    if tag in ('enc2', 'penc2'):
        p = (p, torch.zeros(p.shape[0], dtype=torch.float64, device=DEV))
    w, b = p
    return q, (w if w.dim() == 3 else w[:, :, None], b)


def _conv64(x, w, b, k):
    """x [N, W, I] float64, w [O, I, k] -> [N, W, O] (zero padding per sequence)."""
    y = F.conv1d(x.transpose(1, 2), w, None, padding=k // 2).transpose(1, 2)
    return y if b is None else y + b


@torch.no_grad()
@pytest.mark.parametrize('key', CONV3D_KEYS, ids=[_id(k) for k in CONV3D_KEYS])
def test_conv3d_launch_vs_float64(models, key):
    kind, A, tag, label = CONV3D[key]
    a = key[1]
    xs, xlo, cin, N, _, _, W, _, _, k, _, O, cop, relu, ys, yc0, ylo, out_f32, _ = a
    name = f'{label} {tag}'
    _, Q, P = models[(kind, A)]
    (wp, bias, O_mod, cop_mod), (w64, b64) = _weights(Q, P, tag)
    assert (O_mod, cop_mod) == (O, cop), (name, O_mod, cop_mod)           # the module packs to the launch's couts
    I = w64.shape[1]
    M = N * W
    post = tag.endswith('.post')
    g = torch.Generator(device=DEV).manual_seed(CONV3D_KEYS.index(key) + 900)
    # input rows: split random fp32 in [0, cin) and [xlo, xlo + cin), NaN in every other half of the row
    xv = torch.randn(M, cin, generator=g, device=DEV)
    xb = torch.full((M, xs), float('nan'), device=DEV, dtype=F16)
    xb[:, :cin], xb[:, xlo:xlo + cin] = split(xv)
    dt = F32 if out_f32 else F16
    buf, y = guarded(M * ys, dt, device=DEV)
    yv = y.view(M, ys)
    mask = inside(ys, yc0, O, ylo, not out_f32, device=DEV)
    if post:                                  # zb as the module holds it: split state in every channel, post adds into its slice
        rv = torch.randn(M, 32, generator=g, device=DEV)
        yv[:, :32], yv[:, 32:] = split(rv)
        before = yv.clone()
    conv3d(a, at(xb), wp, bias, at(y) if post else None, at(y))
    torch.cuda.synchronize()
    assert guards_intact(buf, y.numel()), f'{name}: written outside the output'
    if post:
        assert torch.equal(yv[:, ~mask].view(torch.int16), before[:, ~mask].view(torch.int16)), f'{name}: other channels of zb changed'
    else:
        assert not bool(untouched(yv[:, mask]).any()), f'{name}: an output element was not written'
        assert bool(untouched(yv[:, ~mask]).all()), f'{name}: written outside the channel slice'
    got = (yv[:, yc0:yc0 + O].double() if out_f32 else join(yv, yc0, O, ylo)).view(N, W, O)

    x64 = xv.double().view(N, W, cin)[..., :I]
    pre = _conv64(x64, w64, b64, k)
    S = _conv64(x64.abs(), w64.abs(), b64.abs(), k)
    pre_hi = _conv64(x64.half().double(), hi_w(w64), b64, k)             # every operand its hi half alone
    pre_hw = _conv64(x64, hi_w(w64), b64, k)                             # the weights' hi halves alone
    if relu == 2:
        want, want_hi, want_hw, S = F.gelu(pre), F.gelu(pre_hi), F.gelu(pre_hw), GELU_LIP * S
    else:
        want, want_hi, want_hw = pre, pre_hi, pre_hw
    if post:
        r64 = join(before, yc0, O, ylo).view(N, W, O)
        want, want_hi, want_hw, S = want + r64, want_hi + r64, want_hw + r64, S + r64.abs()
    alpha = scr.ALPHA_F32 if out_f32 else scr.ALPHA_SPLIT
    extra = None if out_f32 else scr.FLOOR_F16                            # the lo half's fp16 subnormal floor
    beta = beta_of(k * cin)
    allow = alpha * want.abs() + beta * S + (extra or 0.0)
    bad = ~((got - want).abs() <= allow)
    # the sequence ends of each item and the 128-row tile edges first, so that a leak across items is named
    for b in range(N):
        for t in sorted({0, W - 1}):
            assert not bool(bad[b, t].any()), f'{name}: item {b} frame {t} outside the bound'
    m = torch.arange(M, device=DEV).view(N, W)
    edge = ((m % 128) == 0) | ((m % 128) == 127)
    assert not bool(bad[edge].any()), f'{name}: a 128-row tile edge outside the bound'
    scr.check_bound(got, want, S, alpha, beta, extra, tag=name)
    # the float64 results of hi-only operands break this bar
    for what, wh in (('hi-only operands', want_hi), ('hi-only weights', want_hw)):
        r = scr.excess_ratio(wh, want, S, alpha, extra)
        print(f'{name}: {what} excess / S = {r:.3e} = beta x {r / beta:.1f}')
        assert r > beta, f'{name}: the bar does not see {what}'
    # bit-exact: the last item equals its N = 1 launch; the last rows of a GEMM a launch on those rows alone
    r = W if k == 3 else min(W, 300)
    if k == 3 and N == 1:
        return
    one_buf, one = guarded(r * ys, dt, device=DEV)
    ov = one.view(r, ys)
    if post:
        ov.copy_(before[M - r:])
    conv3d(a, at(xb, (M - r) * xs), wp, bias, at(one) if post else None, at(one), N=1, W=r)
    torch.cuda.synchronize()
    assert guards_intact(one_buf, one.numel())
    assert torch.equal(bits(ov), bits(yv[M - r:])), f'{name}: last {r} rows vs a launch on them alone'


# ---- r3dp_a2m_input ------------------------------------------------------------------------------------------------------------------------
#: (A, Ap, mean) of the input rows: the frame mean at both widths here, the pitch path (mean 0) here and in test_gpu_audio2motion_kernels.py
INPUT_ROWS = {(13, 32, 1), (1024, 1024, 1), (1024, 1024, 0), (13, 32, 0)}


def _close(got, want):
    """hi + lo holds the value to 2^-21 relative, or to the fp16 subnormal step where the remainder is that small."""
    return bool(((got - want).abs() <= 2.0 ** -21 * want.abs() + 2.0 ** -24).all())


@torch.no_grad()
@pytest.mark.parametrize('A', [13, 1024])
@pytest.mark.parametrize('B,Tx', [(1, 8), (3, 1032), (1, 30000)])
def test_input_frame_mean(A, B, Tx):
    Ap = (A + 31) // 32 * 32
    T = Tx // 2
    C = Ap
    ys = 2 * C + 8                                                        # a frame stride beyond ylo + C
    audio = torch.randn(B, Tx, A, generator=torch.Generator().manual_seed(Tx + A), device='cpu').to(DEV)
    buf, y = guarded(B * T * ys, F16, device=DEV)
    capi.check(capi.lib().r3dp_a2m_input(capi.ptr(audio), B, Tx, A, Ap, 1, None, None, None, None, None, float(F0_MEL_MIN),
                                         float(F0_MEL_MAX - F0_MEL_MIN), at(y), ys, C, None, 576, 288, capi.stream()))
    torch.cuda.synchronize()
    yv = y.view(B * T, ys)
    assert guards_intact(buf, y.numel()) and bool(untouched(yv[:, 2 * C:]).all()), 'written beyond ylo + C'
    want = 0.5 * (audio[:, 0::2].double() + audio[:, 1::2].double())
    got = join(yv, 0, C, C).view(B, T, C)
    assert _close(got[..., :A], want)
    assert bool((yv[:, A:C] == 0).all()) and bool((yv[:, C + A:2 * C] == 0).all()), 'pad columns not zero'


@torch.no_grad()
@pytest.mark.parametrize('mouth,eye', [(True, False), (True, True), (False, False), (False, True)])
@pytest.mark.parametrize('blink', ['runs', 'none'])
def test_input_blink_and_amplitudes(mouth, eye, blink):
    """The pitch model's pack into the module's buffers: xin [B*T, hi C | lo C] and the block at columns 256 / 544 of gcat [B*T, 576]."""
    B, Tx, A = 3, 1032, 1024
    T, Ap, C = Tx // 2, 1024, 1024 + 128
    batch = ref.make_batch(B, Tx, A, seed=7)
    bl = batch['blink'].view(B, Tx).clone()
    bl[2] = 1 - bl[2]                                                     # item 2: runs of zeros in ones
    bl_d = bl.to(DEV).contiguous() if blink == 'runs' else None
    mouth_d = torch.tensor([0.45, 0.1, 1.3e-5], device=DEV) if mouth else None
    eye_d = torch.tensor([0.2, 0.7, 3.1], device=DEV) if eye else None
    audio, f0 = batch['audio'].to(DEV), batch['f0'].to(DEV)
    table = torch.randn(300, 128, generator=torch.Generator().manual_seed(2)).to(DEV)
    xbuf, xin = guarded(B * T * 2 * C, F16, device=DEV)
    gbuf, gcat = guarded(B * T * 576, F16, device=DEV)
    capi.check(capi.lib().r3dp_a2m_input(capi.ptr(audio), B, Tx, A, Ap, 0, capi.ptr(f0), capi.ptr(bl_d, torch.int64), capi.ptr(mouth_d),
                                         capi.ptr(eye_d), capi.ptr(table), float(F0_MEL_MIN), float(F0_MEL_MAX - F0_MEL_MIN), at(xin), 2 * C, C,
                                         at(gcat, 256), 576, 288, capi.stream()))
    torch.cuda.synchronize()
    assert guards_intact(xbuf, xin.numel()) and guards_intact(gbuf, gcat.numel())
    gv = gcat.view(B * T, 576)
    block = torch.zeros(576, dtype=torch.bool, device=DEV)
    block[256:288] = block[544:576] = True
    assert bool(untouched(gv[:, ~block]).all()), 'the block written outside gcat columns 256..287 / 544..575'
    got = join(gv, 256, 32, 288).view(B, T, 32)
    b0 = bl[:, ::2].to(DEV) if blink == 'runs' else torch.zeros(B, T, dtype=torch.long, device=DEV)
    assert torch.equal(got[..., 0], (b0 == 0).double()) and torch.equal(got[..., 1], (b0 == 1).double())
    for col, amp in ((2, mouth_d), (3, eye_d)):
        want = torch.zeros(B, T, dtype=torch.float64, device=DEV) if amp is None else amp.double()[:, None].expand(B, T)
        assert _close(got[..., col], want), col
    assert bool((gv[:, 260:288] == 0).all()) and bool((gv[:, 544:546] == 0).all()) and bool((gv[:, 548:576] == 0).all())
    assert _close(join(xin.view(B * T, 2 * C), 0, A, C).view(B, T, A), audio[:, ::2].double())


# ---- r3dp_a2m_split / _latent / _store -------------------------------------------------------------------------------------------------------
@torch.no_grad()
@pytest.mark.parametrize('which', ['y1', 'y4', 'both'])
@pytest.mark.parametrize('R,C', [(4, 128), (1032, 64), (15000, 128)])
def test_split_exact(which, R, C):
    x = torch.randn(R, C, generator=torch.Generator().manual_seed(R + C), device='cpu').to(DEV) * 3.0
    x[0, :4] = torch.tensor([0.0, 1e-6, -7e-8, 65000.0])                  # zero, subnormal remainders, a large value
    b1, y1 = guarded(R * 2 * C, F16, device=DEV)
    b4, y4 = guarded(R * 2 * C, F16, device=DEV)
    capi.check(capi.lib().r3dp_a2m_split(capi.ptr(x), R, C, at(y1) if which != 'y4' else None, at(y4) if which != 'y1' else None,
                                         capi.stream()))
    torch.cuda.synchronize()
    hi, lo = split(x)
    assert guards_intact(b1, y1.numel()) and guards_intact(b4, y4.numel())
    if which != 'y4':
        assert torch.equal(y1.view(R, 2 * C), torch.cat([hi, lo], 1))
    else:
        assert bool(untouched(y1).all())
    if which != 'y1':
        assert torch.equal(y4.view(R // 4, 8 * C), torch.cat([hi.reshape(R // 4, 4 * C), lo.reshape(R // 4, 4 * C)], 1))
    else:
        assert bool(untouched(y4).all())


@torch.no_grad()
@pytest.mark.parametrize('temperature', [0.0, 0.2, 1.0])
@pytest.mark.parametrize('B,T4', [(1, 1), (3, 129), (4, 3750)])
def test_latent_exact(temperature, B, T4):
    z = torch.randn(B, 16, T4, generator=torch.Generator().manual_seed(B * T4), device='cpu').to(DEV)
    buf, y = guarded(B * T4 * 64, F16, device=DEV)
    capi.check(capi.lib().r3dp_a2m_latent(capi.ptr(z), B, T4, temperature, at(y), capi.stream()))
    torch.cuda.synchronize()
    v = torch.zeros(B * T4, 32, device=DEV)
    v[:, :16] = (z * torch.tensor(temperature, dtype=F32, device=DEV)).transpose(1, 2).reshape(B * T4, 16)
    hi, lo = split(v)
    assert guards_intact(buf, y.numel())
    yv = y.view(B * T4, 64)
    assert torch.equal(yv, torch.cat([hi, lo], 1)) and bool((yv[:, 16:32] == 0).all()) and bool((yv[:, 48:] == 0).all())


@torch.no_grad()
@pytest.mark.parametrize('masked', [False, True])
@pytest.mark.parametrize('ld', [64, 146])
@pytest.mark.parametrize('N', [1, 1032, 15000])
def test_store_exact(masked, ld, N):
    g = torch.Generator().manual_seed(N + ld)
    x = torch.randn(N, 64, generator=g).to(DEV)
    mask = (torch.rand(N, generator=g) < 0.8).float().to(DEV) if masked else None
    buf, out = guarded(N * ld, F32, device=DEV)
    capi.check(capi.lib().r3dp_a2m_store(capi.ptr(x), capi.ptr(mask), N, 64, at(out), ld, capi.stream()))
    torch.cuda.synchronize()
    ov = out.view(N, ld)
    assert guards_intact(buf, out.numel()) and bool(untouched(ov[:, 64:]).all())
    assert torch.equal(ov[:, :64], x * mask[:, None] if masked else x)


# ---- the recorded launches -----------------------------------------------------------------------------------------------------------------
def _has_row(fn, a):
    """Whether a launch (entry point, non-pointer arguments) has a float64 row here or in test_gpu_audio2motion_kernels.py."""
    import test_gpu_audio2motion_kernels as kern
    if fn == 'r3dp_mf_conv3d':
        return (fn, a) in CONV3D
    if fn == 'r3dp_a2m_wn_layer':
        _, B, T, hidden, k, _, _ = a                  # every case runs as first, middle and last layer; B only sets the grid's y
        return any(H == hidden and kk == k and Tc >= T for H, kk, Tc, _ in kern.CASES)
    if fn == 'r3dp_a2m_input':
        return (a[2], a[3], a[4]) in INPUT_ROWS
    if fn == 'r3dp_a2m_split':
        return a[1] in (64, 128) and a[0] <= 15000
    if fn == 'r3dp_a2m_latent':
        return a[0] * a[1] <= 4 * 3750
    if fn == 'r3dp_a2m_store':
        return a[1] == 64 and a[2] in (64, 146) and a[0] <= 15000
    return False


@torch.no_grad()
def test_forward_launches_have_rows(models):
    launched, missing = {}, []
    with Recorder(capi.lib(), lambda n: n.startswith('r3dp_a2m_') or n == 'r3dp_mf_conv3d') as rec:
        for kind, A, B, Tx in PLANS:
            m = models[(kind, A)][0]
            batch = {k: v.to(DEV) for k, v in ref.make_batch(B, Tx, A, seed=Tx, pitch=kind == 'pitch').items()}
            rec.calls.clear()
            m(batch, {}, temperature=0.2)
            got = [call_signature(n, a) for n, a in rec.calls]
            label = _label(kind, A, B, Tx)
            assert_plan(got, [ref.launch_signature(f, a) for _, f, a in ref.launch_plan(kind, A, B, Tx, temperature=0.2)], label)
            if kind == 'pitch':
                assert len(got) == 42
            for fn, a in got:
                launched.setdefault((fn, a), label)
                if not _has_row(fn, a):
                    missing.append(f'{label}: {fn}{a}')
        torch.cuda.synchronize()
    largest = _label(*LARGEST)
    rows = {ref.launch_signature(f, a) for _, f, a in ref.launch_plan(*LARGEST[:2], *LARGEST[2:]) if f == 'r3dp_mf_conv3d'}
    stale = [f'{CONV3D[k][2]}: {k}' for k in CONV3D if (k in rows or CONV3D[k][3] == largest) and k not in launched]
    assert_rows(missing, stale, f'the {largest} forward')
