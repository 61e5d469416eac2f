"""SegFormerSECC2PlaneBackbone(precision='tc_exact') on the H100.

1. Every split entry point of the backbone (secc2plane_exact_reference.SPLIT_ENTRY_POINTS) at each distinct launch of `forward` at 512^2
   (B = 4, 1), 480^2, 96^2 and 32^2 (B = 3), against float64 of the operands it reads (hi + lo of split operands):
       |got - ref| <= alpha |ref| + beta S + floor,  S = max |ref|,
   alpha the storage rounding (2^-22 for split rows, 2^-24 for fp32), floor half the fp16 subnormal spacing (the lo half), beta per entry
   point about 2x the worst value measured (BETA).  Every output sits between sentinel guards and every element is written.  The same
   launch fed the hi halves alone (fp32 operands: rounded to fp16), and its output's hi half alone, break the bar.
2. Every distinct split r3dp_mf_conv3d and r3dp_sr_tcx_conv launch of `forward` at its exact arguments, on the module's packing of seeded
   float64 weights, against float64 (S: the same conv on |x|, |w|, |b|); the recorded calls of `forward` equal launch_plan_exact and every
   call has a row here.
3. The whole backbone against the float64 restatement at 512^2 (B = 4, 1), 480^2, 96^2 and 32^2 in both pncc_cond_modes, and against the
   reference's fixture, at BAR (at least 10x below the `tc` tests' 3e-3 of range); the `tc` module fails BAR on the same inputs.
4. planes_cl == forward bit for bit.
5. FrameEngine(sr_mode='tc_exact') with a tc_exact backbone: every frame equals RenderHead.synthesis on (canonical, backbone.planes_cl(secc))
   bit for bit, for the plain head, the torso head, the coefficient path with blink, and a second clip through the same graphs; and the
   concat_debug strips equal their restatement."""
import random

import pytest
import torch
import torch.nn.functional as F

import real3dportrait_b200 as r3
import secc2plane_exact_reference as xref
import secc2plane_reference as ref
import sr_conv_reference as scr
from conftest import load_golden
from launch_harness import (GUARD, Recorder, assert_plan, assert_rows, assert_written, call_signature, conv3d, guarded, inside, split_store)
from real3dportrait_b200 import _capi as capi, engine, secc2plane as sp, sr_tc, synthetic as syn
from torso_motion_reference import ref_conv

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
F16, F32, F64 = torch.float16, torch.float32, torch.float64
PLAN_SIZES = [(512, 4), (512, 1), (480, 3), (96, 3), (32, 3)]
ALPHA = {'split': scr.ALPHA_SPLIT, 'f32': scr.ALPHA_F32}
FLOOR = scr.FLOOR_F16
#: per entry point, about 2x the worst beta measured over its rows on an H100 80GB HBM3 (700 W power limit; DESIGN.md, "SECC -> plane
#: backbone in tc_exact").  Worst rows: upsample2_flip_split 1.27e-5 (the fp32 interpolation weights, as in the tc kernel), attention_split
#: 1.01e-6 (512^2 stage 4), dwconv_gelu_split 7.7e-8, layernorm_split 6.3e-8, head_fuse_split 5.3e-8; leaky_split and patches_split 0
BETA = {'r3dp_sp_layernorm_split': 1.3e-7, 'r3dp_sp_patches_split': 0.0, 'r3dp_sp_attention_split': 2e-6, 'r3dp_sp_dwconv_gelu_split': 1.5e-7,
        'r3dp_sp_head_fuse_split': 1.1e-7, 'r3dp_sp_leaky_split': 1.5e-8, 'r3dp_sp_upsample2_flip_split': 2.5e-5}
#: split r3dp_mf_conv3d / r3dp_sr_tcx_conv against S = the conv on |x|, |w|, |b|, 1 tap (GEMMs) and 9 taps: worst measured 1.17e-6 (512^2
#: stage 1 sr, K = 2048) and 2.52e-6 (512^2 to_plane_cnn.0 on r3dp_sr_tcx_conv)
BETA_CONV = {1: 2.5e-6, 9: 5e-6}
#: the whole backbone: |got - ref| <= BAR * max |ref|; measured at most 3.9e-5 (512^2), the `tc` module 7.1e-4 to 9.8e-4 on the same inputs
BAR = 1e-4
P = capi.ptr


def _rows(fns):
    out = {}
    for H, B in PLAN_SIZES:
        for tag, f, a in xref.launch_plan_exact(H, B):
            if f in fns:
                out.setdefault(ref.launch_signature(f, a), f'{H}^2-B{B}-{tag}')
    return out


SP_ROWS = _rows(set(xref.SPLIT_ENTRY_POINTS))
SP_KEYS = list(SP_ROWS)
CONV_ROWS = _rows({'r3dp_mf_conv3d', 'r3dp_sr_tcx_conv'})
CONV_KEYS = list(CONV_ROWS)


def _g(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _rand(shape, g, scale=1.0):
    return torch.randn(shape, generator=g, device=DEV) * scale


def _split(v):
    """fp32 [..., C] -> split rows [..., 2C] and the float64 value they hold."""
    t = split_store(v, 2 * v.shape[-1], v.shape[-1], True)
    return t, t[..., :v.shape[-1]].double() + t[..., v.shape[-1]:].double()


def _hi_only(t):
    """split rows with the lo half zeroed"""
    u = t.clone()
    u[..., u.shape[-1] // 2:] = 0
    return u


def _joined(y, C):
    return y[..., :C].double() + y[..., C:].double()


def _excess(got, want, alpha):
    S = float(want.abs().max())
    e = (got.double() - want).abs() - alpha * want.abs() - FLOOR
    return max(float(e.max()), 0.0) / S


# ---- 1. the split sp entry points -------------------------------------------------------------------------------------------------------
def _launch_sp(fn, a, g, hi_only):
    """One launch at plan row a on seeded operands -> (outputs [(name, guarded buf, output, row width, form, float64 ref)], hi-only-ref
    check done by the caller).  hi_only: split inputs with their lo halves zeroed, fp32 inputs rounded to fp16."""
    L, st = capi.lib(), capi.stream()
    r16 = (lambda v: v.half().float()) if hi_only else (lambda v: v)                  # noqa: E731
    lo0 = _hi_only if hi_only else (lambda t: t)                                       # noqa: E731
    if fn == 'r3dp_sp_layernorm_split':
        R, C, eps, yhs, yhlo = a
        x, t = _rand((R, C), g, 2.0), _rand((R, C), g)
        gam, bet = 1 + _rand((C,), g, 0.2), _rand((C,), g, 0.1)
        xk, tk = r16(x), r16(t)
        bx, xo = guarded(R * C, F32, device=DEV)
        by, yh = guarded(R * yhs, F16, device=DEV)
        capi.check(L.r3dp_sp_layernorm_split(P(xk), P(tk), R, C, P(gam), P(bet), eps, P(xo), P(yh, F16), yhs, yhlo, st))
        v = xk.double() + tk.double()
        return [('xo', bx, xo, C, 'f32', v), ('y', by, yh, yhs, 'split', F.layer_norm(v, (C,), gam.double(), bet.double(), eps))]
    if fn == 'r3dp_sp_patches_split':
        B, h, _, C, k, s, p = a
        x, xv = _split(_rand((B, h, h, C), g))
        x = lo0(x)
        xv = x[..., :C].double() + x[..., C:].double()
        ho = (h + 2 * p - k) // s + 1
        K = k * k * C
        by, y = guarded(B * ho * ho * 2 * K, F16, device=DEV)
        capi.check(L.r3dp_sp_patches_split(P(x, F16), B, h, h, C, k, s, p, P(y, F16), st))
        cols = F.unfold(xv.permute(0, 3, 1, 2), k, padding=p, stride=s)
        want = cols.view(B, C, k * k, -1).permute(0, 3, 2, 1).reshape(B * ho * ho, K)
        return [('y', by, y, 2 * K, 'split', want)]
    if fn == 'r3dp_sp_attention_split':
        C, kvs, B, Tq, Tk, heads, scale, os_, olo = a
        q, kv = r16(_rand((B * Tq, C), g)), r16(_rand((B * Tk, kvs), g))
        bo, o = guarded(B * Tq * os_, F16, device=DEV)
        capi.check(L.r3dp_sp_attention_split(P(q), C, P(kv), kvs, B, Tq, Tk, heads, scale, P(o, F16), os_, olo, st))
        qd = q.double().view(B, Tq, heads, 32).transpose(1, 2)
        kd = kv.double()[:, :C].view(B, Tk, heads, 32).transpose(1, 2)
        vd = kv.double()[:, C:].view(B, Tk, heads, 32).transpose(1, 2)
        want = ((qd @ kd.transpose(-1, -2)) * float(torch.tensor(scale, dtype=F32))).softmax(-1) @ vd
        return [('o', bo, o, os_, 'split', want.transpose(1, 2).reshape(B * Tq, C))]
    if fn == 'r3dp_sp_dwconv_gelu_split':
        B, h, w, C = a
        x = r16(_rand((B, h, w, C), g))
        wt, b = _rand((C, 9), g, 1 / 3), _rand((C,), g, 0.1)
        by, y = guarded(B * h * w * 2 * C, F16, device=DEV)
        capi.check(L.r3dp_sp_dwconv_gelu_split(P(x), B, h, w, C, P(wt), P(b), P(y, F16), st))
        z = F.conv2d(x.double().permute(0, 3, 1, 2), wt.double().view(C, 1, 3, 3), b.double(), 1, 1, groups=C)
        return [('y', by, y, 2 * C, 'split', F.gelu(z).permute(0, 2, 3, 1).reshape(-1, C))]
    if fn == 'r3dp_sp_head_fuse_split':
        hs, B = a[:4], a[4]
        gs = [r16(_rand((B, hh, hh, 256), g)) for hh in hs]
        bias = _rand((256,), g, 0.1)
        by, y = guarded(B * hs[0] * hs[0] * 512, F16, device=DEV)
        capi.check(L.r3dp_sp_head_fuse_split(P(gs[0]), hs[0], P(gs[1]), hs[1], P(gs[2]), hs[2], P(gs[3]), hs[3], B, P(bias), P(y, F16), st))
        acc = bias.double()[None, :, None, None]
        for t, hh in zip(gs, hs):
            t = t.double().permute(0, 3, 1, 2)
            acc = acc + (F.interpolate(t, size=(hs[0], hs[0]), mode='bilinear', align_corners=False) if hh != hs[0] else t)
        return [('y', by, y, 512, 'split', acc.relu().permute(0, 2, 3, 1).reshape(-1, 256))]
    if fn == 'r3dp_sp_leaky_split':
        Pn, C, slope = a
        x, _ = _split(_rand((Pn, C), g))
        x = lo0(x)
        xv = _joined(x, C)
        by, y = guarded(Pn * 2 * C, F16, device=DEV)
        y.copy_(x.view(-1))
        capi.check(L.r3dp_sp_leaky_split(P(y, F16), Pn, C, slope, st))
        return [('y', by, y, 2 * C, 'split', torch.where(xv >= 0, xv, xv * float(torch.tensor(slope, dtype=F32))))]
    if fn == 'r3dp_sp_upsample2_flip_split':
        B, h, w, C = a
        x, _ = _split(_rand((B, h, w, C), g))
        x = lo0(x)
        xv = _joined(x, C)
        n = B * 4 * h * w * 2 * C
        br, yr = guarded(n, F16, device=DEV)
        brc, yrc = guarded(n, F16, device=DEV)
        capi.check(L.r3dp_sp_upsample2_flip_split(P(x, F16), B, h, w, C, P(yr, F16), P(yrc, F16), st))
        u = F.interpolate(xv.permute(0, 3, 1, 2), scale_factor=2.0, mode='bilinear', align_corners=True)
        return [('yr', br, yr, 2 * C, 'split', u.flip(2).permute(0, 2, 3, 1).reshape(-1, C)),
                ('yrc', brc, yrc, 2 * C, 'split', u.flip(2, 3).permute(0, 2, 3, 1).reshape(-1, C))]
    raise AssertionError(fn)


@torch.no_grad()
@pytest.mark.parametrize('key', SP_KEYS, ids=[f'{SP_ROWS[k]}' for k in SP_KEYS])
def test_split_entry_point_vs_float64(key):
    fn, a = key
    tag = SP_ROWS[key]
    beta = BETA[fn]
    outs = _launch_sp(fn, a, _g(SP_KEYS.index(key) + 900), False)
    for name, buf, y, vs, form, want in outs:
        C = want.shape[-1]
        assert_written(buf, y, vs, inside(vs, 0, C, C, form == 'split', device=DEV), f'{tag} {name}')
        yv = y.view(-1, vs)
        got = _joined(yv, C) if form == 'split' else yv.double()
        b = _excess(got, want, ALPHA[form])
        print(f'{tag} {name}: beta = {b:.2e} (bar {beta:.1e})')
        assert b <= beta, (tag, name, b, beta)
        if form == 'split':
            assert _excess(yv[:, :C].double(), want, ALPHA[form]) > beta, f'{tag} {name}: the output hi half alone meets the bar'
    # the same launch fed the hi halves alone breaks the bar on its split output
    outs = _launch_sp(fn, a, _g(SP_KEYS.index(key) + 900), True)
    name, _, y, vs, form, _ = outs[-1]
    C = outs[-1][-1].shape[-1]
    full = [o for o in _launch_sp(fn, a, _g(SP_KEYS.index(key) + 900), False) if o[0] == name][0][-1]
    hi = _joined(y.view(-1, vs), C)
    assert _excess(hi, full, ALPHA[form]) > beta, f'{tag}: fed hi halves alone, it still meets the bar'


# ---- 2. the split convolutions ----------------------------------------------------------------------------------------------------------
@torch.no_grad()
@pytest.mark.parametrize('key', CONV_KEYS, ids=[CONV_ROWS[k] for k in CONV_KEYS])
def test_split_conv_launch_vs_float64(key):
    fn, a = key
    tag = CONV_ROWS[key]
    g = _g(CONV_KEYS.index(key) + 1700)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV, dtype=F64)               # noqa: E731
    if fn == 'r3dp_sr_tcx_conv':
        N, _, I, O, H, W, k, act = a
        conv = torch.nn.Conv2d(I, O, 3, 1, 1).to(DEV)
        conv.weight.data.copy_(rn(O, I, 3, 3) / (9 * I) ** 0.5)
        conv.bias.data.copy_(0.1 * rn(O))
        wp, bias, _ = sr_tc.pack_plain(conv, I, split=True)
        x, xv = _split(torch.randn(N, H, W, I, generator=g, device=DEV))
        buf, y = guarded(N * H * W * 2 * O, F16, device=DEV)

        def run(xx, yy):
            capi.check(capi.lib().r3dp_sr_tcx_conv(P(xx, F16), P(wp, F16), P(bias), N, 1, I, O, H, W, k, act, P(yy, F16), capi.stream()))
        run(x, y)
        assert_written(buf, y, 2 * O, inside(2 * O, 0, O, O, True, device=DEV), tag)
        w64 = conv.weight.double()
        pre = F.conv2d(xv.permute(0, 3, 1, 2), w64, conv.bias.double(), 1, 1)
        want = F.leaky_relu(pre, 0.01).permute(0, 2, 3, 1)
        S = F.conv2d(xv.abs().permute(0, 3, 1, 2), w64.abs(), conv.bias.double().abs(), 1, 1).permute(0, 2, 3, 1)
        got = _joined(y.view(N, H, W, 2 * O), O)
        taps = 9
        alpha, extra = scr.ALPHA_SPLIT, FLOOR
        xh = _hi_only(x)
        _, yh = guarded(N * H * W * 2 * O, F16, device=DEV)
        run(xh, yh)
        got_hi = _joined(yh.view(N, H, W, 2 * O), O)
    else:
        xs, xlo, cin, N, D, H, W, kd, kh, kw, _, O, cop, _, ys, yc0, ylo, out_f32, _ = a
        taps = kd * kh * kw
        if taps == 9:
            w, b = rn(O, cin, 3, 3) / (9 * cin) ** 0.5, 0.1 * rn(O)
            pk = sp._pack_taps(w, b, DEV, split=True)
        else:
            w, b = rn(O, cin) / cin ** 0.5, 0.1 * rn(O)
            pk = sp._pack_gemm(w, b, DEV, split=True)
        assert pk.cop == cop, (tag, pk.cop, cop)
        M = N * D * H * W
        v = torch.randn(N, D, H, W, cin, generator=g, device=DEV)
        x = split_store(v, xs, xlo, True)
        xv = x[..., :cin].double() + x[..., xlo:xlo + cin].double()
        dt = F32 if out_f32 else F16
        buf, y = guarded(M * ys, dt, tail=max(GUARD, (cop - O) * ys), device=DEV)
        conv3d(a, x, pk.w, pk.bias, None, y)
        assert_written(buf, y, ys, inside(ys, yc0, O, ylo, not out_f32, device=DEV), tag)
        wv = pk.w.double().view(taps, cop, 2 * cin)
        wd = ((wv[..., :cin] + wv[..., cin:]) / 1024.0)[None, :, :O]
        k0 = N - 1 if taps == 9 and H >= 256 else 0                 # a 256^2 last conv is checked on its last image
        xd = xv[k0:].permute(0, 4, 1, 2, 3)
        want = ref_conv(xd, wd, (kd, kh, kw), False, pk.bias[:O].double()).permute(0, 2, 3, 4, 1)
        S = ref_conv(xd.abs(), wd.abs(), (kd, kh, kw), False, pk.bias[:O].double().abs()).permute(0, 2, 3, 4, 1)

        def out_of(yy):
            yv = yy.view(N, D, H, W, ys)[k0:]
            return yv[..., yc0:yc0 + O].double() if out_f32 else yv[..., yc0:yc0 + O].double() + yv[..., ylo + yc0:ylo + yc0 + O].double()
        got = out_of(y)
        alpha, extra = (scr.ALPHA_F32, 0.0) if out_f32 else (scr.ALPHA_SPLIT, FLOOR)
        xh = x.clone()
        xh[..., xlo:xlo + cin] = 0
        _, yh = guarded(M * ys, dt, tail=max(GUARD, (cop - O) * ys), device=DEV)
        conv3d(a, xh, pk.w, pk.bias, None, yh)
        got_hi = out_of(yh)
    beta = BETA_CONV[taps]
    scr.check_bound(got, want, S, alpha, beta, extra, tag=tag)
    assert scr.excess_ratio(got_hi, want, S, alpha, extra) > beta, f'{tag}: fed hi halves alone, it still meets the bar'


@torch.no_grad()
def test_backbone_launches_equal_the_plan_and_have_rows():
    m = _module(precision='tc_exact', seed=3)
    m._prepared()
    sel = lambda n: n.startswith('r3dp_sp_') or n in ('r3dp_mf_conv3d', 'r3dp_sr_tcx_conv', 'r3dp_sr_tc_conv', 'r3dp_hb_layernorm')  # noqa: E731
    missing = []
    with Recorder(capi.lib(), sel) as rec:
        for H, B in PLAN_SIZES:
            cano, src, tgt = ref.make_inputs(B, H, 11)
            rec.calls.clear()
            m(torch.cat([cano.expand(B, -1, -1, -1), src.expand(B, -1, -1, -1), tgt], 1).to(DEV))
            got = [call_signature(n, a) for n, a in rec.calls]
            assert_plan(got, [ref.launch_signature(f, a) for _, f, a in xref.launch_plan_exact(H, B)], f'tc_exact {H}^2 B={B}')
            for s in got:
                if s[0] in xref.SPLIT_ENTRY_POINTS and s not in SP_ROWS or s[0] in ('r3dp_mf_conv3d', 'r3dp_sr_tcx_conv') and s not in CONV_ROWS:
                    missing.append(f'{H}^2 B={B}: {s}')
        torch.cuda.synchronize()
    assert_rows(missing, [], 'the tc_exact backbone')


# ---- 3, 4. the whole backbone ------------------------------------------------------------------------------------------------------------
def _module(mode='cano_src_tgt', seed=7, precision='tc_exact'):
    m = r3.SegFormerSECC2PlaneBackbone(pncc_cond_mode=mode, precision=precision)
    m.load_state_dict(ref.make_params({k: v.shape for k, v in m.state_dict().items()}, seed), strict=True)
    return m.to(DEV).eval()


def _rel(got, want):
    return float((got.double() - want.double()).abs().max()) / float(want.double().abs().max())


@torch.no_grad()
def test_backbone_matches_reference_fixture():
    gd = load_golden('secc2plane_small')
    cano, src, tgt = ref.make_inputs(1, int(gd['size']), int(gd['input_seed']))
    x = torch.cat([cano, src, tgt], 1).to(DEV)
    r = _rel(_module(seed=int(gd['param_seed']))(x)[..., ::2, ::2].cpu(), gd['planes_s2'])
    r_tc = _rel(_module(seed=int(gd['param_seed']), precision='tc')(x)[..., ::2, ::2].cpu(), gd['planes_s2'])
    print(f'secc2plane tc_exact 128^2 vs reference fixture: max err / range = {r:.2e} (tc {r_tc:.2e})')
    assert r < BAR, r


@torch.no_grad()
@pytest.mark.parametrize('H,B', [(512, 4), (512, 1), (480, 3), (96, 3), (32, 3)])
@pytest.mark.parametrize('mode', ['cano_src_tgt', 'cano_tgt'])
def test_backbone_matches_float64(H, B, mode):
    m, mt = _module(mode), _module(mode, precision='tc')
    sd = ref.to64(m.state_dict(), DEV)
    cano, src, tgt = ref.make_inputs(B, H, 3)
    parts = [cano, src] if mode == 'cano_src_tgt' else [cano]
    x = torch.cat([p.expand(B, -1, -1, -1) for p in parts] + [tgt], 1).to(DEV)
    want = ref.forward(sd, x.double())
    r, r_tc = _rel(m(x), want), _rel(mt(x), want)
    print(f'secc2plane {H}^2 B={B} ({mode}) vs float64: tc_exact {r:.2e}, tc {r_tc:.2e} of range')
    assert r < BAR, r
    assert r_tc > BAR, r_tc                                      # the bar tells split fp16 from fp16


@torch.no_grad()
def test_planes_cl_equals_forward():
    m = _module()
    cano, src, tgt = (t.to(DEV) for t in ref.make_inputs(2, 512, 5))
    full = m(torch.cat([cano.expand(2, -1, -1, -1), src.expand(2, -1, -1, -1), tgt], 1))
    m.begin_clip(cano, src)
    pcl = m.planes_cl(tgt)
    assert pcl.layout == 'hwpc' and tuple(pcl.data.shape) == (2, 256, 256, 3, 32) and pcl.data.dtype == F32
    assert torch.equal(pcl.data.permute(0, 3, 4, 1, 2), full)
    m.begin_clip(-cano, src)
    full2 = m(torch.cat([-cano.expand(2, -1, -1, -1), src.expand(2, -1, -1, -1), tgt], 1))
    assert torch.equal(m.planes_cl(tgt).data.permute(0, 3, 4, 1, 2), full2)
    for k in range(2):                                           # frame k alone is bit-identical to frame k of the batch
        assert torch.equal(m(torch.cat([cano, src, tgt[k:k + 1]], 1)), full[k:k + 1])


# ---- 5. the engine ----------------------------------------------------------------------------------------------------------------------
EB = 2
TORSO_HP = dict(syn.WARP_HPARAMS, htbsr_head_weight_fuse_mode='v2', num_samples_fine=48, neural_rendering_resolution=64)


def _engine(torso=False, **kw):
    kw.setdefault('out_uint8', True)
    if torso:
        eng = engine.FrameEngine(batch=EB, sr_mode='tc_exact', hp=TORSO_HP, torso_model=syn.StubTorsoModel(), secc2plane=_module(), **kw)
        eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_warp_params(seed=6, fuse_mode='v2'))
        inp = syn.make_warp_inputs(1, seed=3)
        eng.begin_clip(*(inp[k].to(DEV) for k in ('ref_torso_rgb', 'ref_bg_rgb', 'segmap', 'kp_s')))
    else:
        eng = engine.FrameEngine(batch=EB, sr_mode='tc_exact', hp={'num_samples_fine': 0}, secc2plane=_module(), **kw)
        eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_params(seed=5))
    return eng


def _steps(n, torso, seed=40):
    out = []
    for s in range(n):
        _, _, tgt = ref.make_inputs(EB, 512, seed + s)
        u_c, u_f = syn.make_jitter(EB, 4096, 48, 48 if torso else 0, seed=seed + s + 100)
        kp = (torch.rand(EB, 68, 3, generator=torch.Generator().manual_seed(seed + s + 300)) * 2 - 1).to(DEV) if torso else None
        out.append((tgt.to(DEV), syn.make_cameras(EB, seed=seed + s + 200).to(DEV), u_c.to(DEV), None if u_f is None else u_f.to(DEV), kp))
    return out


def _clip(seed):
    cano, src, _ = ref.make_inputs(1, 512, seed)
    return syn.make_planes(1, seed=seed).to(DEV), cano.to(DEV), src.to(DEV)


def _synthesis(eng, secc, f):
    """RenderHead.synthesis on (the clip's canonical planes, the engine's backbone's planes_cl(secc)), as the step calls it."""
    cond = None
    if eng.torso:
        cond = eng._cond(f[4])
    over = {'u_coarse': f[2]} if f[3] is None else {'u_coarse': f[2], 'u_fine': f[3]}
    return eng.head.synthesis((eng._cano_cl, eng.secc.planes_cl(secc)), f[1], cond=cond, lean=True, out_uint8=eng.out_uint8, **over)['image']


def _check_clip(eng, steps, kw_of, secc_of):
    for f in steps:
        got = eng.step(None, *f[1:4], **kw_of(f)).clone()
        assert torch.equal(got, _synthesis(eng, secc_of(f), f))


@torch.no_grad()
@pytest.mark.parametrize('torso', [False, True])
def test_engine_frames_equal_synthesis_on_the_backbone_planes(torso):
    eng = _engine(torso)
    assert eng.secc.precision == 'tc_exact'
    steps = _steps(2, torso)
    kw_of = (lambda f: {'cond_tgt': f[0], 'kp_d': f[4]}) if torso else (lambda f: {'cond_tgt': f[0]})      # noqa: E731
    eng.begin_planes(*_clip(1))
    _check_clip(eng, steps, kw_of, lambda f: f[0])
    graph = eng.graph
    # prepare(): zero-copy graphs, then a second clip refilled in place through the same graphs
    assert eng.prepare([f[:5] if torso else f[:3] for f in steps]) == len(steps)
    _check_clip(eng, steps, kw_of, lambda f: f[0])
    eng.begin_planes(*_clip(2))
    assert eng.graph is graph
    _check_clip(eng, steps, kw_of, lambda f: f[0])


@torch.no_grad()
def test_engine_coefficients_with_blink(tmp_path):
    r = r3.SECC_Renderer(512, device=DEV, **syn.write_bfm_folder(str(tmp_path), seed=0))
    eng = _engine(secc_renderer=r, blink=True)
    sched = r3.period_blink_schedule(3 * EB, rng=random.Random(3))
    steps = []
    for s, f in enumerate(_steps(3, False)):
        cc = syn.make_coeffs(EB, seed=50 + s)
        steps.append((torch.cat([cc['id'], cc['exp'], sched[s * EB:(s + 1) * EB].float()], 1).to(DEV),) + f[1:])

    def secc_of(f):
        secc = r.render(f[0][:, :144])[1]
        r.blink(secc, rows=f[0][:, 144:])
        return secc
    for clip in (1, 2):
        c = syn.make_coeffs(1, seed=clip)
        eng.begin_planes(syn.make_planes(1, seed=clip).to(DEV), coeff_src=torch.cat([c['id'], c['exp']], 1).to(DEV))
        _check_clip(eng, steps, lambda f: {'coeff': f[0]}, secc_of)


@torch.no_grad()
def test_engine_concat_debug():
    import test_gpu_debug_engine as tde
    dbg, fin = _engine(out_mode='concat_debug'), _engine(out_uint8=False)
    cano, c_cano, c_src = _clip(1)
    for e in (dbg, fin):
        e.begin_planes(cano, c_cano, c_src)
    steps = [f[:3] + (None, None) for f in _steps(2, False)]
    got, want = tde._run_clip(dbg, fin, steps, 2 * EB, tde._ref_gt(), lambda f: f[0], lambda f: {'cond_tgt': f[0]})
    assert torch.equal(got, want)


@torch.no_grad()
def test_tc_backbone_in_a_tc_exact_engine_is_unchanged():
    """FrameEngine(sr_mode='tc_exact') with a `tc` backbone renders the `tc` planes."""
    eng = engine.FrameEngine(batch=EB, sr_mode='tc_exact', hp={'num_samples_fine': 0}, secc2plane=_module(precision='tc'), out_uint8=True)
    eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_params(seed=5))
    eng.begin_planes(*_clip(1))
    assert eng.secc.precision == 'tc'
    _check_clip(eng, _steps(1, False), lambda f: {'cond_tgt': f[0]}, lambda f: f[0])
