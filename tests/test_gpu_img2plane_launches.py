"""Every launch of Img2PlaneModel.forward at its exact arguments against float64, and a recorded-launch check that keeps these rows equal to
what the module launches.

* ROWS holds one row per distinct launch of img2plane_reference.launch_plan over PLAN_SIZES (512^2 at B = 4 and 1, 144^2 and 32^2 at
  B = 3, 16^2 at B = 1) and 64^2 at the small and large scales, keyed by img2plane_reference.row_key: the non-pointer arguments, and for
  r3dp_mf_conv3d whether it adds a residual and its input's channel offset, for r3dp_sp_layernorm which of t / xo / yf / yh it is given and
  whether xo is x (the in-place update of the residual stream).
* r3dp_mf_conv3d rows pack seeded float64 weights with the module's own packer (img2plane._Conv: the (1,3,3) taps, the 1x1 GEMM, the patch
  rows padded to a multiple of 32), so the padded couts (cop > cout) carry its zero filters.  Bound: sr_conv_reference's
  |got - ref| <= alpha |ref| + extra + beta S, S the same conv / GEMM on |x|, |w|, |b| (and |res|), beta per tap count (BETA below).
  Outputs sit between sentinel guards of at least (cop - cout) ys elements: every element of the slice is written and nothing else is.
  Bit-exact: the last image of a box conv equals its N = 1 launch, the last rows of a GEMM a launch on those rows alone.
* r3dp_sp_layernorm (every form the module passes, the in-place xo = x among them), r3dp_sp_dwconv_gelu (C = 2048), r3dp_sp_leaky
  (slope 0.01 and 0), r3dp_ip_attention at the module's strides (q 1024, kv 2048, o 1024) and the other r3dp_ip_* entry points, against
  float64 with the bars of tests/test_gpu_img2plane_kernels.py and tests/test_gpu_secc2plane_kernels.py, in sentinel-guarded outputs.
  r3dp_sp_patches_dil's rows are PATCH_ROWS of tests/test_gpu_img2plane_kernels.py (derived from the same plan).
* test_launches_have_rows records forward at every size above: the calls equal launch_plan, every launch has a row (the r3dp_sr_tc_conv
  ones IMG2PLANE_PRODUCTION of tests/test_gpu_sr_conv_conformance.py) and every row is launched.
* test_teacher_forced_forward runs forward at 512^2 (B = 1), 144^2 (B = 3) and 16^2 (B = 1) with make_params weights, one launch at a time:
  each launch's output against float64 of snapshots of the buffers and slices launch_plan says it reads, as earlier launches wrote them
  (not the pointers it was given), at the bars above; its weights against an independent float64 fold of the state_dict with the module's
  BatchNorm eps, rounded to fp16 (at most isolated 1-ulp ties, counted); its LayerNorm and dwconv parameters against the state_dict's own."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

import img2plane_reference as ref
import sr_conv_reference as scr
import test_gpu_img2plane_kernels as ikern
import test_gpu_secc2plane_kernels as skern
import test_gpu_sr_conv_conformance as srcc
from launch_harness import (GUARD, Recorder, assert_plan, assert_rows, at, bits, call_signature, conv3d, given, guarded, guards_intact, inside,
                            untouched)
from real3dportrait_b200 import _capi as capi
from real3dportrait_b200 import img2plane as ip
from real3dportrait_b200.img2plane import Img2PlaneModel

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
F16, F32, F64 = torch.float16, torch.float32, torch.float64
#: (H, B) of the standard-scale forwards the rows come from; RECORDED adds 64^2 at the other two scales
PLAN_SIZES = [(512, 4), (512, 1), (144, 3), (32, 3), (16, 1)]
RECORDED = [(H, B, 'standard') for H, B in PLAN_SIZES] + [(64, 1, 'small'), (64, 1, 'large')]
#: r3dp_mf_conv3d's beta per tap count (1: GEMMs on token / patch rows, 9: the (1,3,3) convs), about 2x the worst ratio over the rows on
#: an H100 80GB HBM3 (700 W power limit, max SM clock 1980 MHz): GEMMs 8.44e-7 (144^2 tri.block1.sr, K = 4096, fp32 out; fp16 out
#: 4.52e-7, layer4.0.conv2 at K = 4608), convs 5.23e-7 (512^2 B = 4 tri.final_conv, fp32 out; fp16 out 2.49e-7)
BETA = {1: 1.7e-6, 9: 1.1e-6}
P = capi.ptr


def _table():
    rows = {}
    for H, B, scale in RECORDED:
        for launch in ref.launch_plan(H, B, scale):
            rows.setdefault(ref.row_key(launch.fn, launch.args, launch.reads, launch.writes), (f'{H}-B{B}-{scale}-{launch.tag}', launch))
    return rows


ROWS = _table()


def _keys(fn):
    return [k for k in ROWS if k[0] == fn]


def _id(key):
    label, launch = ROWS[key]
    return label + '-' + 'x'.join(f'{v:g}' if isinstance(v, float) else str(v) for v in launch.args)


def _gen(key):
    return torch.Generator(device=DEV).manual_seed(list(ROWS).index(key) + 900)


# ---- r3dp_mf_conv3d ------------------------------------------------------------------------------------------------------------------------
@torch.no_grad()
@pytest.mark.parametrize('key', _keys('r3dp_mf_conv3d'), ids=_id)
def test_conv3d_launch(key):
    label, launch = ROWS[key]
    a = launch.args
    xs, _, cin, N, D, H, W, kd, kh, kw, _, O, cop, relu, ys, yc0, _, f32, _ = a
    has_res, xc0 = key[-2], key[-1]
    ci, k, s, p, d = launch.conv
    g = _gen(key)
    w = torch.randn(O, ci, k, k, generator=g, device=DEV, dtype=F64) / math.sqrt(ci * k * k)
    b64 = 0.1 * torch.randn(O, generator=g, device=DEV, dtype=F64)
    cv = ip._Conv(w, b64, k, s, p, d, DEV)
    wp, bias, _, cop_mod = cv.pk
    assert cop_mod == cop and wp.shape[-1] == cin, (label, cop_mod, tuple(wp.shape))       # the module packs the launch's K and cop
    ew, eb = _expected_packing(launch, w, b64)                  # tap / patch-row column order, zero padding: the packer against w itself
    assert torch.equal(wp.reshape(ew.shape), ew) and torch.equal(bias, eb), f'{label}: packed weights differ from w'
    box = kh == 3
    assert box == cv.box
    M = N * D * H * W
    x = torch.randn(N * D * H * W, xs, generator=g, device=DEV).half()
    r = torch.randn(M, O, generator=g, device=DEV).half() if has_res else None
    assert not has_res or ys == O
    dt = F32 if f32 else F16
    buf, y = guarded(M * ys, dt, tail=max(GUARD, (cop - O) * ys), device=DEV)
    conv3d(a, at(x, xc0), wp, bias, r, at(y))
    torch.cuda.synchronize()
    assert guards_intact(buf, M * ys), f'{label}: written past the output'
    yv = y.view(M, ys)
    mask = inside(ys, yc0, O, device=DEV)
    assert not bool(untouched(yv[:, mask]).any()), f'{label}: an output element was not written'
    assert bool(untouched(yv[:, ~mask]).all()), f'{label}: written outside the channel slice'
    alpha = scr.ALPHA_F32 if f32 else scr.ALPHA_F16
    extra = None if f32 else 2 * scr.FLOOR_F16
    bv = bias[:O].double()
    worst = 0.0
    if box:
        wv = wp.double().view(3, 3, cop, cin)[:, :, :O].permute(2, 3, 0, 1)
        for n in range(N):                                       # one image at a time bounds the float64 memory
            xi = x.view(N, H, W, xs)[n, :, :, xc0:xc0 + cin].double().permute(2, 0, 1)[None]
            want = F.conv2d(xi, wv, bv, 1, 1)[0].permute(1, 2, 0)
            S = F.conv2d(xi.abs(), wv.abs(), bv.abs(), 1, 1)[0].permute(1, 2, 0)
            if relu:
                want = want.clamp_min(0)
            if has_res:
                rn = r.view(N, H, W, O)[n].double()
                want, S = want + rn, S + rn.abs()
            got = yv[n * H * W:(n + 1) * H * W, yc0:yc0 + O].view(H, W, O)
            worst = max(worst, scr.check_bound(got, want, S, alpha, BETA[9], extra, tag=f'{label} image {n}'))
    else:
        wv = wp[:O].double()
        step = max(1, (1 << 25) // max(O, cin))
        for r0 in range(0, M, step):                             # row chunks bound the float64 memory
            xv = x[r0:r0 + step, xc0:xc0 + cin].double()
            want = xv @ wv.T + bv
            S = xv.abs() @ wv.abs().T + bv.abs()
            if relu:
                want = want.clamp_min(0)
            if has_res:
                rv = r[r0:r0 + step].double()
                want, S = want + rv, S + rv.abs()
            worst = max(worst, scr.check_bound(yv[r0:r0 + step, yc0:yc0 + O], want, S, alpha, BETA[1], extra, tag=f'{label} rows {r0}+'))
    print(f'conv3d {_id(key)}: worst excess / S = {worst:.3e} (beta {BETA[9 if box else 1]:.2e})')
    # bit-exact: the last image of a box conv equals its N = 1 launch, the last rows of a GEMM a launch on those rows alone
    if box and N > 1:
        ob, one = guarded(H * W * ys, dt, device=DEV)
        conv3d(a, at(x[(N - 1) * H * W:].contiguous(), xc0), wp, bias, None if r is None else r[(N - 1) * H * W:].contiguous(), at(one), N=1)
        torch.cuda.synchronize()
        assert torch.equal(bits(one.view(H * W, ys)[:, mask]), bits(yv[-H * W:, mask])), \
            f'{label}: the last image vs its N = 1 launch'
    elif not box:
        t = min(M, 300)
        ob, tail = guarded(t * ys, dt, device=DEV)
        conv3d(a, at(x[M - t:].contiguous(), xc0), wp, bias, None if r is None else r[M - t:].contiguous(), at(tail), N=1, H=t)
        torch.cuda.synchronize()
        assert torch.equal(bits(tail.view(t, ys)[:, mask]), bits(yv[-t:, mask])), \
            f'{label}: the last {t} rows vs a launch on them alone'


# ---- r3dp_sp_layernorm, r3dp_sp_dwconv_gelu, r3dp_sp_leaky -----------------------------------------------------------------------------
@torch.no_grad()
@pytest.mark.parametrize('key', _keys('r3dp_sp_layernorm'), ids=_id)
def test_layernorm_launch(key):
    label, launch = ROWS[key]
    R, C, eps, ldyh = launch.args
    roles, inplace = key[-2], key[-1]
    g = _gen(key)
    x0 = torch.randn(R, C, generator=g, device=DEV) * 2.0
    t = torch.randn(R, C, generator=g, device=DEV) * 0.5 if 't' in roles else None
    gam = 1 + 0.1 * torch.randn(C, generator=g, device=DEV)
    bet = 0.1 * torch.randn(C, generator=g, device=DEV)
    xbuf, x = guarded(R * C, F32, device=DEV)
    x.copy_(x0.view(-1))
    outs = {}
    for role, dt in (('xo', F32), ('yf', F32), ('yh', F16)):
        if role in roles and not (role == 'xo' and inplace):
            outs[role] = guarded(R * C, dt, device=DEV)
    xo = x if inplace else outs.get('xo', (None, None))[1]
    capi.check(capi.lib().r3dp_sp_layernorm(P(x), P(t), R, C, P(gam), P(bet), eps, P(xo), P(outs.get('yf', (None, None))[1]),
                                            P(outs.get('yh', (None, None))[1], F16), ldyh, capi.stream()))
    torch.cuda.synchronize()
    assert guards_intact(xbuf, R * C), f'{label}: written around x'
    v = x0.double() + (0.0 if t is None else t.double())
    want = F.layer_norm(v, (C,), gam.double(), bet.double(), eps)
    if 'xo' in roles:
        assert torch.equal(xo.view(R, C), x0 + t), f'{label}: the residual stream is not x + t in fp32'
    else:
        assert torch.equal(x.view(R, C), x0), f'{label}: x changed without an xo'
    for role, (buf, y) in outs.items():
        assert guards_intact(buf, R * C) and not bool(untouched(y).any()), f'{label} {role}: output not written exactly'
        if role != 'xo':
            skern.check_bar(f'sp_layernorm {label} {role}', y.view(R, C), want)


@torch.no_grad()
@pytest.mark.parametrize('key', _keys('r3dp_sp_dwconv_gelu'), ids=_id)
def test_dwconv_gelu_launch(key):
    label, launch = ROWS[key]
    B, h, w, C = launch.args
    g = _gen(key)
    x = torch.randn(B, h, w, C, generator=g, device=DEV).half()
    wt, b = 0.3 * torch.randn(C, 9, generator=g, device=DEV), 0.1 * torch.randn(C, generator=g, device=DEV)
    buf, y = guarded(B * h * w * C, F16, device=DEV)
    capi.check(capi.lib().r3dp_sp_dwconv_gelu(P(x, F16), B, h, w, C, P(wt), P(b), P(y, F16), capi.stream()))
    torch.cuda.synchronize()
    assert guards_intact(buf, y.numel()) and not bool(untouched(y).any()), f'{label}: output not written exactly'
    y = y.view(B, h, w, C)
    for n in range(B):
        want = F.gelu(F.conv2d(x[n:n + 1].double().permute(0, 3, 1, 2), wt.double().view(C, 1, 3, 3), b.double(), 1, 1, groups=C))
        skern.check_bar(f'sp_dwconv_gelu {label} image {n}', y[n], want[0].permute(1, 2, 0))


@torch.no_grad()
@pytest.mark.parametrize('key', _keys('r3dp_sp_leaky'), ids=_id)
def test_leaky_launch(key):
    label, launch = ROWS[key]
    n, slope = launch.args
    buf, y = guarded(n, F16, device=DEV)
    y.copy_(torch.randn(n, generator=_gen(key), device=DEV).half())
    want = F.leaky_relu(y.double(), slope)
    capi.check(capi.lib().r3dp_sp_leaky(P(y, F16), n, slope, capi.stream()))
    torch.cuda.synchronize()
    assert guards_intact(buf, n)
    if slope == 0.0:
        assert torch.equal(y.double(), want), f'{label}: ReLU is exact'
    skern.check_bar(f'sp_leaky {label}', y, want)


# ---- r3dp_ip_* -------------------------------------------------------------------------------------------------------------------------------
@torch.no_grad()
@pytest.mark.parametrize('key', _keys('r3dp_ip_attention'), ids=_id)
def test_attention_launch(key):
    """At the module's strides: q and o 1024 halves per token, kv 2048 (k | v)."""
    label, launch = ROWS[key]
    qs, kvs, B, Tq, Tk, heads, scale, os_ = launch.args
    C, hd = qs, qs // heads
    g = _gen(key)
    q = torch.randn(B * Tq, qs, generator=g, device=DEV).half()
    kv = torch.randn(B * Tk, kvs, generator=g, device=DEV).half()
    buf, o = guarded(B * Tq * os_, F16, device=DEV)
    capi.check(capi.lib().r3dp_ip_attention(P(q, F16), qs, P(kv, F16), kvs, B, Tq, Tk, heads, scale, P(o, F16), os_, capi.stream()))
    torch.cuda.synchronize()
    assert guards_intact(buf, o.numel()) and not bool(untouched(o).any()), f'{label}: output not written exactly'
    o, q, kv = o.view(B, Tq, os_), q.view(B, Tq, qs), kv.view(B, Tk, kvs)
    S = float(kv[..., C:].abs().max())
    for b in range(B):
        for hh in range(heads):
            cs = slice(hh * hd, (hh + 1) * hd)
            qh, kh = q[b, :, cs].double(), kv[b, :, cs].double()
            vh = kv[b, :, C + hh * hd:C + (hh + 1) * hd].double()
            want = ((qh @ kh.T) * scale).softmax(-1) @ vh
            ikern.check_bar(f'attention {label} b{b} h{hh}', o[b, :, cs], want, S)


@torch.no_grad()
@pytest.mark.parametrize('key', _keys('r3dp_ip_channel_mean'), ids=_id)
def test_channel_mean_launch(key):
    label, launch = ROWS[key]
    B, HW, C = launch.args
    x = torch.randn(B, HW, C, generator=_gen(key), device=DEV).half()
    buf, m = guarded(B * C, F16, device=DEV)
    capi.check(capi.lib().r3dp_ip_channel_mean(P(x, F16), B, HW, C, P(m, F16), capi.stream()))
    torch.cuda.synchronize()
    assert guards_intact(buf, m.numel())
    ikern.check_bar(f'mean {label}', m.view(B, C), x.double().mean(1))


@torch.no_grad()
@pytest.mark.parametrize('key', _keys('r3dp_ip_broadcast'), ids=_id)
def test_broadcast_launch(key):
    label, launch = ROWS[key]
    B, HW, Cb, ys, yc0 = launch.args
    v = torch.randn(B, Cb, generator=_gen(key), device=DEV).half()
    buf, y = guarded(B * HW * ys, F16, device=DEV)
    capi.check(capi.lib().r3dp_ip_broadcast(P(v, F16), B, HW, Cb, P(y, F16), ys, yc0, capi.stream()))
    torch.cuda.synchronize()
    assert guards_intact(buf, y.numel())
    y = y.view(B, HW, ys)
    assert torch.equal(y[..., yc0:yc0 + Cb], v[:, None].expand(B, HW, Cb)) and bool(untouched(y[..., :yc0]).all())


@torch.no_grad()
@pytest.mark.parametrize('key', _keys('r3dp_ip_pixel_shuffle'), ids=_id)
def test_pixel_shuffle_launch(key):
    label, launch = ROWS[key]
    B, h, w, C, ys, yc0 = launch.args
    g = _gen(key)
    x, t = torch.randn(B * h * w, 4 * C, generator=g, device=DEV), torch.randn(B * h * w, 4 * C, generator=g, device=DEV)
    buf, y = guarded(B * 4 * h * w * ys, F16, device=DEV)
    capi.check(capi.lib().r3dp_ip_pixel_shuffle(P(x), P(t), B, h, w, C, P(y, F16), ys, yc0, capi.stream()))
    torch.cuda.synchronize()
    assert guards_intact(buf, y.numel())
    y = y.view(B, 2 * h, 2 * w, ys)
    want = F.pixel_shuffle((x + t).view(B, h, w, 4 * C).permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1).half()
    assert torch.equal(y[..., yc0:yc0 + C], want), f'{label}: fp16(x + t), shuffled'
    assert bool(untouched(y[..., :yc0]).all()) and bool(untouched(y[..., yc0 + C:]).all()), f'{label}: written outside its slice'


@torch.no_grad()
@pytest.mark.parametrize('key', _keys('r3dp_ip_upsample2'), ids=_id)
def test_upsample2_launch(key):
    label, launch = ROWS[key]
    B, h, w, C = launch.args
    x = torch.randn(B, h, w, C, generator=_gen(key), device=DEV).half()
    buf, y = guarded(B * 4 * h * w * C, F16, device=DEV)
    capi.check(capi.lib().r3dp_ip_upsample2(P(x, F16), B, h, w, C, P(y, F16), capi.stream()))
    torch.cuda.synchronize()
    assert guards_intact(buf, y.numel()) and not bool(untouched(y).any())
    y = y.view(B, 2 * h, 2 * w, C)
    for n in range(B):
        want = F.interpolate(x[n:n + 1].permute(0, 3, 1, 2).double(), scale_factor=2.0, mode='bilinear', align_corners=True)
        ikern.check_bar(f'upsample2 {label} image {n}', y[n], want[0].permute(1, 2, 0))


@torch.no_grad()
@pytest.mark.parametrize('key', _keys('r3dp_ip_input') + _keys('r3dp_ip_maxpool') + _keys('r3dp_ip_flip_hwpc'), ids=_id)
def test_copy_launch(key):
    """The exact copies: input packing (rgb + the two coordinate channels + 3 zero pads, fp16), the 3x3/2 max-pool and the planes' flip."""
    label, launch = ROWS[key]
    fn, g = launch.fn, _gen(key)
    if fn == 'r3dp_ip_input':
        B, H, W = launch.args
        x = torch.rand(B, 3, H, W, generator=g, device=DEV) * 2 - 1
        buf, y = guarded(B * H * W * 8, F16, device=DEV)
        capi.check(capi.lib().r3dp_ip_input(P(x), B, H, W, P(y, F16), capi.stream()))
        want = ref.with_coords(x.double()).permute(0, 2, 3, 1)
        want = torch.cat([want, torch.zeros(B, H, W, 3, device=DEV, dtype=F64)], -1).half().reshape(-1)
    elif fn == 'r3dp_ip_maxpool':
        B, H, W, C = launch.args
        x = torch.randn(B, H, W, C, generator=g, device=DEV).half()
        ho, wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        buf, y = guarded(B * ho * wo * C, F16, device=DEV)
        capi.check(capi.lib().r3dp_ip_maxpool(P(x, F16), B, H, W, C, P(y, F16), capi.stream()))
        want = F.max_pool2d(x.permute(0, 3, 1, 2).float(), 3, 2, 1).permute(0, 2, 3, 1).half().reshape(-1)
    else:
        B, H, W = launch.args
        x = torch.randn(B, H, W, 96, generator=g, device=DEV)
        buf, y = guarded(B * H * W * 96, F32, device=DEV)
        capi.check(capi.lib().r3dp_ip_flip_hwpc(P(x), B, H, W, P(y), capi.stream()))
        want = ref.flip_planes(x.permute(0, 3, 1, 2)).permute(0, 3, 4, 1, 2).reshape(-1)
    torch.cuda.synchronize()
    assert guards_intact(buf, y.numel())
    assert torch.equal(y, want), f'{label}: not an exact copy'


# ---- the recorded launches -------------------------------------------------------------------------------------------------------------------
def _recorded(name):
    return name.startswith(('r3dp_ip_', 'r3dp_sp_')) or name in ('r3dp_mf_conv3d', 'r3dp_sr_tc_conv')


class _RowKeys(Recorder):
    """Records every r3dp_ip_*, r3dp_sp_*, r3dp_mf_conv3d and r3dp_sr_tc_conv call as its row key; capi.ptr is wrapped too, so an offset
    pointer (a channel slice of cat448) resolves to its tensor."""

    def __init__(self, lib):
        super().__init__(lib, _recorded, ptrs=True)

    def record(self, name, args):
        sig = call_signature(name, args)
        if name == 'r3dp_mf_conv3d':
            x = args[0].value                                   # its channel offset in the tensor it points into (fp16 elements)
            return sig + (given(args[6]), (x - self.tensor(x).data_ptr()) // 2 % args[1])
        if name == 'r3dp_sp_layernorm':
            roles = tuple(r for r, v in zip(('t', 'xo', 'yf', 'yh'), (args[1], args[7], args[8], args[9])) if given(v))
            return sig + (roles, given(args[7]) and args[7].value == args[0].value)
        return sig


@torch.no_grad()
def test_launches_have_rows():
    models = {}
    for scale in ('small', 'standard', 'large'):
        m = Img2PlaneModel(hp={'img2plane_backbone_scale': scale})
        m.load_state_dict(ref.make_params({k: v.shape for k, v in m.state_dict().items()}, 5), strict=True)
        models[scale] = m.to(DEV).eval()
        models[scale]._prepared()                                # the weight packing, not recorded
    launched, missing = set(), []
    sr_rows = {srcc.row_signature(row) for row in srcc.CASES}
    patch_rows = {(B, H, H, C, k, s, p, d, (k * k * C + 31) // 32 * 32) for B, H, C, k, s, p, d in ikern.PATCH_ROWS}
    with _RowKeys(capi.lib()) as rec:
        for H, B, scale in RECORDED:
            rec.clear()
            models[scale](ref.make_inputs(B, H, 11).to(DEV))
            got = rec.calls[:]
            assert_plan(got, [ref.row_key(launch.fn, launch.args, launch.reads, launch.writes) for launch in ref.launch_plan(H, B, scale)],
                        f'{H}^2 B={B} {scale}')
            for k in got:
                launched.add(k)
                if k[0] == 'r3dp_sr_tc_conv':
                    N, Nw, I, O, h, w, ksize, act = k[1]
                    ok = srcc.row_signature(('conv_res', N, Nw, I, O, h, w, {'ksize': ksize, 'act': act})) in sr_rows
                elif k[0] == 'r3dp_sp_patches_dil':
                    ok = k[1] in patch_rows
                else:
                    ok = k in ROWS
                if not ok:
                    missing.append(f'{H}^2 B={B} {scale}: {k}')
        torch.cuda.synchronize()
    print(f'{len(launched)} distinct launches over {len(RECORDED)} forwards')
    stale = [ROWS[k][0] for k in ROWS if k not in launched]
    stale += [f'IMG2PLANE_PRODUCTION {row}' for row in srcc.IMG2PLANE_PRODUCTION
              if ('r3dp_sr_tc_conv', (*row[1:7], row[7].get('ksize', 3), row[7]['act'])) not in launched]
    assert_rows(missing, stale, 'the forwards')


# ---- the teacher-forced forward ------------------------------------------------------------------------------------------------------------
#: the forwards replayed launch by launch: (H, B) at the standard scale
TEACHER = [(512, 1), (144, 3), (16, 1)]
#: plan tag prefix -> state_dict prefix
_SD = {'low': 'low_reso_vit', 'tri': 'triplane_predictor_vit', 'high': 'high_reso_encoder'}
_ENC, _ASPP = 'low_reso_encoder.encoder', 'low_reso_encoder.decoder.0'
#: the pointer argument each entry point writes through
_OUT = {'r3dp_ip_input': [4], 'r3dp_ip_maxpool': [5], 'r3dp_ip_channel_mean': [4], 'r3dp_ip_broadcast': [4], 'r3dp_ip_pixel_shuffle': [6],
        'r3dp_ip_upsample2': [5], 'r3dp_ip_flip_hwpc': [4], 'r3dp_ip_attention': [9], 'r3dp_sp_patches_dil': [9], 'r3dp_sp_dwconv_gelu': [7],
        'r3dp_sp_leaky': [0], 'r3dp_sp_layernorm': [7, 8, 9], 'r3dp_mf_conv3d': [18], 'r3dp_sr_tc_conv': [11]}
_LN_ROLES = {7: 'xo', 8: 'yf', 9: 'yh'}


def _sd_keys(tag):
    """Plan tag of a conv / linear / LayerNorm / dwconv launch -> (state_dict prefix, BatchNorm prefix or None)."""
    if tag == 'stem':
        return _ENC + '.conv1', _ENC + '.bn1'
    if tag.startswith('layer'):
        layer, blk, name = tag.split('.')
        p = f'{_ENC}.{layer}.{blk}'
        if name == 'downsample':
            return p + '.downsample.0', p + '.downsample.1'
        return f'{p}.{name}', f'{p}.bn{name[-1]}'
    if tag.startswith('aspp.'):
        i = tag.split('.')[1]
        return {'pool': _ASPP + '.convs.4.1', 'project': _ASPP + '.project.0'}.get(i, f'{_ASPP}.convs.{i}.0'), None
    if tag == 'decoder':
        return 'low_reso_encoder.decoder.1', None
    head, rest = tag.split('.', 1)
    p = _SD[head]
    if rest in ('pe', 'pe_norm'):
        return p + ('.patch_embed.proj' if rest == 'pe' else '.patch_embed.norm'), None
    if rest.startswith('block'):
        blk, name = rest.split('.')
        sub = {'q': 'attn.q', 'kv': 'attn.kv', 'proj': 'attn.proj', 'sr': 'attn.sr', 'sr_norm': 'attn.norm', 'fc1': 'mlp.fc1', 'fc2': 'mlp.fc2',
               'dwconv': 'mlp.dwconv.dwconv'}.get(name, name)
        return f'{p}.{blk}.{sub}', None
    return f'{p}.{rest}', None


def _fold(model, sd, tag):
    """Independent float64 fold of one conv / linear from the state_dict -> (W [O, I, k, k] or [O, K], bias [O]); BatchNorm's eps is the
    module's own BatchNorm2d eps."""
    p, bn = _sd_keys(tag)
    w = sd[p + '.weight']
    b = sd.get(p + '.bias')
    b = torch.zeros(w.shape[0], dtype=F64, device=DEV) if b is None else b
    if bn is not None:
        s = sd[bn + '.weight'] / torch.sqrt(sd[bn + '.running_var'] + model.get_submodule(bn).eps)
        b = sd[bn + '.bias'] - sd[bn + '.running_mean'] * s
        w = w * s.view(-1, *([1] * (w.ndim - 1)))
    return w, b


def _expected_packing(launch, w, b):
    """The fp16 weights and fp32 bias an r3dp_mf_conv3d / r3dp_sr_tc_conv launch must read, from the float64 fold: (1,3,3) taps [9, cop, I]
    (tap ky*3 + kx), GEMM rows [cop, K] (patch rows: column tap * C + c, C the input's channels, zero up to K), tc taps [9, O, I]."""
    O = w.shape[0]
    if launch.fn == 'r3dp_sr_tc_conv':
        return w.permute(2, 3, 0, 1).reshape(9, O, -1).half(), b.float()
    a = launch.args
    cop, K = a[12], a[2]
    if w.ndim == 2:
        rows = w
    elif a[8] == 3:
        wt = torch.zeros(9, cop, w.shape[1], dtype=F64, device=DEV)
        wt[:, :O] = w.permute(2, 3, 0, 1).reshape(9, O, -1)
        bb = torch.zeros(cop, dtype=F32, device=DEV)
        bb[:O] = b.float()
        return wt.half(), bb
    else:
        C = launch.conv[0]
        wc = torch.zeros(O, C, *w.shape[2:], dtype=F64, device=DEV)
        wc[:, :w.shape[1]] = w                                          # the stems' 5 input channels in the packed input's 8
        rows = wc.permute(0, 2, 3, 1).reshape(O, -1)
    wt = torch.zeros(cop, K, dtype=F64, device=DEV)
    wt[:O, :rows.shape[1]] = rows
    bb = torch.zeros(cop, dtype=F32, device=DEV)
    bb[:O] = b.float()
    return wt.half(), bb


def _same_bits(what, got, want, stats):
    """Equal, but for isolated 1-ulp ties of the fp16 / fp32 rounding of two float64 folds (counted)."""
    it = torch.int16 if got.dtype == F16 else torch.int32
    d = (got.reshape(-1).view(it).long() - want.reshape(-1).view(it).long()).abs()
    n = int((d != 0).sum())
    stats['ties'] += n
    stats['values'] += d.numel()
    assert int(d.max()) <= 1 and n <= max(2, d.numel() // 10000), f'{what}: {n} of {d.numel()} values differ from the fold (max {int(d.max())} ulp)'


class _TeacherForcer(_RowKeys):
    """Runs forward launch by launch against launch_plan: after each launch, the float64 reference of what it wrote is computed from the
    snapshots of the buffers the plan says it reads (earlier launches' outputs), not from the pointers it was given, and its weights are
    checked against the state_dict's fold."""

    def __init__(self, lib, plan, model, sd, x):
        super().__init__(lib)
        self.plan, self.model, self.sd, self.i = plan, model, sd, 0
        self.width = {}
        for launch in plan:
            for b, c0, c1 in list(launch.reads.values()) + list(launch.writes.values()):
                self.width[b] = max(self.width.get(b, 0), c1)
        self.store = {'img': x}
        self.stats = {'ties': 0, 'values': 0, 'launches': 0}

    def rd(self, launch, role):
        b, c0, c1 = launch.reads[role]
        return self.store[b][:, c0:c1]

    def __getattr__(self, name):
        fn = getattr(self.lib, name)
        if not _recorded(name):
            return fn

        def call(*args):
            assert self.i < len(self.plan), f'{name}: a launch past the plan'
            launch = self.plan[self.i]
            assert self.record(name, args) == ref.row_key(launch.fn, launch.args, launch.reads, launch.writes), f'launch {self.i}: {launch.tag}'
            rc = fn(*args)
            torch.cuda.synchronize()
            outs = {}
            for j in _OUT[name]:
                if args[j].value is not None:
                    t = self.tensor(args[j].value)
                    role = _LN_ROLES[j] if name == 'r3dp_sp_layernorm' else {'r3dp_sp_leaky': 'x', 'r3dp_ip_attention': 'o'}.get(name, 'y')
                    outs[role] = t.reshape(-1, self.width[launch.writes[role][0]])
            self.check(launch, args, outs)
            for role, t in outs.items():
                self.store[launch.writes[role][0]] = t.clone()
            self.i += 1
            self.stats['launches'] += 1
            return rc
        return call

    # float64 of each launch from the plan's operands
    def check(self, L, args, outs):
        fn, a, tag = L.fn, L.args, L.tag
        what = f'{tag} ({fn})'
        if fn == 'r3dp_ip_input':
            B, H, W = a
            want = ref.with_coords(self.store['img']).permute(0, 2, 3, 1)
            want = torch.cat([want, torch.zeros(B, H, W, 3, device=DEV)], -1).half().reshape(-1, 8)
            assert torch.equal(outs['y'], want), what
        elif fn == 'r3dp_sp_patches_dil':
            B, H, W, C, k, s, p, d, ldy = a
            x = self.rd(L, 'x').reshape(B, H, W, C).permute(0, 3, 1, 2).float()
            cols = F.unfold(x, k, dilation=d, padding=p, stride=s)
            cols = cols.view(B, C, k * k, -1).permute(0, 3, 2, 1).reshape(-1, k * k * C).half()
            assert torch.equal(outs['y'][:, :k * k * C], cols) and bool((outs['y'][:, k * k * C:] == 0).all()), what
        elif fn in ('r3dp_mf_conv3d', 'r3dp_sr_tc_conv'):
            self.check_conv(L, args, outs['y'], what)
        elif fn == 'r3dp_ip_maxpool':
            B, H, W, C = a
            x = self.rd(L, 'x').reshape(B, H, W, C).permute(0, 3, 1, 2).float()
            assert torch.equal(outs['y'], F.max_pool2d(x, 3, 2, 1).permute(0, 2, 3, 1).reshape(-1, C).half()), what
        elif fn == 'r3dp_ip_channel_mean':
            B, HW, C = a
            ikern.check_bar(f'mean {what}', outs['y'].reshape(B, C), self.rd(L, 'x').reshape(B, HW, C).double().mean(1))
        elif fn == 'r3dp_ip_broadcast':
            B, HW, C, ys, yc0 = a
            got = outs['y'].reshape(B, HW, ys)[..., yc0:yc0 + C]
            assert torch.equal(got, self.rd(L, 'x').reshape(B, 1, C).expand(B, HW, C)), what
        elif fn == 'r3dp_sp_layernorm':
            R, C, eps, _ = a
            p, _ = _sd_keys(tag)
            g, b = self.tensor(args[4].value), self.tensor(args[5].value)
            assert torch.equal(g, self.sd[p + '.weight'].float()) and torch.equal(b, self.sd[p + '.bias'].float()), f'{what}: not {p}'
            assert ctypes.c_float(eps).value == ctypes.c_float(self.model.get_submodule(p).eps).value, f'{what}: eps'
            x = self.rd(L, 'x')
            v = x.double()
            if 't' in L.reads:
                t = self.rd(L, 't')
                v = v + t.double()
            if 'xo' in outs:
                assert torch.equal(outs['xo'], x + t), f'{what}: the residual stream is not x + t in fp32'
            want = F.layer_norm(v, (C,), g.double(), b.double(), eps)
            for role in ('yf', 'yh'):
                if role in outs:
                    skern.check_bar(f'sp_layernorm {what} {role}', outs[role], want)
        elif fn == 'r3dp_ip_attention':
            qs, kvs, B, Tq, Tk, heads, scale, _ = a
            q, kv, o = self.rd(L, 'q').reshape(B, Tq, qs), self.rd(L, 'kv').reshape(B, Tk, kvs), outs['o'].reshape(B, Tq, -1)
            hd = qs // heads
            S = float(kv[..., qs:].abs().max())
            for bb in range(B):
                for h in range(heads):
                    cs = slice(h * hd, (h + 1) * hd)
                    want = ((q[bb, :, cs].double() @ kv[bb, :, cs].double().T) * scale).softmax(-1) @ kv[bb, :, qs + h * hd:qs + (h + 1) * hd].double()
                    ikern.check_bar(f'attention {what} b{bb} h{h}', o[bb, :, cs], want, S)
        elif fn == 'r3dp_sp_dwconv_gelu':
            B, h, w, C = a
            p, _ = _sd_keys(tag)
            wt, bt = self.tensor(args[5].value), self.tensor(args[6].value)
            assert torch.equal(wt.reshape(C, 9), self.sd[p + '.weight'].float().reshape(C, 9)) and torch.equal(bt, self.sd[p + '.bias'].float()), \
                f'{what}: not {p}'
            x = self.rd(L, 'x').reshape(B, h, w, C)
            y = outs['y'].reshape(B, h, w, C)
            for n in range(B):
                want = F.gelu(F.conv2d(x[n:n + 1].double().permute(0, 3, 1, 2), wt.double().view(C, 1, 3, 3), bt.double(), 1, 1, groups=C))
                skern.check_bar(f'sp_dwconv_gelu {what} image {n}', y[n], want[0].permute(1, 2, 0))
        elif fn == 'r3dp_sp_leaky':
            n, slope = a
            skern.check_bar(f'sp_leaky {what}', outs['x'], F.leaky_relu(self.rd(L, 'x').double(), slope))
        elif fn == 'r3dp_ip_pixel_shuffle':
            B, h, w, C, ys, yc0 = a
            v = (self.rd(L, 'x') + self.rd(L, 't')).reshape(B, h, w, 4 * C).permute(0, 3, 1, 2)
            want = F.pixel_shuffle(v, 2).permute(0, 2, 3, 1).half()
            assert torch.equal(outs['y'].reshape(B, 2 * h, 2 * w, ys)[..., yc0:yc0 + C], want), what
        elif fn == 'r3dp_ip_upsample2':
            B, h, w, C = a
            x = self.rd(L, 'x').reshape(B, h, w, C).permute(0, 3, 1, 2).double()
            want = F.interpolate(x, scale_factor=2.0, mode='bilinear', align_corners=True).permute(0, 2, 3, 1)
            ikern.check_bar(f'upsample2 {what}', outs['y'].reshape(B, 2 * h, 2 * w, C), want)
        elif fn == 'r3dp_ip_flip_hwpc':
            B, H, W = a
            x = self.rd(L, 'x').reshape(B, H, W, 96).permute(0, 3, 1, 2)
            assert torch.equal(outs['y'].reshape(-1), ref.flip_planes(x).permute(0, 3, 4, 1, 2).reshape(-1)), what
        else:
            raise AssertionError(f'{what}: no reference')

    def check_conv(self, L, args, y, what):
        a, tc = L.args, L.fn == 'r3dp_sr_tc_conv'
        wr, br = (self.tensor(args[1].value), self.tensor(args[2].value)) if tc else (self.tensor(args[4].value), self.tensor(args[5].value))
        w, b = _fold(self.model, self.sd, L.tag)
        ew, eb = _expected_packing(L, w, b)
        _same_bits(f'{what} weights', wr.reshape(ew.shape), ew, self.stats)
        _same_bits(f'{what} bias', br.reshape(-1)[:eb.numel()], eb, self.stats)
        x = self.rd(L, 'x')
        if tc:
            N, _, I, O, h, _, _, act = a
            wv = wr.reshape(9, O, I).double().permute(1, 2, 0).reshape(O, I, 3, 3)
            bv = br[:O].double()
            xi = x.reshape(N, h, h, I).double().permute(0, 3, 1, 2)
            for n in range(N):
                want = scr.bias_act(F.conv2d(xi[n:n + 1], wv, None, 1, 1), bv, act)
                S = scr.act_gain(act) * (F.conv2d(xi[n:n + 1].abs(), wv.abs(), None, 1, 1) + bv.abs().view(1, -1, 1, 1))
                got = y.reshape(N, h, h, O)[n:n + 1].double().permute(0, 3, 1, 2)
                scr.check_bound(got, want, S, scr.ALPHA_F16, scr.BETA['tc'], scr.FLOOR_F16, tag=f'{what} image {n}')
            return
        xs, _, cin, N, D, H, W, kd, kh, kw, _, O, cop, relu, ys, yc0, _, f32, _ = a
        alpha, extra = (scr.ALPHA_F32, None) if f32 else (scr.ALPHA_F16, 2 * scr.FLOOR_F16)
        res = self.rd(L, 'res') if 'res' in L.reads else None
        got = y[:, yc0:yc0 + O]
        bv = br[:O].double()
        if kh == 3:
            wv = wr.reshape(3, 3, cop, cin)[:, :, :O].double().permute(2, 3, 0, 1)
            xi = x.reshape(N, H, W, cin)
            for n in range(N):
                xn = xi[n].double().permute(2, 0, 1)[None]
                want = F.conv2d(xn, wv, bv, 1, 1)[0].permute(1, 2, 0)
                S = F.conv2d(xn.abs(), wv.abs(), bv.abs(), 1, 1)[0].permute(1, 2, 0)
                if relu:
                    want = want.clamp_min(0)
                if res is not None:
                    rn = res.reshape(N, H, W, O)[n].double()
                    want, S = want + rn, S + rn.abs()
                scr.check_bound(got.reshape(N, H, W, O)[n], want, S, alpha, BETA[9], extra, tag=f'{what} image {n}')
        else:
            wv = wr.reshape(cop, cin)[:O].double()
            xv = x.double()
            want, S = xv @ wv.T + bv, xv.abs() @ wv.abs().T + bv.abs()
            if relu:
                want = want.clamp_min(0)
            if res is not None:
                want, S = want + res.double(), S + res.double().abs()
            scr.check_bound(got, want, S, alpha, BETA[1], extra, tag=what)


@torch.no_grad()
@pytest.mark.parametrize('H,B', TEACHER, ids=lambda v: str(v))
def test_teacher_forced_forward(H, B):
    """forward with make_params weights, each launch checked against float64 of the buffers launch_plan says it reads, as the earlier
    launches wrote them: a launch that reads the wrong buffer or slice, or races with its own in-place write, fails, as does a weight
    that is not the state_dict's (the wrong block's LayerNorm, a fold with another BatchNorm eps)."""
    m = Img2PlaneModel()
    sd = ref.make_params({k: v.shape for k, v in m.state_dict().items()}, 5)
    m.load_state_dict(sd, strict=True)
    m = m.to(DEV).eval()
    m._prepared()
    sd = {k: (v.to(DEV, F64) if v.is_floating_point() else v.to(DEV)) for k, v in sd.items()}
    x = ref.make_inputs(B, H, 11).to(DEV)
    with _TeacherForcer(capi.lib(), ref.launch_plan(H, B), m, sd, x) as tf:
        out = m(x)
        torch.cuda.synchronize()
    assert tf.i == len(tf.plan), f'{tf.i} of {len(tf.plan)} launches'
    assert torch.equal(out.permute(0, 3, 4, 1, 2).reshape(-1), tf.store['planes'].reshape(-1))
    print(f'teacher-forced {H}^2 B={B}: {tf.stats["launches"]} launches; weights: {tf.stats["ties"]} of {tf.stats["values"]} values 1 ulp '
          'from the fold')
