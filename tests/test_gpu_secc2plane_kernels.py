"""Every r3dp_sp_* entry point at the shapes of a 512^2 SegFormerSECC2PlaneBackbone('b0') call, B = 1 and 4, and at every launch of
`forward` at H = 32, 96, 224 and 480 (B = 1 and 3; the *_sizes tests, rows from secc2plane_reference.launch_plan), against float64 computed
on the device from the very operands the kernel reads.  The *_sizes tests also fill every output with a sentinel between guard runs: every
element must be written and nothing past it.  Bar (the form of test_gpu_sr_conv_conformance.py):

    |got - ref| <= ALPHA * |ref| + beta * S,   S = max |ref|

ALPHA is the rounding of the stored type (2^-11 for fp16 outputs, 2^-23 for fp32); beta is the measured arithmetic error of the kernel
(accumulation order, expf / erff / rsqrtf), one bar per kernel asserted with margin (BETA) and recorded in DESIGN.md.  A wrong tap, offset,
mirror or an unwritten tail costs O(S)."""
import math

import pytest
import torch
import torch.nn.functional as F

from real3dportrait_b200 import _capi as capi
import secc2plane_reference as sref
from launch_harness import GUARD, guarded, guards_intact, untouched

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
F16, F32, F64 = torch.float16, torch.float32, torch.float64
ALPHA = {F16: 2.0 ** -11, F32: 2.0 ** -23}
#: per kernel: about 2x the worst beta measured over every row of this file on an H100 80GB HBM3 (700 W power limit), DESIGN.md.  Worst
#: rows: upsample2_flip 7.9e-6 (rows+cols, 480^2 B = 3: the fp32 interpolation weights of h = 120), embed 7.6e-7, attention 1.8e-7
#: (480^2 stage 2, Tk = 225), layernorm 9.4e-8, prenet 8.7e-8, head_fuse 3.2e-8, dwconv_gelu 2.4e-8, leaky 6.7e-9
BETA = {'sp_upsample2_flip': 2e-5, 'sp_embed': 1.5e-6, 'sp_attention': 4e-7, 'sp_layernorm': 2e-7, 'sp_prenet': 2e-7, 'sp_head_fuse': 7e-8,
        'sp_dwconv_gelu': 5e-8, 'sp_leaky': 1.5e-8}
L = None


def lib():
    global L
    L = L or capi.lib()
    return L


def _beta(got, ref):
    ref = ref.to(F64)
    S = float(ref.abs().max())
    excess = (got.to(F64) - ref).abs() - ALPHA[got.dtype] * ref.abs()
    return max(float(excess.max()), 0.0) / S


def check_bar(name, got, ref):
    b = _beta(got, ref)
    bar = BETA[name.split()[0]]
    print(f'{name}: beta = {b:.2e} (bar {bar:.1e})')
    assert b <= bar, (name, b, bar)


def _g(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _rand(shape, seed, dtype=F32, scale=1.0):
    return (torch.randn(shape, generator=_g(seed), device=DEV) * scale).to(dtype).contiguous()


P = capi.ptr


@pytest.mark.parametrize('B', [1, 4])
def test_prenet_and_embed(B):
    H = 512
    cano_src = _rand((1, 6, H, H), 1)
    tgt = _rand((B, 3, H, H), 2)
    w = _rand((3, 9), 3, scale=0.3)
    b = _rand((3,), 4)
    wpe, bpe = _rand((32, 3, 7, 7), 5, scale=0.1), _rand((32,), 6)
    st = capi.stream()
    base = torch.empty(1, 3, H, H, device=DEV)
    capi.check(lib().r3dp_sp_prenet(P(cano_src), 1, 6, H, H, P(w[:, :6].contiguous()), P(b), P(base), st))
    ref_base = torch.einsum('cj,njhw->nchw', w[:, :6].double(), cano_src.double()) + b.double()[None, :, None, None]
    check_bar('sp_prenet', base, ref_base)
    # per-frame embed on the cached image (the operands it reads: base, tgt, w[:, 6:])
    y = torch.empty(B, (H // 4) ** 2, 32, device=DEV)
    capi.check(lib().r3dp_sp_embed(P(tgt), B, 3, H, H, P(w[:, 6:].contiguous()), P(base), None, P(wpe), P(bpe), P(y), st))
    pre = base.double() + torch.einsum('cj,njhw->nchw', w[:, 6:].double(), tgt.double())
    ref = F.conv2d(pre, wpe.double(), bpe.double(), 4, 3).flatten(2).transpose(1, 2)
    check_bar('sp_embed (cached image)', y, ref)
    # the whole 9-channel input, no cached image
    x = torch.cat([cano_src.expand(B, -1, -1, -1), tgt], 1).contiguous()
    capi.check(lib().r3dp_sp_embed(P(x), B, 9, H, H, P(w), None, P(b), P(wpe), P(bpe), P(y), st))
    pre = torch.einsum('cj,njhw->nchw', w.double(), x.double()) + b.double()[None, :, None, None]
    check_bar('sp_embed (full input)', y, F.conv2d(pre, wpe.double(), bpe.double(), 4, 3).flatten(2).transpose(1, 2))


@pytest.mark.parametrize('B', [1, 4])
@pytest.mark.parametrize('C,hw', [(32, 128), (64, 64), (160, 32), (256, 16)])
def test_layernorm(B, C, hw):
    R = B * hw * hw
    x, t = _rand((R, C), 10, scale=2.0), _rand((R, C), 11)
    g, b = 1 + _rand((C,), 12, scale=0.2), _rand((C,), 13, scale=0.1)
    xo, yf, yh = torch.empty_like(x), torch.empty_like(x), torch.empty(R, C, device=DEV, dtype=F16)
    capi.check(lib().r3dp_sp_layernorm(P(x), P(t), R, C, P(g), P(b), 1e-6, P(xo), P(yf), P(yh, F16), C, capi.stream()))
    v = x.double() + t.double()
    ref = F.layer_norm(v, (C,), g.double(), b.double(), 1e-6)
    check_bar(f'sp_layernorm residual C={C}', xo, v)
    check_bar(f'sp_layernorm fp32 C={C}', yf, ref)
    check_bar(f'sp_layernorm fp16 C={C}', yh, ref)


@pytest.mark.parametrize('B', [1, 4])
@pytest.mark.parametrize('hw,C,k,s,p', [(128, 32, 8, 8, 0), (64, 64, 4, 4, 0), (32, 160, 2, 2, 0), (128, 32, 3, 2, 1), (64, 64, 3, 2, 1),
                                        (32, 160, 3, 2, 1)])
def test_patches(B, hw, C, k, s, p):
    x = _rand((B, hw, hw, C), 20, F16)
    ho = (hw + 2 * p - k) // s + 1
    y = torch.empty(B * ho * ho, k * k * C, device=DEV, dtype=F16)
    capi.check(lib().r3dp_sp_patches(P(x, F16), B, hw, hw, C, k, s, p, P(y, F16), capi.stream()))
    cols = F.unfold(x.permute(0, 3, 1, 2).float(), k, padding=p, stride=s)              # [B, C*k*k, L], column c*k*k + tap
    ref = cols.view(B, C, k * k, -1).permute(0, 3, 2, 1).reshape(B * ho * ho, k * k * C)
    assert torch.equal(y.float(), ref)


@pytest.mark.parametrize('B', [1, 4])
@pytest.mark.parametrize('hw,heads,tk', [(128, 1, 256), (64, 2, 256), (32, 5, 256), (16, 8, 256)])
def test_attention(B, hw, heads, tk):
    C, T = heads * 32, hw * hw
    q = _rand((B, T, C), 30, F16)
    kv = _rand((B, tk, 2 * C), 31, F16, scale=1.5)
    o = torch.empty(B, T, C, device=DEV, dtype=F16)
    capi.check(lib().r3dp_sp_attention(P(q, F16), C, P(kv, F16), 2 * C, B, T, tk, heads, 32 ** -0.5, P(o, F16), C, capi.stream()))
    qh = q.double().view(B, T, heads, 32).transpose(1, 2)
    kh = kv.double()[..., :C].view(B, tk, heads, 32).transpose(1, 2)
    vh = kv.double()[..., C:].view(B, tk, heads, 32).transpose(1, 2)
    ref = ((qh @ kh.transpose(-2, -1)) * 32 ** -0.5).softmax(-1) @ vh
    check_bar(f'sp_attention heads={heads}', o, ref.transpose(1, 2).reshape(B, T, C))


@pytest.mark.parametrize('B', [1, 4])
@pytest.mark.parametrize('hw,C', [(128, 128), (64, 256), (32, 640), (16, 1024)])
def test_dwconv_gelu(B, hw, C):
    x = _rand((B, hw, hw, C), 40, F16)
    w, b = _rand((C, 9), 41, scale=0.3), _rand((C,), 42, scale=0.1)
    y = torch.empty_like(x)
    capi.check(lib().r3dp_sp_dwconv_gelu(P(x, F16), B, hw, hw, C, P(w), P(b), P(y, F16), capi.stream()))
    ref = F.gelu(F.conv2d(x.double().permute(0, 3, 1, 2), w.double().view(C, 1, 3, 3), b.double(), 1, 1, groups=C)).permute(0, 2, 3, 1)
    check_bar(f'sp_dwconv_gelu C={C}', y, ref)


@pytest.mark.parametrize('B', [1, 4])
def test_head_fuse(B):
    sizes = (128, 64, 32, 16)
    g = [_rand((B, h, h, 256), 50 + i) for i, h in enumerate(sizes)]
    bias = _rand((256,), 55)
    y = torch.empty(B, 128, 128, 256, device=DEV, dtype=F16)
    capi.check(lib().r3dp_sp_head_fuse(P(g[0]), 128, P(g[1]), 64, P(g[2]), 32, P(g[3]), 16, B, P(bias), P(y, F16), capi.stream()))
    acc = bias.double()[None, :, None, None] + g[0].double().permute(0, 3, 1, 2)
    for t in g[1:]:
        acc = acc + F.interpolate(t.double().permute(0, 3, 1, 2), size=(128, 128), mode='bilinear', align_corners=False)
    check_bar('sp_head_fuse', y, torch.relu(acc).permute(0, 2, 3, 1))


@pytest.mark.parametrize('B', [1, 4])
def test_leaky(B):
    x = _rand((B, 128, 128, 256), 60, F16)
    ref = F.leaky_relu(x.double(), 0.01)
    capi.check(lib().r3dp_sp_leaky(P(x, F16), x.numel(), 0.01, capi.stream()))
    check_bar('sp_leaky', x, ref)


@pytest.mark.parametrize('B', [1, 4])
def test_upsample2_flip(B):
    x = _rand((B, 128, 128, 256), 70, F16)
    yr, yrc = torch.empty(B, 256, 256, 256, device=DEV, dtype=F16), torch.empty(B, 256, 256, 256, device=DEV, dtype=F16)
    capi.check(lib().r3dp_sp_upsample2_flip(P(x, F16), B, 128, 128, 256, P(yr, F16), P(yrc, F16), capi.stream()))
    up = F.interpolate(x.double().permute(0, 3, 1, 2), scale_factor=2.0, mode='bilinear', align_corners=True).permute(0, 2, 3, 1)
    check_bar('sp_upsample2_flip rows', yr, up.flip(1))
    check_bar('sp_upsample2_flip rows+cols', yrc, up.flip(1, 2))


# ---- every size class the module accepts ---------------------------------------------------------------------------------------------------
#: (H, B) of the launch tables below: 512^2 at B = 1 and 4, and H = 32, 96, 224, 480 at B = 1 and 3.  Below 512^2 the query counts leave a
#: partial 128-query tile (576, 3136, 14400), the attentions see Tk = 1, 9, 49 or 225 keys, LayerNorm row counts are not multiples of its
#: 8 rows per block, and the head fuses levels down to 1 x 1.
SP_SIZES = [(512, 1), (512, 4)] + [(H, B) for H in (32, 96, 224, 480) for B in (1, 3)]


def _sp_table():
    """{(entry point, non-pointer arguments): (H, B, tag)} of every distinct r3dp_sp_* launch of forward over SP_SIZES."""
    rows = {}
    for H, B in SP_SIZES:
        for tag, fn, a in sref.launch_plan(H, B):
            if fn.startswith('r3dp_sp_'):
                rows.setdefault(sref.launch_signature(fn, a), (H, B, tag))
    return rows


SP = _sp_table()


def sp_signatures():
    return set(SP)


def sp_rows_at(H):
    """[(entry point, arguments, (H, B))] of the rows first launched at size H."""
    return [(fn, a, v[:2]) for (fn, a), v in SP.items() if v[0] == H]


def _keys(fn):
    return [k for k in SP if k[0] == fn]


def _kid(k):
    H, B, tag = SP[k]
    return f'{H}-B{B}-{tag}-' + 'x'.join(f'{v:g}' if isinstance(v, float) else str(v) for v in k[1])


def _guarded(shape, dtype):
    """(output view of `shape`, whole guarded buffer)."""
    buf, y = guarded(math.prod(shape), dtype, device=DEV)
    return y.view(shape), buf


def _written(name, buf):
    y = buf[GUARD:-GUARD]
    assert guards_intact(buf, y.numel()), f'{name}: written outside the output'
    assert not bool(untouched(y).any()), f'{name}: output elements left unwritten'


@pytest.mark.parametrize('key', _keys('r3dp_sp_attention'), ids=_kid)
def test_attention_sizes(key):
    C, _, B, T, tk, heads, scale, _ = key[1]
    q = _rand((B, T, C), 130 + tk, F16)
    kv = _rand((B, tk, 2 * C), 131 + tk, F16, scale=1.5)
    o, buf = _guarded((B, T, C), F16)
    capi.check(lib().r3dp_sp_attention(P(q, F16), C, P(kv, F16), 2 * C, B, T, tk, heads, 32 ** -0.5, P(o, F16), C, capi.stream()))
    torch.cuda.synchronize()
    _written(_kid(key), buf)
    qh = q.double().view(B, T, heads, 32).transpose(1, 2)
    kh = kv.double()[..., :C].view(B, tk, heads, 32).transpose(1, 2)
    vh = kv.double()[..., C:].view(B, tk, heads, 32).transpose(1, 2)
    ref = ((qh @ kh.transpose(-2, -1)) * 32 ** -0.5).softmax(-1) @ vh
    check_bar(f'sp_attention {_kid(key)}', o, ref.transpose(1, 2).reshape(B, T, C))


@pytest.mark.parametrize('key', _keys('r3dp_sp_layernorm'), ids=_kid)
def test_layernorm_sizes(key):
    R, C, eps, _ = key[1]
    x, t = _rand((R, C), 140 + R % 97, scale=2.0), _rand((R, C), 141)
    g, b = 1 + _rand((C,), 142, scale=0.2), _rand((C,), 143, scale=0.1)
    (xo, bxo), (yf, byf), (yh, byh) = _guarded((R, C), F32), _guarded((R, C), F32), _guarded((R, C), F16)
    capi.check(lib().r3dp_sp_layernorm(P(x), P(t), R, C, P(g), P(b), eps, P(xo), P(yf), P(yh, F16), C, capi.stream()))
    torch.cuda.synchronize()
    for name, buf in (('xo', bxo), ('yf', byf), ('yh', byh)):
        _written(f'{_kid(key)} {name}', buf)
    v = x.double() + t.double()
    ref = F.layer_norm(v, (C,), g.double(), b.double(), eps)
    check_bar(f'sp_layernorm residual {_kid(key)}', xo, v)
    check_bar(f'sp_layernorm fp32 {_kid(key)}', yf, ref)
    check_bar(f'sp_layernorm fp16 {_kid(key)}', yh, ref)


@pytest.mark.parametrize('key', _keys('r3dp_sp_dwconv_gelu'), ids=_kid)
def test_dwconv_gelu_sizes(key):
    B, hw, _, C = key[1]
    x = _rand((B, hw, hw, C), 150 + hw, F16)
    w, b = _rand((C, 9), 151, scale=0.3), _rand((C,), 152, scale=0.1)
    y, buf = _guarded((B, hw, hw, C), F16)
    capi.check(lib().r3dp_sp_dwconv_gelu(P(x, F16), B, hw, hw, C, P(w), P(b), P(y, F16), capi.stream()))
    torch.cuda.synchronize()
    _written(_kid(key), buf)
    ref = F.gelu(F.conv2d(x.double().permute(0, 3, 1, 2), w.double().view(C, 1, 3, 3), b.double(), 1, 1, groups=C)).permute(0, 2, 3, 1)
    check_bar(f'sp_dwconv_gelu {_kid(key)}', y, ref)


@pytest.mark.parametrize('key', _keys('r3dp_sp_head_fuse'), ids=_kid)
def test_head_fuse_sizes(key):
    *sizes, B = key[1]
    h1 = sizes[0]
    g = [_rand((B, h, h, 256), 160 + i) for i, h in enumerate(sizes)]
    bias = _rand((256,), 165)
    y, buf = _guarded((B, h1, h1, 256), F16)
    capi.check(lib().r3dp_sp_head_fuse(P(g[0]), sizes[0], P(g[1]), sizes[1], P(g[2]), sizes[2], P(g[3]), sizes[3], B, P(bias), P(y, F16),
                                       capi.stream()))
    torch.cuda.synchronize()
    _written(_kid(key), buf)
    acc = bias.double()[None, :, None, None] + g[0].double().permute(0, 3, 1, 2)
    for t in g[1:]:
        acc = acc + F.interpolate(t.double().permute(0, 3, 1, 2), size=(h1, h1), mode='bilinear', align_corners=False)
    check_bar(f'sp_head_fuse {_kid(key)}', y, torch.relu(acc).permute(0, 2, 3, 1))


@pytest.mark.parametrize('key', _keys('r3dp_sp_upsample2_flip'), ids=_kid)
def test_upsample2_flip_sizes(key):
    B, h, _, C = key[1]
    x = _rand((B, h, h, C), 170 + h, F16)
    (yr, br), (yrc, brc) = _guarded((B, 2 * h, 2 * h, C), F16), _guarded((B, 2 * h, 2 * h, C), F16)
    capi.check(lib().r3dp_sp_upsample2_flip(P(x, F16), B, h, h, C, P(yr, F16), P(yrc, F16), capi.stream()))
    torch.cuda.synchronize()
    _written(f'{_kid(key)} rows', br)
    _written(f'{_kid(key)} rows+cols', brc)
    up = F.interpolate(x.double().permute(0, 3, 1, 2), scale_factor=2.0, mode='bilinear', align_corners=True).permute(0, 2, 3, 1)
    check_bar(f'sp_upsample2_flip rows {_kid(key)}', yr, up.flip(1))
    check_bar(f'sp_upsample2_flip rows+cols {_kid(key)}', yrc, up.flip(1, 2))


@pytest.mark.parametrize('key', _keys('r3dp_sp_leaky'), ids=_kid)
def test_leaky_sizes(key):
    n, slope = key[1]
    y, buf = _guarded((n,), F16)
    y.copy_(_rand((n,), 180, F16))
    ref = F.leaky_relu(y.double(), slope)
    capi.check(lib().r3dp_sp_leaky(P(y, F16), n, slope, capi.stream()))
    torch.cuda.synchronize()
    _written(_kid(key), buf)
    check_bar(f'sp_leaky {_kid(key)}', y, ref)


@pytest.mark.parametrize('key', _keys('r3dp_sp_embed'), ids=_kid)
def test_embed_sizes(key):
    """The forward's 9-channel launch, and the 3-channel launch on the clip's cached image (planes_cl) at the same size."""
    B, cin, H, _ = key[1]
    x = _rand((B, cin, H, H), 190 + H)
    w, b = _rand((3, cin), 191, scale=0.3), _rand((3,), 192)
    wpe, bpe = _rand((32, 3, 7, 7), 193, scale=0.1), _rand((32,), 194)
    base = _rand((1, 3, H, H), 195)
    st, ho = capi.stream(), (H - 1) // 4 + 1
    y, buf = _guarded((B, ho * ho, 32), F32)
    capi.check(lib().r3dp_sp_embed(P(x), B, cin, H, H, P(w), None, P(b), P(wpe), P(bpe), P(y), st))
    torch.cuda.synchronize()
    _written(f'{_kid(key)} full input', buf)
    pre = torch.einsum('cj,njhw->nchw', w.double(), x.double()) + b.double()[None, :, None, None]
    check_bar(f'sp_embed (full input) {_kid(key)}', y, F.conv2d(pre, wpe.double(), bpe.double(), 4, 3).flatten(2).transpose(1, 2))
    y, buf = _guarded((B, ho * ho, 32), F32)
    tgt = x[:, -3:].contiguous()
    wt = w[:, -3:].contiguous()
    capi.check(lib().r3dp_sp_embed(P(tgt), B, 3, H, H, P(wt), P(base), None, P(wpe), P(bpe), P(y), st))
    torch.cuda.synchronize()
    _written(f'{_kid(key)} cached image', buf)
    pre = base.double() + torch.einsum('cj,njhw->nchw', wt.double(), tgt.double())
    check_bar(f'sp_embed (cached image) {_kid(key)}', y, F.conv2d(pre, wpe.double(), bpe.double(), 4, 3).flatten(2).transpose(1, 2))


@pytest.mark.parametrize('key', _keys('r3dp_sp_patches'), ids=_kid)
def test_patches_sizes(key):
    B, hw, _, C, k, s, p = key[1]
    x = _rand((B, hw, hw, C), 200 + hw, F16)
    ho = (hw + 2 * p - k) // s + 1
    y, buf = _guarded((B * ho * ho, k * k * C), F16)
    capi.check(lib().r3dp_sp_patches(P(x, F16), B, hw, hw, C, k, s, p, P(y, F16), capi.stream()))
    torch.cuda.synchronize()
    _written(_kid(key), buf)
    cols = F.unfold(x.permute(0, 3, 1, 2).float(), k, padding=p, stride=s)
    ref = cols.view(B, C, k * k, -1).permute(0, 3, 2, 1).reshape(B * ho * ho, k * k * C)
    assert torch.equal(y.float(), ref)


# ---- a second device ------------------------------------------------------------------------------------------------------------------------
def test_attention_on_second_device():
    """The stage-1 attention (Tk = 256 keys: 64 KB of dynamic shared memory, over the 48 KB default) on cuda:1 after cuda:0 in one process.
    The shared-memory limit is an attribute of the current device's function, so the launcher has to set it on every device it runs on."""
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two visible CUDA devices')
    B, T, tk, heads, C = 1, 128 * 128, 256, 1, 32
    outs = []
    for dev in ('cuda:0', 'cuda:1'):
        with torch.cuda.device(dev):
            g = torch.Generator().manual_seed(210)
            q = torch.randn(B, T, C, generator=g).half().to(dev)
            kv = (1.5 * torch.randn(B, tk, 2 * C, generator=g)).half().to(dev)
            o = torch.empty(B, T, C, device=dev, dtype=F16)
            capi.check(lib().r3dp_sp_attention(P(q, F16), C, P(kv, F16), 2 * C, B, T, tk, heads, 32 ** -0.5, P(o, F16), C, capi.stream()))
            torch.cuda.synchronize()
            qh, kh, vh = q.double(), kv.double()[..., :C], kv.double()[..., C:]
            ref = ((qh @ kh.transpose(-2, -1)) * 32 ** -0.5).softmax(-1) @ vh
            check_bar(f'sp_attention on {dev}', o, ref)
            outs.append(o.cpu())
    assert torch.equal(outs[0], outs[1])
