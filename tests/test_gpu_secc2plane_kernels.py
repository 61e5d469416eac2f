"""Every r3dp_sp_* entry point at the shapes of a 512^2 SegFormerSECC2PlaneBackbone('b0') call, B = 1 and 4, against float64 computed on the
device from the very operands the kernel reads.  Bar (the form of test_gpu_sr_conv_conformance.py):

    |got - ref| <= ALPHA * |ref| + beta * S,   S = max |ref|

ALPHA is the rounding of the stored type (2^-11 for fp16 outputs, 2^-23 for fp32); beta is the measured arithmetic error of the kernel
(accumulation order, expf / erff / rsqrtf), asserted with margin and recorded in DESIGN.md.  A wrong tap, offset or mirror costs O(S)."""
import pytest
import torch
import torch.nn.functional as F

from real3dportrait_b200 import _capi as capi

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
F16, F32, F64 = torch.float16, torch.float32, torch.float64
ALPHA = {F16: 2.0 ** -11, F32: 2.0 ** -23}
BETA = 1e-5          # measured on an H100: at most 3.8e-6 (sp_upsample2_flip), 6.2e-7 (sp_embed), 1.4e-7 or less elsewhere (DESIGN.md)
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


def _check(name, got, ref):
    b = _beta(got, ref)
    print(f'{name}: beta = {b:.2e}')
    assert b <= BETA, (name, b)


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
    _check('sp_prenet', base, ref_base)
    # per-frame embed on the cached image (the operands it reads: base, tgt, w[:, 6:])
    y = torch.empty(B, (H // 4) ** 2, 32, device=DEV)
    capi.check(lib().r3dp_sp_embed(P(tgt), B, 3, H, H, P(w[:, 6:].contiguous()), P(base), None, P(wpe), P(bpe), P(y), st))
    pre = base.double() + torch.einsum('cj,njhw->nchw', w[:, 6:].double(), tgt.double())
    ref = F.conv2d(pre, wpe.double(), bpe.double(), 4, 3).flatten(2).transpose(1, 2)
    _check('sp_embed (cached image)', y, ref)
    # the whole 9-channel input, no cached image
    x = torch.cat([cano_src.expand(B, -1, -1, -1), tgt], 1).contiguous()
    capi.check(lib().r3dp_sp_embed(P(x), B, 9, H, H, P(w), None, P(b), P(wpe), P(bpe), P(y), st))
    pre = torch.einsum('cj,njhw->nchw', w.double(), x.double()) + b.double()[None, :, None, None]
    _check('sp_embed (full input)', y, F.conv2d(pre, wpe.double(), bpe.double(), 4, 3).flatten(2).transpose(1, 2))


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
    _check(f'sp_layernorm residual C={C}', xo, v)
    _check(f'sp_layernorm fp32 C={C}', yf, ref)
    _check(f'sp_layernorm fp16 C={C}', yh, ref)


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
    _check(f'sp_attention heads={heads}', o, ref.transpose(1, 2).reshape(B, T, C))


@pytest.mark.parametrize('B', [1, 4])
@pytest.mark.parametrize('hw,C', [(128, 128), (64, 256), (32, 640), (16, 1024)])
def test_dwconv_gelu(B, hw, C):
    x = _rand((B, hw, hw, C), 40, F16)
    w, b = _rand((C, 9), 41, scale=0.3), _rand((C,), 42, scale=0.1)
    y = torch.empty_like(x)
    capi.check(lib().r3dp_sp_dwconv_gelu(P(x, F16), B, hw, hw, C, P(w), P(b), P(y, F16), capi.stream()))
    ref = F.gelu(F.conv2d(x.double().permute(0, 3, 1, 2), w.double().view(C, 1, 3, 3), b.double(), 1, 1, groups=C)).permute(0, 2, 3, 1)
    _check(f'sp_dwconv_gelu C={C}', y, ref)


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
    _check('sp_head_fuse', y, torch.relu(acc).permute(0, 2, 3, 1))


@pytest.mark.parametrize('B', [1, 4])
def test_leaky(B):
    x = _rand((B, 128, 128, 256), 60, F16)
    ref = F.leaky_relu(x.double(), 0.01)
    capi.check(lib().r3dp_sp_leaky(P(x, F16), x.numel(), 0.01, capi.stream()))
    _check('sp_leaky', x, ref)


@pytest.mark.parametrize('B', [1, 4])
def test_upsample2_flip(B):
    x = _rand((B, 128, 128, 256), 70, F16)
    yr, yrc = torch.empty(B, 256, 256, 256, device=DEV, dtype=F16), torch.empty(B, 256, 256, 256, device=DEV, dtype=F16)
    capi.check(lib().r3dp_sp_upsample2_flip(P(x, F16), B, 128, 128, 256, P(yr, F16), P(yrc, F16), capi.stream()))
    up = F.interpolate(x.double().permute(0, 3, 1, 2), scale_factor=2.0, mode='bilinear', align_corners=True).permute(0, 2, 3, 1)
    _check('sp_upsample2_flip rows', yr, up.flip(1))
    _check('sp_upsample2_flip rows+cols', yrc, up.flip(1, 2))
