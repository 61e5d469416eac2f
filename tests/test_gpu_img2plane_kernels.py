"""Every new entry point of the canonical plane backbone (r3dp_ip_*, r3dp_sp_patches_dil, r3dp_sp_layernorm at C = 1024) against float64
of the very operands the kernel reads, at every launch shape of Img2PlaneModel.forward at 512^2 (B = 1, 4), 144^2 (B = 3) and 16^2 (B = 1),
and at odd sizes.  Outputs sit between sentinel guards: every element must be written and nothing past it.  Bar (the form of
test_gpu_sr_conv_conformance.py):

    |got - ref| <= ALPHA * |ref| + beta * S

ALPHA is the rounding of the stored type.  Attention: S = max |v|; rounding P to fp16 for P.V bounds the error by 2^-11 * sum p |v| <=
2^-11 max |v| = 4.9e-4; beta is asserted at about twice the worst measured (BETA, DESIGN.md), which an fp16 softmax or an fp16 channel-mean
accumulation exceeds.  The copies (input packing, max-pool, broadcast,
patch rows, flip) are exact."""
import math

import pytest
import torch
import torch.nn.functional as F

import img2plane_reference as iref
from real3dportrait_b200 import _capi as capi

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
F16, F32, F64 = torch.float16, torch.float32, torch.float64
ALPHA = {F16: 2.0 ** -11, F32: 2.0 ** -23}
#: about 2x the worst beta measured here and in tests/test_gpu_img2plane_launches.py on an H100 80GB HBM3 (700 W power limit): attention
#: 1.14e-4 (16^2's Tq = 16, Tk = 4 at padded strides; 7.1e-5 at the module's), channel mean 4.73e-7 (512^2 B = 4), layernorm 9.6e-8,
#: upsample2 3.96e-6
BETA = {'attention': 2.5e-4, 'layernorm': 2e-7, 'mean': 1e-6, 'shuffle': 0.0, 'upsample2': 2e-5}
P = capi.ptr


def lib():
    return capi.lib()


def _g(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _rand(shape, seed, dtype=F32, scale=1.0):
    return (torch.randn(shape, generator=_g(seed), device=DEV) * scale).to(dtype).contiguous()


def check_bar(name, got, ref, S=None):
    ref = ref.to(F64)
    S = float(ref.abs().max()) if S is None else S
    excess = (got.to(F64) - ref).abs() - ALPHA[got.dtype] * ref.abs()
    b = max(float(excess.max()), 0.0) / S
    bar = BETA[name.split()[0]]
    print(f'{name}: beta = {b:.2e} (bar {bar:.1e})')
    assert b <= bar, (name, b, bar)


#: the forwards whose launches the tables below hold (img2plane_reference.launch_plan), as tests/test_gpu_img2plane_launches.py records them
PLAN = [(512, 4, 'standard'), (512, 1, 'standard'), (144, 3, 'standard'), (32, 3, 'standard'), (16, 1, 'standard'), (64, 1, 'small'),
        (64, 1, 'large')]


def _plan_rows(fn, pick):
    rows = []
    for H, B, scale in PLAN:
        for launch in iref.launch_plan(H, B, scale):
            if launch.fn == fn and pick(launch.args) not in rows:
                rows.append(pick(launch.args))
    return rows


# (B, Tq, Tk) of every attention launch of forward: LowResolutionViT (Tq = Tk = (H/16)^2), TriplanePredictorViT ((H/4)^2, (H/8)^2); then
# odd shapes.  Here at padded strides; tests/test_gpu_img2plane_launches.py runs the forward's launches at the module's strides.
ATT_ROWS = _plan_rows('r3dp_ip_attention', lambda a: (a[2], a[3], a[4])) + [(2, 200, 77), (1, 129, 65), (2, 64, 1)]


@pytest.mark.parametrize('B,Tq,Tk', ATT_ROWS, ids=lambda v: str(v))
def test_attention(B, Tq, Tk):
    C, heads, qs, kvs, os_ = 1024, 4, 1024 + 64, 2048 + 8, 1024 + 16
    q = _rand((B, Tq, qs), 1, F16)
    kv = _rand((B, Tk, kvs), 2, F16)
    o = torch.full((B * Tq + 1, os_), float('nan'), device=DEV, dtype=F16)
    capi.check(lib().r3dp_ip_attention(P(q, F16), qs, P(kv, F16), kvs, B, Tq, Tk, heads, 1.0 / 16.0, P(o, F16), os_, capi.stream()))
    torch.cuda.synchronize()
    got = o[:B * Tq].view(B, Tq, os_)
    assert not torch.isnan(got[..., :C]).any(), 'unwritten output'
    assert torch.isnan(got[..., C:]).all() and torch.isnan(o[B * Tq:]).all(), 'write past the output'
    S = float(kv[..., C:2 * C].abs().max())
    for b in range(B):
        for h in range(heads):
            qh = q[b, :, h * 256:(h + 1) * 256].to(F64)
            kh = kv[b, :, h * 256:(h + 1) * 256].to(F64)
            vh = kv[b, :, C + h * 256:C + (h + 1) * 256].to(F64)
            ref = ((qh @ kh.T) / 16.0).softmax(-1) @ vh
            check_bar(f'attention B{B} Tq{Tq} Tk{Tk} b{b} h{h}', got[b, :, h * 256:(h + 1) * 256], ref, S)


# R of every C = 1024 LayerNorm launch: LowResolutionViT (H/16)^2 B, TriplanePredictorViT queries (H/4)^2 B and sr keys (H/8)^2 B, at
# 512^2 B = 1 and 4, 144^2 B = 3, 16^2 B = 1; plus odd counts
@pytest.mark.parametrize('R', [1024, 16384, 4096, 1024 * 4, 16384 * 4, 4096 * 4, 243, 3888, 972, 1, 16, 4, 7])
def test_layernorm_1024(R):
    C = 1024
    x, t = _rand((R, C), 3), _rand((R, C), 4, scale=0.5)
    g, b = 1 + 0.1 * _rand((C,), 5), 0.1 * _rand((C,), 6)
    xo = torch.empty_like(x)
    yf = torch.empty_like(x)
    yh = torch.full((R, C + 8), float('nan'), device=DEV, dtype=F16)
    capi.check(lib().r3dp_sp_layernorm(P(x), P(t), R, C, P(g), P(b), 1e-5, P(xo), P(yf), P(yh, F16), C + 8, capi.stream()))
    torch.cuda.synchronize()
    v = x.to(F64) + t.to(F64)
    ref = F.layer_norm(v, (C,), g.to(F64), b.to(F64), 1e-5)
    assert torch.equal(xo, x + t)
    check_bar(f'layernorm R{R} yf', yf, ref)
    check_bar(f'layernorm R{R} yh', yh[:, :C], ref)
    assert torch.isnan(yh[:, C:]).all()


# (B, H, C, k, s, p, d) of every patch-row launch of the PLAN forwards: stems, layer2's strided conv and downsample, the dilated
# layer3 / layer4 / ASPP convs, the patch embeds and the sr conv; then layer2's two at B = 2
PATCH_ROWS = _plan_rows('r3dp_sp_patches_dil', lambda a: (a[0], a[1], *a[3:8])) + [(2, 128, 64, 3, 2, 1, 1), (2, 128, 64, 1, 2, 0, 1)]


@pytest.mark.parametrize('B,H,C,k,s,p,d', PATCH_ROWS, ids=lambda v: str(v))
def test_patches_dil(B, H, C, k, s, p, d):
    x = _rand((B, H, H, C), 7, F16)
    ho = (H + 2 * p - d * (k - 1) - 1) // s + 1
    ldy = (k * k * C + 31) // 32 * 32
    y = torch.full((B * ho * ho + 1, ldy), float('nan'), device=DEV, dtype=F16)
    capi.check(lib().r3dp_sp_patches_dil(P(x, F16), B, H, H, C, k, s, p, d, P(y, F16), ldy, capi.stream()))
    torch.cuda.synchronize()
    ref = F.unfold(x.permute(0, 3, 1, 2).float(), k, dilation=d, padding=p, stride=s)       # [B, C*k*k, L], column c*k*k + tap
    ref = ref.view(B, C, k * k, -1).permute(0, 3, 2, 1).reshape(B * ho * ho, k * k * C).to(F16)
    assert torch.equal(y[:-1, :k * k * C], ref)
    assert (y[:-1, k * k * C:] == 0).all()
    assert torch.isnan(y[-1]).all()


@pytest.mark.parametrize('B,H', [(1, 512), (4, 512), (3, 144), (1, 16), (2, 20)])
def test_input_packing(B, H):
    x = _rand((B, 3, H, H), 8)
    y = torch.full((B * H * H + 1, 8), float('nan'), device=DEV, dtype=F16)
    capi.check(lib().r3dp_ip_input(P(x), B, H, H, P(y, F16), capi.stream()))
    torch.cuda.synchronize()
    i = (torch.arange(H, device=DEV, dtype=F32) / H).view(1, H, 1).expand(B, H, H)
    j = (torch.arange(H, device=DEV, dtype=F32) / H).view(1, 1, H).expand(B, H, H)
    ref = torch.stack([x[:, 0], x[:, 1], x[:, 2], i, j] + [torch.zeros_like(i)] * 3, -1).reshape(-1, 8).to(F16)
    assert torch.equal(y[:-1], ref)
    assert torch.isnan(y[-1]).all()


@pytest.mark.parametrize('B,H,C', [(1, 256, 64), (4, 256, 64), (3, 72, 64), (1, 8, 64), (2, 7, 16)])
def test_maxpool(B, H, C):
    x = _rand((B, H, H, C), 9, F16)
    ho = (H - 1) // 2 + 1
    y = torch.full((B * ho * ho + 1, C), float('nan'), device=DEV, dtype=F16)
    capi.check(lib().r3dp_ip_maxpool(P(x, F16), B, H, H, C, P(y, F16), capi.stream()))
    torch.cuda.synchronize()
    ref = F.max_pool2d(x.permute(0, 3, 1, 2).float(), 3, 2, 1).permute(0, 2, 3, 1).reshape(-1, C).to(F16)
    assert torch.equal(y[:-1], ref)
    assert torch.isnan(y[-1]).all()


@pytest.mark.parametrize('B,HW,C', [(1, 4096, 512), (4, 4096, 512), (3, 324, 512), (1, 4, 512), (2, 1, 64)])
def test_channel_mean_and_broadcast(B, HW, C):
    x = _rand((B, HW, C), 10, F16)
    m = torch.full((B + 1, C), float('nan'), device=DEV, dtype=F16)
    capi.check(lib().r3dp_ip_channel_mean(P(x, F16), B, HW, C, P(m, F16), capi.stream()))
    ys, yc0, Cb = 1280, 1024, 256
    y = torch.full((B, HW, ys), float('nan'), device=DEV, dtype=F16)
    v = _rand((B, Cb), 11, F16)
    capi.check(lib().r3dp_ip_broadcast(P(v, F16), B, HW, Cb, P(y, F16), ys, yc0, capi.stream()))
    torch.cuda.synchronize()
    check_bar(f'mean B{B} HW{HW}', m[:B], x.to(F64).mean(1))
    assert torch.isnan(m[B]).all()
    assert torch.equal(y[..., yc0:], v[:, None, :].expand(B, HW, Cb))
    assert torch.isnan(y[..., :yc0]).all()


@pytest.mark.parametrize('B,h,ys,yc0', [(1, 32, 256, 0), (4, 32, 256, 0), (1, 128, 448, 0), (4, 128, 448, 0), (3, 9, 256, 0),
                                        (3, 36, 448, 0), (1, 1, 256, 0), (1, 4, 448, 0), (2, 5, 260, 2)])
def test_pixel_shuffle(B, h, ys, yc0):
    C = 256
    x, t = _rand((B, h * h, 4 * C), 12), _rand((B, h * h, 4 * C), 13)
    y = torch.full((B, 2 * h, 2 * h, ys), float('nan'), device=DEV, dtype=F16)
    capi.check(lib().r3dp_ip_pixel_shuffle(P(x), P(t), B, h, h, C, P(y, F16), ys, yc0, capi.stream()))
    torch.cuda.synchronize()
    ref = F.pixel_shuffle((x + t).view(B, h, h, 4 * C).permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1).to(F16)
    assert torch.equal(y[..., yc0:yc0 + C], ref)
    assert torch.isnan(y[..., :yc0]).all() and torch.isnan(y[..., yc0 + C:]).all()


@pytest.mark.parametrize('B,h,C', [(1, 64, 256), (4, 64, 256), (1, 128, 128), (4, 128, 128), (3, 18, 256), (3, 36, 128), (1, 2, 256),
                                   (1, 4, 128), (2, 1, 8)])
def test_upsample2(B, h, C):
    x = _rand((B, h, h, C), 14, F16)
    y = torch.full((B * 4 * h * h + 1, C), float('nan'), device=DEV, dtype=F16)
    capi.check(lib().r3dp_ip_upsample2(P(x, F16), B, h, h, C, P(y, F16), capi.stream()))
    torch.cuda.synchronize()
    ref = F.interpolate(x.permute(0, 3, 1, 2).to(F64), scale_factor=2.0, mode='bilinear', align_corners=True).permute(0, 2, 3, 1).reshape(-1, C)
    check_bar(f'upsample2 B{B} h{h}', y[:-1], ref)
    assert torch.isnan(y[-1]).all()


@pytest.mark.parametrize('B,H', [(1, 256), (4, 256), (3, 72), (1, 8), (2, 5)])
def test_flip_hwpc(B, H):
    x = _rand((B, H, H, 96), 15)
    out = torch.full((B * H * H * 96 + 7,), float('nan'), device=DEV)
    capi.check(lib().r3dp_ip_flip_hwpc(P(x), B, H, H, P(out), capi.stream()))
    torch.cuda.synchronize()
    p = x.permute(0, 3, 1, 2).reshape(B, 3, 32, H, H)
    planes = torch.stack([p[:, 0].flip(2), p[:, 1].flip(2), p[:, 2].flip(2, 3)], 1)       # img2plane_model.py:72-81
    assert torch.equal(out[:-7].view(B, H, H, 3, 32), planes.permute(0, 3, 4, 1, 2))
    assert torch.isnan(out[-7:]).all()
