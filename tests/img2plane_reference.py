"""Float64 restatement of Img2PlaneModel (modules/img2plane/img2plane_model.py:12-81, 'rgb' input, tri-planes) on plain
torch.nn.functional, from a state_dict with the reference's keys.  Written from the network's semantics; it imports nothing from the library:
the tests compare the library against it, and it against the fixture the reference's own class wrote (tests/golden/img2plane_small.npz).

Also here: the seeded synthetic parameters and inputs the fixture and the tests share, and the shims that let the reference's class be
built without timm, pretrainedmodels, the global hparams or a network connection (tests/golden/make_golden_img2plane.py)."""
import math
import os
import socket
import sys
import types
import zlib
from typing import NamedTuple, Optional

import torch
import torch.nn.functional as F

from launch_harness import launch_signature

LAYERS = [3, 4, 6, 3]
DILATION = [1, 1, 2, 4]
RATES = (12, 24, 36)
SCALES = {'small': (2, 1), 'standard': (5, 1), 'large': (10, 3)}
ENC = 'low_reso_encoder.encoder'
ASPP = 'low_reso_encoder.decoder.0'


# ---- seeded synthetic parameters and inputs -------------------------------------------------------------------------------------------
def make_params(shapes, seed=0):
    """{key: shape} -> {key: float32 tensor}, each drawn from its own generator (seed, crc32(key)).  Scales keep every stage's activations
    O(1): He-scaled convs (sqrt(2 / fan_in)), linears 1/sqrt(fan_in), BatchNorm running statistics and LayerNorm affines near identity, and
    the last BatchNorm of each residual branch (bn2) at a gain of ~0.3 so that sixteen residual adds do not grow the stream."""
    out = {}
    for k, shape in shapes.items():
        g = torch.Generator().manual_seed(seed * 1_000_003 + zlib.crc32(k.encode()))
        shape = tuple(shape)
        leaf = k.rsplit('.', 1)[-1]
        mod = k.rsplit('.', 2)[-2] if k.count('.') >= 1 else ''
        if leaf == 'num_batches_tracked':
            out[k] = torch.zeros((), dtype=torch.long)
        elif leaf == 'running_mean':
            out[k] = 0.05 * torch.randn(shape, generator=g)
        elif leaf == 'running_var':
            out[k] = 0.9 + 0.2 * torch.rand(shape, generator=g)
        elif len(shape) == 1:
            if leaf == 'weight':
                gain = 0.3 if mod == 'bn2' else 1.0
                out[k] = gain * (1.0 + 0.1 * torch.randn(shape, generator=g))
            else:
                out[k] = 0.05 * torch.randn(shape, generator=g)
        elif len(shape) == 4:
            fan_in = math.prod(shape[1:])
            out[k] = torch.randn(shape, generator=g) * math.sqrt((1.0 if shape[1] == 1 else 2.0) / fan_in)
        else:
            out[k] = torch.randn(shape, generator=g) / math.sqrt(shape[1])
    return out


def make_inputs(B, H, seed=1):
    """B rgb images in [-1, 1] with some spatial structure: [B,3,H,H] float32."""
    g = torch.Generator().manual_seed(seed)
    base = torch.rand(B, 3, H // 8, H // 8, generator=g) * 2 - 1
    img = F.interpolate(base, size=(H, H), mode='bilinear', align_corners=False)
    return (0.8 * img + 0.2 * (torch.rand(B, 3, H, H, generator=g) * 2 - 1)).clamp(-1, 1)


# ---- the float64 forward ----------------------------------------------------------------------------------------------------------------
def _bn(x, sd, p):
    return F.batch_norm(x, sd[p + '.running_mean'], sd[p + '.running_var'], sd[p + '.weight'], sd[p + '.bias'], False, 0.0, 1e-5)


def _lin(x, sd, p):
    return F.linear(x, sd[p + '.weight'], sd[p + '.bias'])


def _ln(x, sd, p):
    return F.layer_norm(x, x.shape[-1:], sd[p + '.weight'], sd[p + '.bias'], 1e-5)


def _conv(x, sd, p, stride=1, padding=1, dilation=1):
    return F.conv2d(x, sd[p + '.weight'], sd.get(p + '.bias'), stride, padding, dilation)


def with_coords(x):
    """img2plane_model.py:59-64: channel 3 = row / H, channel 4 = column / H (torch.meshgrid 'ij')."""
    B, _, H, W = x.shape
    i = (torch.arange(H, dtype=x.dtype, device=x.device) / H).view(1, 1, H, 1).expand(B, 1, H, W)
    j = (torch.arange(W, dtype=x.dtype, device=x.device) / H).view(1, 1, 1, W).expand(B, 1, H, W)
    return torch.cat([x, i, j], 1)


def encoder(sd, x):
    """ResNet-34 at output stride 8 (every conv of layer3 / layer4 at stride 1, dilation 2 / 4, padding (k // 2) d) -> layer4 [B,512,H/8,H/8]."""
    e = F.relu(_bn(F.conv2d(x, sd[ENC + '.conv1.weight'], None, 2, 3), sd, ENC + '.bn1'))
    e = F.max_pool2d(e, 3, 2, 1)
    for li, (n, d) in enumerate(zip(LAYERS, DILATION)):
        for b in range(n):
            p = f'{ENC}.layer{li + 1}.{b}'
            s = 2 if (li == 1 and b == 0) else 1
            t = F.relu(_bn(F.conv2d(e, sd[p + '.conv1.weight'], None, s, d, d), sd, p + '.bn1'))
            t = _bn(F.conv2d(t, sd[p + '.conv2.weight'], None, 1, d, d), sd, p + '.bn2')
            idn = _bn(F.conv2d(e, sd[p + '.downsample.0.weight'], None, s), sd, p + '.downsample.1') if p + '.downsample.0.weight' in sd else e
            e = F.relu(t + idn)
    return e


def decoder(sd, e):
    """ASPP (no BN, ReLU; the pooling branch is a per-image broadcast; dropout off) then the bias-free 3x3 conv, no activation."""
    h, w = e.shape[2:]
    br = [F.relu(F.conv2d(e, sd[ASPP + '.convs.0.0.weight']))]
    for k, r in enumerate(RATES):
        br.append(F.relu(F.conv2d(e, sd[f'{ASPP}.convs.{k + 1}.0.weight'], None, 1, r, r)))
    pooled = F.relu(F.conv2d(e.mean((2, 3), keepdim=True), sd[ASPP + '.convs.4.1.weight']))
    br.append(pooled.expand(-1, -1, h, w))
    y = F.relu(F.conv2d(torch.cat(br, 1), sd[ASPP + '.project.0.weight']))
    return F.conv2d(y, sd['low_reso_encoder.decoder.1.weight'], None, 1, 1)


def block(sd, p, x, H, W, sr):
    """segformer/base.py Block: 4 heads of 256, qkv bias, scale 1/16, LayerNorm eps 1e-5, DWConv Mlp with exact GELU."""
    B, N, C = x.shape
    y = _ln(x, sd, p + '.norm1')
    q = _lin(y, sd, p + '.attn.q').reshape(B, N, 4, C // 4).permute(0, 2, 1, 3)
    if sr > 1:
        y_ = F.conv2d(y.permute(0, 2, 1).reshape(B, C, H, W), sd[p + '.attn.sr.weight'], sd[p + '.attn.sr.bias'], sr)
        y_ = _ln(y_.reshape(B, C, -1).permute(0, 2, 1), sd, p + '.attn.norm')
    else:
        y_ = y
    kv = _lin(y_, sd, p + '.attn.kv').reshape(B, -1, 2, 4, C // 4).permute(2, 0, 3, 1, 4)
    att = ((q @ kv[0].transpose(-2, -1)) / 16.0).softmax(-1)
    x = x + _lin((att @ kv[1]).transpose(1, 2).reshape(B, N, C), sd, p + '.attn.proj')
    y = _lin(_ln(x, sd, p + '.norm2'), sd, p + '.mlp.fc1')
    hid = y.shape[-1]
    y = F.conv2d(y.transpose(1, 2).reshape(B, hid, H, W), sd[p + '.mlp.dwconv.dwconv.weight'], sd[p + '.mlp.dwconv.dwconv.bias'], 1, 1,
                 groups=hid)
    return x + _lin(F.gelu(y.flatten(2).transpose(1, 2)), sd, p + '.mlp.fc2')


def vit_tokens(sd, p, x, nblocks, sr):
    """OverlapPatchEmbed (3x3/2, LayerNorm) then the blocks -> [B,1024,H,W] (no final norm)."""
    x = _conv(x, sd, p + '.patch_embed.proj', 2, 1)
    B, C, H, W = x.shape
    x = _ln(x.flatten(2).transpose(1, 2), sd, p + '.patch_embed.norm')
    for i in range(1, nblocks + 1):
        x = block(sd, f'{p}.block{i}', x, H, W, sr)
    return x.permute(0, 2, 1).reshape(B, C, H, W)


def low_vit(sd, x, nblocks):
    p = 'low_reso_vit'
    h = F.pixel_shuffle(vit_tokens(sd, p, x, nblocks, 1), 2)
    h = F.relu(_conv(F.interpolate(h, scale_factor=2.0, mode='bilinear', align_corners=True), sd, p + '.conv_after_upsample1'))
    h = F.relu(_conv(F.interpolate(h, scale_factor=2.0, mode='bilinear', align_corners=True), sd, p + '.conv_after_upsample2'))
    return _conv(h, sd, p + '.final_conv')


def high_res(sd, x):
    p = 'high_reso_encoder'
    h = _conv(x, sd, p + '.first', 2, 3)
    for i in (0, 2, 4, 6):
        h = F.leaky_relu(_conv(h, sd, f'{p}.conv_layers.{i}'), 0.01)
    return _conv(h, sd, p + '.final')


def tri_vit(sd, low, high, nblocks):
    p = 'triplane_predictor_vit'
    h = F.leaky_relu(_conv(torch.cat([low, high], 1), sd, p + '.first_conv'), 0.01)
    h = F.leaky_relu(_conv(h, sd, p + '.second_conv'), 0.01)
    h = F.pixel_shuffle(vit_tokens(sd, p, h, nblocks, 2), 2)
    h = torch.cat([h, low], 1)
    for name in ('first_conv_after_cat', 'second_conv_after_cat', 'third_conv_after_cat'):
        h = F.leaky_relu(_conv(h, sd, f'{p}.{name}'), 0.01)
    return _conv(h, sd, p + '.final_conv')


def flip_planes(y):
    """img2plane_model.py:72-81: [B,96,h,w] -> [B,3,32,h,w], planes 0 and 1 flipped along rows, plane 2 along rows and columns."""
    p = y.view(len(y), 3, -1, y.shape[-2], y.shape[-1])
    return torch.stack([p[:, 0].flip(2), p[:, 1].flip(2), p[:, 2].flip(2, 3)], 1)


def forward(sd, x, scale='standard'):
    """x [B,3,H,H] -> planes [B,3,32,H/2,H/2], in the dtype of sd and x (float64 for the tests)."""
    nlow, ntri = SCALES[scale]
    x = with_coords(x)
    low = low_vit(sd, decoder(sd, encoder(sd, x)), nlow)
    return flip_planes(tri_vit(sd, low, high_res(sd, x), ntri))


# ---- the launch plan ------------------------------------------------------------------------------------------------------------------
DIM, MLP, HEADS = 1024, 2048, 4
WIDTHS = [64, 128, 256, 512]


class Launch(NamedTuple):
    """One C call of Img2PlaneModel.forward.  args: the non-pointer arguments in C order.  reads / writes: {role: (buffer, c0, c1)}, the
    channels [c0, c1) of a named NHWC (or row-major) buffer the call reads or writes through the pointer argument `role` (the C argument's
    name: x, t, res, y, xo, yf, yh, q, kv, o).  conv: (cin, k, s, p, d) of the convolution an r3dp_mf_conv3d launch computes (its patch rows'
    geometry for a patch-row GEMM; k = 1 for 1x1 convs and token linears), None for other entry points."""
    tag: str
    fn: str
    args: tuple
    reads: dict
    writes: dict
    conv: Optional[tuple] = None


def ceil32(n):
    return (n + 31) // 32 * 32


def cop_of(cout):
    """Packed couts of an r3dp_mf_conv3d launch: cout rounded up to its cout tile (16, 32, 64 or 128)."""
    bn = 16 if cout <= 16 else 32 if cout <= 32 else 64 if cout <= 64 else 128
    return -(-cout // bn) * bn


def row_key(fn, args, reads, writes):
    """What decides a launch apart from the data: the signature, and what the arguments do not show.  r3dp_mf_conv3d: whether it adds a
    residual and the channel offset of its input; r3dp_sp_layernorm: which of t / xo / yf / yh it is given and whether xo is x (in place)."""
    sig = launch_signature(fn, args)
    if fn == 'r3dp_mf_conv3d':
        return sig + ('res' in reads, reads['x'][1])
    if fn == 'r3dp_sp_layernorm':
        return sig + (tuple(r for r in ('t', 'xo', 'yf', 'yh') if r in reads or r in writes), writes.get('xo', (None,))[0] == reads['x'][0])
    return sig


def tc_route(cin, cout, xs, h, own=True, res=False, out_f32=False):
    """Img2PlaneModel's rule for a stride-1 3x3 conv: r3dp_sr_tc_conv for 128 or 256 outputs on a dense input of a multiple of 64 channels,
    h % 128 == 0 (tiles of 128-pixel rows), written into a tensor of its own without a residual or an fp32 store."""
    return cout in (128, 256) and cin % 64 == 0 and xs == cin and h % 128 == 0 and own and not res and not out_f32


def launch_plan(H, B, scale='standard'):
    """Every C call of Img2PlaneModel.forward on [B, 3, H, H] at `scale`, in order, as Launch records.  Written from the architecture (the
    float64 forward above, DESIGN.md "Canonical plane backbone" -> Launches): r3dp_ip_input packs rgb + coordinates to 8 fp16 channels;
    strided, dilated and non-3x3 convs run as r3dp_sp_patches_dil rows (K padded to a multiple of 32) times the r3dp_mf_conv3d GEMM (rows on
    the H axis), stride-1 1x1 convs and token linears as the GEMM on the input itself, stride-1 3x3 convs as (1,3,3) taps or, by tc_route,
    r3dp_sr_tc_conv with the activation in its epilogue; BatchNorm is folded, ReLU fused (relu = 1), LeakyReLU and the BasicBlock's ReLU
    after the residual add are r3dp_sp_leaky in place.  ASPP's branches fill cat1280 = [1x1 | r12 | r24 | r36 | pooled]; the two
    concatenations of the planes are one buffer cat448 = [shuffled tokens 256 | low 96 | high 96]."""
    nlow, ntri = SCALES[scale]
    plan = []
    bufs = {}                                      # buffer -> channels

    def add(tag, fn, args, reads=None, writes=None, conv=None):
        plan.append(Launch(tag, fn, tuple(args), dict(reads or {}), dict(writes or {}), conv))

    def buf(name, ch):
        bufs[name] = ch
        return name

    def full(name):
        return (name, 0, bufs[name])

    def gemm(tag, src, R, O, y, relu=0, f32=False, res=None, yc0=0, conv=None):
        """r3dp_mf_conv3d GEMM on the rows of `src` (xs = K = its width) -> y[:, yc0:yc0 + O] (y's width ys)."""
        K, ys = bufs[src], bufs[y]
        reads = {'x': full(src)}
        if res is not None:
            reads['res'] = full(res)
        add(tag, 'r3dp_mf_conv3d', (K, 0, K, 1, 1, R, 1, 1, 1, 1, 0, O, cop_of(O), relu, ys, yc0, 0, int(f32), 0), reads,
            {'y': (y, yc0, yc0 + O)}, conv or (K, 1, 1, 0, 1))

    def conv(tag, src, h, cin, O, k, s, p, d, act=None, y=None, yc0=0, res=None, f32=False, xc0=0):
        """One convolution of src's channels [xc0, xc0 + cin) on h x h -> (output buffer, ho), by the module's route."""
        ho = (h + 2 * p - d * (k - 1) - 1) // s + 1
        own = y is None
        if own:
            y = buf(tag, O)
        relu = int(act == 'relu')
        xs = bufs[src]
        if k == 3 and s == 1 and p == 1 and d == 1:
            if tc_route(cin, O, xs, h, own, res is not None, f32):
                add(tag, 'r3dp_sr_tc_conv', (B, 1, cin, O, h, h, 3, {None: 0, 'leaky': 2, 'relu': 3}[act]), {'x': full(src)}, {'y': full(y)})
                return y, ho
            reads = {'x': (src, xc0, xc0 + cin)}
            if res is not None:
                reads['res'] = full(res)
            add(tag, 'r3dp_mf_conv3d', (xs, 0, cin, B, 1, h, h, 1, 3, 3, 0, O, cop_of(O), relu, bufs[y], yc0, 0, int(f32), 0), reads,
                {'y': (y, yc0, yc0 + O)}, (cin, 3, 1, 1, 1))
        elif k == 1 and s == 1:
            gemm(tag, src, B * h * h, O, y, relu, f32, res, yc0)
        else:
            assert xs == cin and xc0 == 0
            ldy = ceil32(k * k * cin)
            pt = buf(tag + '.patches', ldy)
            add(tag + '.patches', 'r3dp_sp_patches_dil', (B, h, h, cin, k, s, p, d, ldy), {'x': full(src)}, {'y': full(pt)})
            gemm(tag, pt, B * ho * ho, O, y, relu, f32, res, yc0, (cin, k, s, p, d))
        if act == 'leaky':
            add(tag + '.leaky', 'r3dp_sp_leaky', (B * ho * ho * O, 0.01), {'x': full(y)}, {'x': full(y)})
        return y, ho

    def layernorm(tag, x, R, t=None, xo=None, yf=None, yh=None):
        reads = {'x': full(x)}
        writes = {}
        if t is not None:
            reads['t'] = full(t)
        for role, b in (('xo', xo), ('yf', yf), ('yh', yh)):
            if b is not None:
                writes[role] = full(b)
        add(tag, 'r3dp_sp_layernorm', (R, DIM, 1e-5, DIM), reads, writes)

    def vit(p, src, h, cin, nblocks, sr):
        t0, hv = conv(p + '.pe', src, h, cin, DIM, 3, 2, 1, 1, f32=True)
        R = B * hv * hv
        xres = buf(p + '.xres', DIM)
        layernorm(p + '.pe_norm', t0, R, yf=xres)
        a = buf(p + '.a', DIM)
        layernorm(p + '.block1.norm1', xres, R, yh=a)
        t = None
        for i in range(1, nblocks + 1):
            b = f'{p}.block{i}'
            q = buf(b + '.q', DIM)
            gemm(b + '.q', a, R, DIM, q)
            if sr > 1:
                r, hk = conv(b + '.sr', a, hv, DIM, DIM, sr, sr, 0, 1, f32=True)
                a2 = buf(b + '.sr_norm', DIM)
                layernorm(b + '.sr_norm', r, B * hk * hk, yh=a2)
                kv, tk = buf(b + '.kv', 2 * DIM), hk * hk
                gemm(b + '.kv', a2, B * hk * hk, 2 * DIM, kv)
            else:
                kv, tk = buf(b + '.kv', 2 * DIM), hv * hv
                gemm(b + '.kv', a, R, 2 * DIM, kv)
            o = buf(b + '.attn', DIM)
            add(b + '.attn', 'r3dp_ip_attention', (DIM, 2 * DIM, B, hv * hv, tk, HEADS, 1.0 / 16.0, DIM), {'q': full(q), 'kv': full(kv)},
                {'o': full(o)})
            t = buf(b + '.proj', DIM)
            gemm(b + '.proj', o, R, DIM, t, f32=True)
            layernorm(b + '.norm2', xres, R, t=t, xo=xres, yh=a)
            f1 = buf(b + '.fc1', MLP)
            gemm(b + '.fc1', a, R, MLP, f1)
            f2 = buf(b + '.dwconv', MLP)
            add(b + '.dwconv', 'r3dp_sp_dwconv_gelu', (B, hv, hv, MLP), {'x': full(f1)}, {'y': full(f2)})
            t = buf(b + '.fc2', DIM)
            gemm(b + '.fc2', f2, R, DIM, t, f32=True)
            if i < nblocks:
                layernorm(f'{p}.block{i + 1}.norm1', xres, R, t=t, xo=xres, yh=a)
        return xres, t, hv

    H2 = H // 2
    buf('img', 3)
    xin = buf('xin', 8)
    add('input', 'r3dp_ip_input', (B, H, H), {'x': full('img')}, {'y': full(xin)})
    # ResNet-34 stem and the high-resolution encoder's 7x7/2 conv: one set of patch rows, two GEMMs
    h1 = (H - 1) // 2 + 1
    pt = buf('stem.patches', ceil32(49 * 8))
    add('stem.patches', 'r3dp_sp_patches_dil', (B, H, H, 8, 7, 2, 3, 1, bufs[pt]), {'x': full(xin)}, {'y': full(pt)})
    e = buf('stem', 64)
    gemm('stem', pt, B * h1 * h1, 64, e, relu=1, conv=(8, 7, 2, 3, 1))
    hi = buf('high.first', 64)
    gemm('high.first', pt, B * h1 * h1, 64, hi, conv=(8, 7, 2, 3, 1))
    h = (h1 - 1) // 2 + 1
    y = buf('maxpool', 64)
    add('maxpool', 'r3dp_ip_maxpool', (B, h1, h1, 64), {'x': full(e)}, {'y': full(y)})
    prev = 64
    for li, (n, c, d) in enumerate(zip(LAYERS, WIDTHS, DILATION)):
        for bi in range(n):
            p = f'layer{li + 1}.{bi}'
            s = 2 if (li == 1 and bi == 0) else 1
            t, ho = conv(p + '.conv1', y, h, prev, c, 3, s, d, d, act='relu')
            res = conv(p + '.downsample', y, h, prev, c, 1, s, 0, 1)[0] if (bi == 0 and li > 0) else y
            z, _ = conv(p + '.conv2', t, ho, c, c, 3, 1, d, d, res=res)
            add(p + '.relu', 'r3dp_sp_leaky', (B * ho * ho * c, 0.0), {'x': full(z)}, {'x': full(z)})
            y, h, prev = z, ho, c
    # ASPP into cat1280, then the projection and the decoder's 3x3 conv
    h8 = h
    cat = buf('cat1280', 1280)
    conv('aspp.0', y, h8, 512, 256, 1, 1, 0, 1, act='relu', y=cat, yc0=0)
    for i, r in enumerate(RATES):
        conv(f'aspp.{i + 1}', y, h8, 512, 256, 3, 1, r, r, act='relu', y=cat, yc0=256 * (i + 1))
    mean = buf('aspp.mean', 512)
    add('aspp.mean', 'r3dp_ip_channel_mean', (B, h8 * h8, 512), {'x': full(y)}, {'y': full(mean)})
    pooled = buf('aspp.pool', 256)
    gemm('aspp.pool', mean, B, 256, pooled, relu=1)
    add('aspp.broadcast', 'r3dp_ip_broadcast', (B, h8 * h8, 256, 1280, 1024), {'x': full(pooled)}, {'y': (cat, 1024, 1280)})
    proj, _ = conv('aspp.project', cat, h8, 1280, 256, 1, 1, 0, 1, act='relu')
    dec, _ = conv('decoder', proj, h8, 256, 256, 3, 1, 1, 1)
    # LowResolutionViT -> cat448[256:352]
    cat448 = buf('cat448', 448)
    xres, t, hv = vit('low', dec, h8, 256, nlow, 1)
    ps = buf('low.shuffle', 256)
    add('low.shuffle', 'r3dp_ip_pixel_shuffle', (B, hv, hv, 256, 256, 0), {'x': full(xres), 't': full(t)}, {'y': full(ps)})
    hu = 2 * hv
    for i, cout in ((1, 128), (2, 128)):
        up = buf(f'low.up{i}', bufs[ps])
        add(f'low.up{i}', 'r3dp_ip_upsample2', (B, hu, hu, bufs[ps]), {'x': full(ps)}, {'y': full(up)})
        hu *= 2
        ps, _ = conv(f'low.conv_after_upsample{i}', up, hu, bufs[up], cout, 3, 1, 1, 1, act='relu')
    conv('low.final_conv', ps, hu, 128, 96, 3, 1, 1, 1, y=cat448, yc0=256)
    # HighResoEncoder -> cat448[352:448]
    z = hi
    for i, cin in enumerate((64, 96, 96, 96)):
        z, _ = conv(f'high.conv_layers.{2 * i}', z, H2, cin, 96, 3, 1, 1, 1, act='leaky')
    conv('high.final', z, H2, 96, 96, 3, 1, 1, 1, y=cat448, yc0=352)
    # TriplanePredictorViT: first_conv on cat448[256:448], the shuffled tokens into cat448[0:256], first_conv_after_cat on cat448[0:352]
    z, _ = conv('tri.first_conv', cat448, H2, 192, 256, 3, 1, 1, 1, act='leaky', xc0=256)
    z, _ = conv('tri.second_conv', z, H2, 256, 128, 3, 1, 1, 1, act='leaky')
    xres, t, hv = vit('tri', z, H2, 128, ntri, 2)
    add('tri.shuffle', 'r3dp_ip_pixel_shuffle', (B, hv, hv, 256, 448, 0), {'x': full(xres), 't': full(t)}, {'y': (cat448, 0, 256)})
    z, _ = conv('tri.first_conv_after_cat', cat448, H2, 352, 256, 3, 1, 1, 1, act='leaky')
    z, _ = conv('tri.second_conv_after_cat', z, H2, 256, 128, 3, 1, 1, 1, act='leaky')
    z, _ = conv('tri.third_conv_after_cat', z, H2, 128, 128, 3, 1, 1, 1, act='leaky')
    yf, _ = conv('tri.final_conv', z, H2, 128, 96, 3, 1, 1, 1, f32=True)
    out = buf('planes', 96)
    add('flip', 'r3dp_ip_flip_hwpc', (B, H2, H2), {'x': full(yf)}, {'y': full(out)})
    return plan


def launch_count(H, scale='standard'):
    """len(launch_plan(H, B, scale)) from the block counts: 116 launches outside the ViT blocks, 9 per LowResolutionViT block and 12 per
    TriplanePredictorViT block (its sr conv: patch rows, GEMM, LayerNorm), less one (the first block's norm1 follows the patch embed's
    LayerNorm), and the three tensor-core convs at H/2 % 128 == 0 (fused LeakyReLU: 1 launch each) or r3dp_mf_conv3d + r3dp_sp_leaky (2)."""
    nlow, ntri = SCALES[scale]
    return 116 + 9 * nlow + 12 * ntri + 3 * (1 if (H // 2) % 128 == 0 else 2)


# ---- shims for building the reference's class ---------------------------------------------------------------------------------------
class NetworkBlocked(RuntimeError):
    pass


def block_network():
    """Every name lookup and socket connection raises: a missed shim fails instead of reaching a server (or a DNS resolver)."""
    def refuse(*a, **k):
        raise NetworkBlocked('network access is blocked while the reference class is built')
    socket.getaddrinfo = refuse
    socket.gethostbyname = refuse
    socket.gethostbyname_ex = refuse
    socket.socket.connect = refuse
    socket.socket.connect_ex = refuse
    socket.socket.sendto = refuse
    socket.create_connection = refuse


def reference_class(root, hp):
    """The reference's Img2PlaneModel with timm, pretrainedmodels and utils.commons.hparams shimmed, and model_zoo.load_url returning a
    locally built torchvision resnet34(weights=None) state_dict.  Installs the network guard first."""
    block_network()
    import torch.utils.model_zoo as model_zoo
    import torchvision

    def to_2tuple(v):
        return tuple(v) if isinstance(v, (tuple, list)) else (v, v)

    layers = types.ModuleType('timm.models.layers')
    layers.DropPath = lambda p: torch.nn.Identity()
    layers.to_2tuple = to_2tuple
    layers.trunc_normal_ = lambda t, std=1.0, **k: torch.nn.init.normal_(t, 0.0, std)
    timm = types.ModuleType('timm')
    timm.models = types.ModuleType('timm.models')
    timm.models.layers = layers
    pm = types.ModuleType('pretrainedmodels')
    pm.models = types.ModuleType('pretrainedmodels.models')
    tv = types.ModuleType('pretrainedmodels.models.torchvision_models')
    tv.pretrained_settings = {n: {'imagenet': {'url': f'local://{n}', 'input_space': 'RGB', 'input_size': [3, 224, 224], 'input_range': [0, 1],
                                               'mean': [0.485, 0.456, 0.406], 'std': [0.229, 0.224, 0.225], 'num_classes': 1000}}
                              for n in ('resnet18', 'resnet34', 'resnet50', 'resnet101', 'resnet152')}
    pm.models.torchvision_models = tv
    hpm = types.ModuleType('utils.commons.hparams')
    hpm.hparams = dict(hp)
    sys.modules.update({'timm': timm, 'timm.models': timm.models, 'timm.models.layers': layers, 'pretrainedmodels': pm,
                        'pretrainedmodels.models': pm.models, 'pretrainedmodels.models.torchvision_models': tv,
                        'utils': types.ModuleType('utils'), 'utils.commons': types.ModuleType('utils.commons'), 'utils.commons.hparams': hpm})

    def load_url(url, *a, **k):
        if url != 'local://resnet34':
            raise RuntimeError(f'unexpected weights {url}')
        return torchvision.models.resnet34(weights=None).state_dict()
    model_zoo.load_url = load_url
    if root not in sys.path:
        sys.path.insert(0, root)
    from modules.img2plane.img2plane_model import Img2PlaneModel
    return Img2PlaneModel


def reference_checkout():
    root = os.environ.get('R3DP_REFERENCE')
    return root if root and os.path.isdir(os.path.join(root, 'modules', 'img2plane')) else None
