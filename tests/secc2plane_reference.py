"""Float64 restatement of SegFormerSECC2PlaneBackbone('b0') (modules/real3d/segformer.py:60-733) on plain torch.nn.functional, from a
state_dict with the reference's keys.  It imports nothing from the library: the tests compare the library against it, and it against the
fixture the reference's own class wrote (tests/golden/secc2plane_small.npz).

Also here: the seeded synthetic parameters and inputs the fixture and the tests share, and the shims that let the reference's segformer.py
import without timm / mmcv (tests/golden/make_golden_secc2plane.py)."""
import math
import sys
import types
import zlib

import torch
import torch.nn as nn
import torch.nn.functional as F

from launch_harness import launch_signature  # noqa: F401  (the launch tests call it through this module)

EMBED = [32, 64, 160, 256]
HEADS = [1, 2, 5, 8]
SR = [8, 4, 2, 1]


# ---- seeded synthetic parameters and inputs -------------------------------------------------------------------------------------------
def make_params(shapes, seed=0):
    """{key: shape} -> {key: float32 tensor}: each tensor drawn from its own generator (seed, crc32(key)), so the set does not depend on key
    order.  Non-degenerate: LayerNorm / BatchNorm affines away from identity, running statistics away from (0, 1)."""
    out = {}
    for k, shape in shapes.items():
        g = torch.Generator().manual_seed(seed * 1_000_003 + zlib.crc32(k.encode()))
        shape = tuple(shape)
        leaf = k.rsplit('.', 1)[-1]
        if leaf == 'num_batches_tracked':
            out[k] = torch.zeros((), dtype=torch.long)
        elif leaf == 'resample_filter':
            f = torch.tensor([1., 3., 3., 1.])
            f = torch.outer(f, f)
            out[k] = f / f.sum()
        elif leaf == 'running_mean':
            out[k] = 0.1 * torch.randn(shape, generator=g)
        elif leaf == 'running_var':
            out[k] = 0.5 + torch.rand(shape, generator=g)
        elif len(shape) == 1:
            is_scale = leaf == 'weight'
            out[k] = (1.0 if is_scale else 0.0) + (0.2 if is_scale else 0.1) * torch.randn(shape, generator=g)
        elif k == 'prenet.weight':
            out[k] = torch.randn(shape, generator=g)               # Conv2dLayer applies 1/sqrt(cin) itself
        else:
            fan_in = math.prod(shape[1:])
            out[k] = torch.randn(shape, generator=g) / math.sqrt(fan_in)
    return out


def make_inputs(B, H, seed=1):
    """Three SECC-like images in [-1, 1]: cano [1,3,H,H], src [1,3,H,H], tgt [B,3,H,H]."""
    g = torch.Generator().manual_seed(seed)
    cano = torch.rand(1, 3, H, H, generator=g) * 2 - 1
    src = torch.rand(1, 3, H, H, generator=g) * 2 - 1
    tgt = torch.rand(B, 3, H, H, generator=g) * 2 - 1
    return cano, src, tgt


# ---- the float64 forward ----------------------------------------------------------------------------------------------------------------
def _ln(x, sd, p, eps):
    return F.layer_norm(x, x.shape[-1:], sd[p + '.weight'], sd[p + '.bias'], eps)


def _lin(x, sd, p):
    return F.linear(x, sd[p + '.weight'], sd[p + '.bias'])


def mit_b0(sd, x):
    """MixVisionTransformer.forward_features (segformer.py:351-390) -> [c1..c4] NCHW."""
    B = x.shape[0]
    outs = []
    for s in range(4):
        pre = f'mix_vit.patch_embed{s + 1}'
        k, st = (7, 4) if s == 0 else (3, 2)
        x = F.conv2d(x, sd[pre + '.proj.weight'], sd[pre + '.proj.bias'], st, k // 2)
        _, C, H, W = x.shape
        x = _ln(x.flatten(2).transpose(1, 2), sd, pre + '.norm', 1e-5)
        for bi in range(2):
            p = f'mix_vit.block{s + 1}.{bi}'
            y = _ln(x, sd, p + '.norm1', 1e-6)
            nh, hd = HEADS[s], C // HEADS[s]
            q = _lin(y, sd, p + '.attn.q').reshape(B, -1, nh, hd).permute(0, 2, 1, 3)
            if SR[s] > 1:
                y_ = y.permute(0, 2, 1).reshape(B, C, H, W)
                y_ = F.conv2d(y_, sd[p + '.attn.sr.weight'], sd[p + '.attn.sr.bias'], SR[s]).reshape(B, C, -1).permute(0, 2, 1)
                y_ = _ln(y_, sd, p + '.attn.norm', 1e-5)
            else:
                y_ = y
            kv = _lin(y_, sd, p + '.attn.kv').reshape(B, -1, 2, nh, hd).permute(2, 0, 3, 1, 4)
            att = ((q @ kv[0].transpose(-2, -1)) * hd ** -0.5).softmax(-1)
            o = (att @ kv[1]).transpose(1, 2).reshape(B, -1, C)
            x = x + _lin(o, sd, p + '.attn.proj')
            y = _lin(_ln(x, sd, p + '.norm2', 1e-6), sd, p + '.mlp.fc1')
            hid = y.shape[-1]
            y = F.conv2d(y.transpose(1, 2).reshape(B, hid, H, W), sd[p + '.mlp.dwconv.dwconv.weight'], sd[p + '.mlp.dwconv.dwconv.bias'], 1, 1,
                         groups=hid)
            y = F.gelu(y.flatten(2).transpose(1, 2))
            x = x + _lin(y, sd, p + '.mlp.fc2')
        x = _ln(x, sd, f'mix_vit.norm{s + 1}', 1e-6)
        x = x.reshape(B, H, W, -1).permute(0, 3, 1, 2).contiguous()
        outs.append(x)
    return outs


def head(sd, feats):
    """SegFormerHead.forward (segformer.py:525-537), unfolded: linear_c*, bilinear resize, cat, 1x1 conv, eval BN, ReLU."""
    c1 = feats[0]
    parts = []
    for i in (4, 3, 2, 1):
        c = feats[i - 1]
        n, _, h, w = c.shape
        t = _lin(c.flatten(2).transpose(1, 2), sd, f'fuse_head.linear_c{i}.proj').permute(0, 2, 1).reshape(n, -1, h, w)
        if i > 1:
            t = F.interpolate(t, size=c1.shape[2:], mode='bilinear', align_corners=False)
        parts.append(t)
    y = F.conv2d(torch.cat(parts, 1), sd['fuse_head.linear_fuse.conv.weight'])
    p = 'fuse_head.linear_fuse.bn'
    y = F.batch_norm(y, sd[p + '.running_mean'], sd[p + '.running_var'], sd[p + '.weight'], sd[p + '.bias'], False, 0.0, 1e-5)
    return F.relu(y)


def to_planes(sd, x):
    """to_plane_cnn and the three flips (segformer.py:692-701,719-731) -> [B,3,32,2h,2w]."""
    for i in (0, 2, 4):
        x = F.leaky_relu(F.conv2d(x, sd[f'to_plane_cnn.{i}.weight'], sd[f'to_plane_cnn.{i}.bias'], 1, 1), 0.01)
    x = F.interpolate(x, scale_factor=2.0, mode='bilinear', align_corners=True)
    x = F.conv2d(x, sd['to_plane_cnn.7.weight'], sd['to_plane_cnn.7.bias'], 1, 1)
    p = x.view(len(x), 3, -1, x.shape[-2], x.shape[-1])
    return torch.stack([torch.flip(p[:, 0], [2]), torch.flip(p[:, 1], [2]), torch.flip(p[:, 2], [2, 3])], 1)


def prenet(sd, x):
    w = sd['prenet.weight']
    return F.conv2d(x, w / math.sqrt(w.shape[1]), sd['prenet.bias'])


def forward(sd, x):
    """SegFormerSECC2PlaneBackbone.forward in the dtype of `sd` / `x` (float64 for the tests)."""
    return to_planes(sd, head(sd, mit_b0(sd, prenet(sd, x))))


def to64(sd, device='cpu'):
    return {k: (v.to(device, torch.float64) if v.is_floating_point() else v.to(device)) for k, v in sd.items()}


# ---- the library's launch sequence, restated from the architecture ----------------------------------------------------------------------
EMB = 256


def cop_of(cout):
    """Packed couts of an r3dp_mf_conv3d launch: cout rounded up to its cout tile (16, 32, 64 or 128)."""
    bn = 16 if cout <= 16 else 32 if cout <= 32 else 64 if cout <= 64 else 128
    return -(-cout // bn) * bn


def launch_plan(H, B, cin=9):
    """Every kernel launch of SegFormerSECC2PlaneBackbone.forward on [B, cin, H, H], as (tag, C entry point, the non-pointer arguments in C
    order), written from the architecture above (MiT-b0 stages, SegFormerHead, to_plane_cnn) rather than from the module's code.  The
    per-launch tests build their tables from it, and a test that records the module's calls holds it to what the module launches."""
    plan = []

    def add(tag, fn, *args):
        plan.append((tag, fn, tuple(args)))

    def gemm(tag, R, K, O, f32):
        add(tag, 'r3dp_mf_conv3d', K, 0, K, 1, 1, 1, R, 1, 1, 1, 0, O, cop_of(O), 0, O, 0, 0, int(f32), 0)

    def ln(tag, R, C, eps):
        add(tag, 'r3dp_sp_layernorm', R, C, eps, C)

    def patches(tag, h, C, k, s, p):
        add(tag, 'r3dp_sp_patches', B, h, h, C, k, s, p)
        return (h + 2 * p - k) // s + 1

    h = (H - 1) // 4 + 1
    add('embed', 'r3dp_sp_embed', B, cin, H, H)
    levels = []
    for s in range(4):
        C, st = EMBED[s], f's{s + 1}'
        if s > 0:
            h = patches(st + '.pe_patches', h, EMBED[s - 1], 3, 2, 1)
            gemm(st + '.pe', B * h * h, 9 * EMBED[s - 1], C, True)
        R = B * h * h
        ln(st + '.pe_norm', R, C, 1e-5)
        ln(st + '.norm1', R, C, 1e-6)
        for bi in range(2):
            gemm(st + '.q', R, C, C, False)
            if SR[s] > 1:
                hk = patches(st + '.sr_patches', h, C, SR[s], SR[s], 0)
                gemm(st + '.sr', B * hk * hk, SR[s] ** 2 * C, C, True)
                ln(st + '.sr_norm', B * hk * hk, C, 1e-5)
                gemm(st + '.kv', B * hk * hk, C, 2 * C, False)
                tk = hk * hk
            else:
                gemm(st + '.kv', R, C, 2 * C, False)
                tk = h * h
            add(st + '.attention', 'r3dp_sp_attention', C, 2 * C, B, h * h, tk, HEADS[s], 32 ** -0.5, C)
            gemm(st + '.proj', R, C, C, True)
            ln(st + '.norm2', R, C, 1e-6)
            gemm(st + '.fc1', R, C, 4 * C, False)
            add(st + '.dwconv', 'r3dp_sp_dwconv_gelu', B, h, h, 4 * C)
            gemm(st + '.fc2', R, 4 * C, C, True)
            ln(st + ('.norm1' if bi == 0 else '.norm'), R, C, 1e-6)
        levels.append(h)
    for i, hh in enumerate(levels):
        gemm(f'G{i + 1}', B * hh * hh, EMBED[i], EMB, True)
    h1 = levels[0]
    add('head_fuse', 'r3dp_sp_head_fuse', levels[0], levels[1], levels[2], levels[3], B)
    for i in (0, 2, 4):
        if h1 % 128 == 0:
            add(f'to_plane_cnn.{i}', 'r3dp_sr_tc_conv', B, 1, EMB, EMB, h1, h1, 3, 2)
        else:
            add(f'to_plane_cnn.{i}', 'r3dp_mf_conv3d', EMB, 0, EMB, B, 1, h1, h1, 1, 3, 3, 0, EMB, EMB, 0, EMB, 0, 0, 0, 0)
            add(f'to_plane_cnn.{i + 1}', 'r3dp_sp_leaky', B * h1 * h1 * EMB, 0.01)
    add('upsample', 'r3dp_sp_upsample2_flip', B, h1, h1, EMB)
    for O, c0 in ((64, 0), (32, 64)):
        add(f'to_plane_cnn.7[{c0}:{c0 + O}]', 'r3dp_mf_conv3d', EMB, 0, EMB, B, 1, 2 * h1, 2 * h1, 1, 3, 3, 0, O, cop_of(O), 0, 96, c0, 0, 1, 0)
    return plan


# ---- shims for importing the reference's segformer.py without timm / mmcv --------------------------------------------------------------
class _DropPath(nn.Module):
    def __init__(self, drop_prob=None):
        super().__init__()
        self.drop_prob = drop_prob

    def forward(self, x):                  # eval only
        return x


class _ConvModule(nn.Module):
    """mmcv.cnn.ConvModule as SegFormerHead builds it (1x1, norm_cfg BN): bias='auto' gives a bias-free conv before the norm; children
    named `conv`, `bn`, `activate` (ReLU), applied in that order."""
    def __init__(self, in_channels, out_channels, kernel_size, norm_cfg=None, **_):
        super().__init__()
        self.conv = nn.Conv2d(in_channels, out_channels, kernel_size, bias=norm_cfg is None)
        self.bn = nn.BatchNorm2d(out_channels) if norm_cfg is not None else None
        self.activate = nn.ReLU()

    def forward(self, x):
        x = self.conv(x)
        if self.bn is not None:
            x = self.bn(x)
        return self.activate(x)


def install_shims():
    """Put minimal timm / mmcv modules in sys.modules (written for these tests; only what segformer.py:14-18 imports)."""
    def mod(name, **attrs):
        m = sys.modules.get(name) or types.ModuleType(name)
        for k, v in attrs.items():
            setattr(m, k, v)
        sys.modules[name] = m
        return m
    mod('timm')
    mod('timm.models')
    mod('timm.models.layers', DropPath=_DropPath, to_2tuple=lambda x: x if isinstance(x, tuple) else (x, x),
        trunc_normal_=lambda t, std=1.0, **_: nn.init.normal_(t, 0.0, std))
    mod('timm.models.registry', register_model=lambda f: f)
    mod('timm.models.vision_transformer', _cfg=lambda **k: dict(k))
    mod('mmcv')
    mod('mmcv.cnn', ConvModule=_ConvModule)
    sys.modules.setdefault('imageio', types.ModuleType('imageio'))


def reference_class(ref_root):
    """The reference's SegFormerSECC2PlaneBackbone, imported from the checkout at `ref_root` behind the shims.  mit_b0's constructor loads
    checkpoints/pretrained_ckpts/mit_b0.pth with strict=False; torch.load returns {} for that path while the class is built."""
    install_shims()
    if ref_root not in sys.path:
        sys.path.insert(0, ref_root)
    from modules.real3d import segformer                       # noqa: E402  (reference)
    orig = torch.load

    def build(*a, **k):
        def fake_load(f, *aa, **kk):
            if isinstance(f, str) and f.endswith('mit_b0.pth'):
                return {}
            return orig(f, *aa, **kk)
        torch.load = fake_load
        try:
            return segformer.SegFormerSECC2PlaneBackbone(*a, **k)
        finally:
            torch.load = orig
    return build
