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

import torch
import torch.nn.functional as F

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
