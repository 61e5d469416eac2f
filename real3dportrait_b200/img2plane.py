"""Img2PlaneModel (modules/img2plane/img2plane_model.py:12-81) on libr3dp_b200: the canonical plane backbone that `cal_cano_plane` runs once
per clip on the source head image (modules/real3d/secc_img2plane.py:50-62).  Its planes are the `cano_planes` of FrameEngine.begin_planes.

The module keeps the reference's constructor and state_dict (keys and shapes) and is a drop-in for it; the parameters are plain containers
and every forward runs the r3dp_ip_* kernels, r3dp_mf_conv3d (every convolution and token GEMM; strided and dilated convolutions on
r3dp_sp_patches_dil rows), r3dp_sp_layernorm, r3dp_sp_dwconv_gelu and r3dp_sp_leaky.  Network (H = input size, square, H % 16 == 0):
  - DeepLabV3 (deeplabv3/decoders/my_model.py): ResNet-34 at output stride 8 (layer3 / layer4: every conv stride 1, dilation 2 / 4,
    deeplabv3/encoders/_utils.py:40-51), ASPP (1x1, 3x3 at rates 12/24/36, image pooling; no BN, ReLU) and a bias-free 3x3 conv -> H/8;
  - LowResolutionViT (segformer/models.py:11-88): 3x3/2 patch embed to 1024, `num_blocks` Blocks (4 heads of 256), PixelShuffle(2),
    two (bilinear x2, 3x3 conv, ReLU), a 3x3 conv to 96 -> H/2;
  - HighResoEncoder (simple_encoders/high_resolution_encoder.py): 7x7/2 conv, four 3x3 convs + LeakyReLU(0.01), a 3x3 conv -> H/2;
  - TriplanePredictorViT (segformer/models.py:91-183): convs on cat[low, high], 3x3/2 patch embed, Blocks with sr_ratio 2, PixelShuffle(2),
    convs on cat[shuffled, low] -> 96 channels at H/2, viewed as 3 planes of 32 and flipped (img2plane_model.py:72-81).
The two concatenations are channel slices of one NHWC buffer of 448 channels: [shuffled 256 | low 96 | high 96].
Weights are folded on the host in float64 and packed once per parameter set (refolded after load_state_dict / .to()): every eval BatchNorm
of the ResNet encoder goes into its conv.  Precision (`tc`): fp16 GEMM operands with fp32 accumulation; the residual stream, LayerNorm
statistics, softmax and GELU in fp32.
"""
from __future__ import annotations

import ctypes
from typing import Optional

import torch
import torch.nn as nn

from . import _capi as capi, conv3d, sr_tc
from .conv3d import pack_gemm, pack_taps
from .prepared import PreparedMixin
from .renderer import PlanesCL
from .secc2plane import _conv_rows

F16 = torch.float16
DIM = 1024                          # both ViTs' embed dim (segformer/models.py:19,103)
HEADS = 4                           # head_dim 256
MLP = 2 * DIM                       # mlp_ratio 2
LAYERS = [3, 4, 6, 3]               # ResNet-34 (deeplabv3/encoders/resnet.py:136-144)
WIDTHS = [64, 128, 256, 512]
DILATION = [1, 1, 2, 4]             # output stride 8: layer3 dilation 2, layer4 dilation 4 (encoders/_base.py:41-65)
RATES = (12, 24, 36)                # ASPP atrous rates (my_decoder.py:41)
#: img2plane_backbone_scale -> (LowResolutionViT blocks, TriplanePredictorViT blocks) (segformer/models.py:21-28,105-110)
SCALES = {'small': (2, 1), 'standard': (5, 1), 'large': (10, 3)}


# ---- parameter containers with the reference's names -------------------------------------------------------------------------------------
class _BasicBlock(nn.Module):
    """torchvision BasicBlock (conv3x3 -> BN -> ReLU -> conv3x3 -> BN, + identity or downsample, ReLU)."""
    def __init__(self, cin, c, down):
        super().__init__()
        self.conv1 = nn.Conv2d(cin, c, 3, 1, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(c)
        self.conv2 = nn.Conv2d(c, c, 3, 1, 1, bias=False)
        self.bn2 = nn.BatchNorm2d(c)
        if down:
            self.downsample = nn.Sequential(nn.Conv2d(cin, c, 1, bias=False), nn.BatchNorm2d(c))


class _ResNet34Encoder(nn.Module):
    def __init__(self, cin):
        super().__init__()
        self.conv1 = nn.Conv2d(cin, 64, 7, 2, 3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        prev = 64
        for i, (n, c) in enumerate(zip(LAYERS, WIDTHS)):
            setattr(self, f'layer{i + 1}', nn.Sequential(*[_BasicBlock(prev if b == 0 else c, c, b == 0 and i > 0) for b in range(n)]))
            prev = c


class _ASPP(nn.Module):
    def __init__(self, cin, c=256):
        super().__init__()
        self.convs = nn.ModuleList([nn.Sequential(nn.Conv2d(cin, c, 1, bias=False), nn.ReLU())] +
                                   [nn.Sequential(nn.Conv2d(cin, c, 3, padding=r, dilation=r, bias=False), nn.ReLU()) for r in RATES] +
                                   [nn.Sequential(nn.AdaptiveAvgPool2d(1), nn.Conv2d(cin, c, 1, bias=False), nn.ReLU())])
        self.project = nn.Sequential(nn.Conv2d(5 * c, c, 1, bias=False), nn.ReLU(), nn.Dropout(0.5))


class _DeepLabV3(nn.Module):
    def __init__(self, cin):
        super().__init__()
        self.encoder = _ResNet34Encoder(cin)
        self.decoder = nn.Sequential(_ASPP(512), nn.Conv2d(256, 256, 3, padding=1, bias=False))


class _PatchEmbed(nn.Module):
    def __init__(self, cin):
        super().__init__()
        self.proj = nn.Conv2d(cin, DIM, 3, 2, 1)
        self.norm = nn.LayerNorm(DIM)


class _Attention(nn.Module):
    def __init__(self, sr):
        super().__init__()
        self.q = nn.Linear(DIM, DIM)
        self.kv = nn.Linear(DIM, 2 * DIM)
        self.proj = nn.Linear(DIM, DIM)
        if sr > 1:
            self.sr = nn.Conv2d(DIM, DIM, sr, sr)
            self.norm = nn.LayerNorm(DIM)


class _DW(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.dwconv = nn.Conv2d(c, c, 3, 1, 1, groups=c)


class _Mlp(nn.Module):
    def __init__(self):
        super().__init__()
        self.fc1 = nn.Linear(DIM, MLP)
        self.dwconv = _DW(MLP)
        self.fc2 = nn.Linear(MLP, DIM)


class _Block(nn.Module):
    def __init__(self, sr):
        super().__init__()
        self.norm1 = nn.LayerNorm(DIM)                             # nn.LayerNorm's default eps 1e-5 (segformer/base.py:127-137)
        self.attn = _Attention(sr)
        self.norm2 = nn.LayerNorm(DIM)
        self.mlp = _Mlp()


class _LowResolutionViT(nn.Module):
    def __init__(self, nblocks):
        super().__init__()
        self.num_blocks = nblocks
        self.patch_embed = _PatchEmbed(256)
        for i in range(1, nblocks + 1):
            setattr(self, f'block{i}', _Block(1))
        self.conv_after_upsample1 = nn.Conv2d(256, 128, 3, 1, 1)
        self.conv_after_upsample2 = nn.Conv2d(128, 128, 3, 1, 1)
        self.final_conv = nn.Conv2d(128, 96, 3, 1, 1)


class _HighResoEncoder(nn.Module):
    def __init__(self, cin):
        super().__init__()
        self.first = nn.Conv2d(cin, 64, 7, 2, 3)
        self.conv_layers = nn.Sequential(nn.Conv2d(64, 96, 3, 1, 1), nn.LeakyReLU(0.01), nn.Conv2d(96, 96, 3, 1, 1), nn.LeakyReLU(0.01),
                                         nn.Conv2d(96, 96, 3, 1, 1), nn.LeakyReLU(0.01), nn.Conv2d(96, 96, 3, 1, 1), nn.LeakyReLU(0.01))
        self.final = nn.Conv2d(96, 96, 3, 1, 1)


class _TriplanePredictorViT(nn.Module):
    def __init__(self, nblocks, out_channels):
        super().__init__()
        self.num_blocks = nblocks
        self.first_conv = nn.Conv2d(192, 256, 3, 1, 1)
        self.second_conv = nn.Conv2d(256, 128, 3, 1, 1)
        self.patch_embed = _PatchEmbed(128)
        for i in range(1, nblocks + 1):
            setattr(self, f'block{i}', _Block(2))
        self.first_conv_after_cat = nn.Conv2d(352, 256, 3, 1, 1)
        self.second_conv_after_cat = nn.Conv2d(256, 128, 3, 1, 1)
        self.third_conv_after_cat = nn.Conv2d(128, 128, 3, 1, 1)
        self.final_conv = nn.Conv2d(128, out_channels, 3, 1, 1)


# ---- host-side folding (float64) ---------------------------------------------------------------------------------------------------------
def fold_conv_bn(conv_w: torch.Tensor, bn: nn.BatchNorm2d):
    """bias-free conv [O,I,k,k] -> eval BatchNorm  ->  (W float64 [O,I,k,k] scaled by s, bias float64 [O]), s = gamma / sqrt(var + eps)."""
    s = bn.weight.detach().double() / torch.sqrt(bn.running_var.detach().double() + bn.eps)
    bias = bn.bias.detach().double() - bn.running_mean.detach().double() * s
    return conv_w.detach().double() * s[:, None, None, None], bias


class _Conv:
    """One convolution's packed weights.  Stride-1 undilated 3x3 convs run as r3dp_mf_conv3d (1,3,3) taps, or on r3dp_sr_tc_conv where it
    applies (128 or 256 outputs, a dense input of a multiple of 64 channels, W % 128 == 0: packed for both, chosen per launch); 1x1 stride-1
    convs as the GEMM; every other conv (7x7/2 stems, 3x3/2, dilated 3x3, 1x1/2, the 2x2/2 `sr`) as r3dp_sp_patches_dil rows (K padded to a
    multiple of 32) times the GEMM."""

    def __init__(self, w, b, k, s, p, d, dev):
        self.k, self.s, self.p, self.d = k, s, p, d
        O, I = w.shape[:2]
        self.cin, self.cout = I, O
        if b is None:
            b = torch.zeros(O, dtype=torch.float64, device=w.device)
        self.box = k == 3 and s == 1 and d == 1 and p == 1
        self.gemm = k == 1 and s == 1
        self.tc = None
        if self.box:
            self.pk = pack_taps(w, b, dev)
            if O in (128, 256) and I % 64 == 0:
                self.tc = sr_tc.pack_plain_weights(w.to(dev)[None], b.to(dev), I)[0]
        elif self.gemm:
            self.pk = pack_gemm(w[:, :, 0, 0], b, dev)
        else:
            rows = _conv_rows(w)
            self.ldy = conv3d.ceil32(rows.shape[1])
            wp = torch.zeros(O, self.ldy, dtype=torch.float64, device=w.device)
            wp[:, :rows.shape[1]] = rows
            self.pk = pack_gemm(wp, b, dev)

    def out_size(self, h: int) -> int:
        return (h + 2 * self.p - self.d * (self.k - 1) - 1) // self.s + 1


class Img2PlaneModel(PreparedMixin, nn.Module):
    """Img2PlaneModel(out_channels=96, hp=None) (img2plane_model.py:12-35) on sm_90a kernels, for img2plane_input_mode 'rgb',
    triplane_feature_type 'triplane', triplane_depth 1 and img2plane_backbone_scale 'small' | 'standard' | 'large' (read from hp).

    forward(x [B,3,H,H]) -> [B,3,32,H/2,H/2], the reference's flipped planes (a view of channels-last data);
    planes_cl(img [B,3,H,H], out=None) -> PlanesCL('hwpc') [B,H/2,H/2,3,32]: the same values in the render's layout (with B = 1 the
    per-clip canonical set, frame stride 0), written into `out` when given (a contiguous fp32 [B,H/2,H/2,3,32] tensor)."""

    def __init__(self, out_channels: int = 96, hp: Optional[dict] = None):
        super().__init__()
        hp = dict(hp or {})
        mode = hp.get('img2plane_input_mode', 'rgb')
        if mode != 'rgb':
            raise NotImplementedError(f'Img2PlaneModel: only img2plane_input_mode="rgb" (the released configuration) is built, got {mode!r}')
        ftype = hp.get('triplane_feature_type', 'triplane')
        if ftype != 'triplane':
            raise NotImplementedError(f'Img2PlaneModel: only triplane_feature_type="triplane" is built, got {ftype!r}')
        depth = hp.get('triplane_depth', 1)
        if depth != 1:
            raise NotImplementedError(f'Img2PlaneModel: only triplane_depth=1 is built, got {depth!r}')
        scale = hp.get('img2plane_backbone_scale', 'standard')
        if scale not in SCALES:
            raise NotImplementedError(f'Img2PlaneModel: img2plane_backbone_scale must be one of {sorted(SCALES)}, got {scale!r}')
        if out_channels != 96:
            raise NotImplementedError(f'Img2PlaneModel: only out_channels=96 (tri-planes of 32 channels) is built, got {out_channels}')
        self.hparams = hp
        self.input_mode, self.backbone_scale = mode, scale
        nlow, ntri = SCALES[scale]
        cin = 3 + 2                                                     # rgb + the two coordinate channels
        self.low_reso_encoder = _DeepLabV3(cin)
        self.high_reso_encoder = _HighResoEncoder(cin)
        self.low_reso_vit = _LowResolutionViT(nlow)
        self.triplane_predictor_vit = _TriplanePredictorViT(ntri, out_channels)

    def _prepared(self):
        return self.prepared('weights', self._build)

    def _build(self):
        enc = self.low_reso_encoder.encoder
        dev = capi.cuda_device(enc.conv1.weight)
        d = lambda t: None if t is None else t.detach().double()           # noqa: E731
        f32 = lambda t: t.detach().to(dev, torch.float32).contiguous()     # noqa: E731

        def stem_w(w):                                                      # the 5 input channels padded to the packed input's 8
            wp = torch.zeros(w.shape[0], 8, *w.shape[2:], dtype=torch.float64, device=w.device)
            wp[:, :w.shape[1]] = w
            return wp

        def conv(m, k=3, s=1, p=1, dil=1):
            return _Conv(d(m.weight), d(m.bias), k, s, p, dil, dev)

        P = {}
        w, b = fold_conv_bn(enc.conv1.weight, enc.bn1)
        P['stem'] = _Conv(stem_w(w), b, 7, 2, 3, 1, dev)
        layers = []
        for i in range(4):
            dil, blocks = DILATION[i], []
            for bi, blk in enumerate(getattr(enc, f'layer{i + 1}')):
                s = 2 if (i == 1 and bi == 0) else 1                        # layer2's first block; layer3/4 strides became dilations
                w1, b1 = fold_conv_bn(blk.conv1.weight, blk.bn1)
                w2, b2 = fold_conv_bn(blk.conv2.weight, blk.bn2)
                e = {'c1': _Conv(w1, b1, 3, s, dil, dil, dev), 'c2': _Conv(w2, b2, 3, 1, dil, dil, dev)}
                if hasattr(blk, 'downsample'):
                    wd, bd = fold_conv_bn(blk.downsample[0].weight, blk.downsample[1])
                    e['down'] = _Conv(wd, bd, 1, s, 0, 1, dev)
                blocks.append(e)
            layers.append(blocks)
        P['layers'] = layers
        aspp, dec_conv = self.low_reso_encoder.decoder[0], self.low_reso_encoder.decoder[1]
        P['aspp0'] = conv(aspp.convs[0][0], 1, 1, 0)
        P['aspp_r'] = [conv(aspp.convs[i + 1][0], 3, 1, r, r) for i, r in enumerate(RATES)]
        P['aspp_pool'] = conv(aspp.convs[4][1], 1, 1, 0)
        P['aspp_proj'] = conv(aspp.project[0], 1, 1, 0)
        P['dec'] = conv(dec_conv)
        ln = lambda m: (f32(m.weight), f32(m.bias), float(m.eps))           # noqa: E731
        lin = lambda m: pack_gemm(d(m.weight), d(m.bias), dev)             # noqa: E731

        def vit(v, sr):
            blocks = []
            for i in range(1, v.num_blocks + 1):
                blk = getattr(v, f'block{i}')
                at = blk.attn
                e = {'norm1': ln(blk.norm1), 'norm2': ln(blk.norm2), 'q': lin(at.q), 'kv': lin(at.kv), 'proj': lin(at.proj),
                     'fc1': lin(blk.mlp.fc1), 'fc2': lin(blk.mlp.fc2),
                     'dw': (f32(blk.mlp.dwconv.dwconv.weight.reshape(-1, 9)), f32(blk.mlp.dwconv.dwconv.bias))}
                if sr > 1:
                    e['sr'] = conv(at.sr, sr, sr, 0)
                    e['sr_norm'] = ln(at.norm)
                blocks.append(e)
            return {'pe': conv(v.patch_embed.proj, 3, 2, 1), 'pe_norm': ln(v.patch_embed.norm), 'blocks': blocks}

        lv = self.low_reso_vit
        P['low'] = vit(lv, 1)
        P['low_c1'], P['low_c2'], P['low_final'] = conv(lv.conv_after_upsample1), conv(lv.conv_after_upsample2), conv(lv.final_conv)
        he = self.high_reso_encoder
        P['high_first'] = _Conv(stem_w(d(he.first.weight)), d(he.first.bias), 7, 2, 3, 1, dev)
        P['high'] = [conv(he.conv_layers[i]) for i in (0, 2, 4, 6)] + [conv(he.final)]
        tv = self.triplane_predictor_vit
        P['tri'] = vit(tv, 2)
        P['tri_pre'] = [conv(tv.first_conv), conv(tv.second_conv)]
        P['tri_post'] = [conv(tv.first_conv_after_cat), conv(tv.second_conv_after_cat), conv(tv.third_conv_after_cat)]
        P['tri_final'] = conv(tv.final_conv)
        return P

    # ---- input checks ------------------------------------------------------------------------------------------------------------------
    @staticmethod
    def _check_image(x: torch.Tensor, what: str) -> torch.Tensor:
        if x.ndim != 4 or x.shape[1] != 3:
            raise ValueError(f'{what}: expected [B,3,H,W] rgb, got {tuple(x.shape)}')
        H, W = x.shape[2:]
        if H != W:
            raise ValueError(f'{what}: the input must be square (LowResolutionViT passes H as the width), got {H}x{W}')
        if H % 16 or H < 16:
            raise ValueError(f'{what}: H must be a positive multiple of 16, got {H}')
        if not x.is_cuda:
            raise RuntimeError('real3dportrait_b200 runs on CUDA tensors only (no CPU fallback); got a CPU tensor')
        return capi.f32(x)

    # ---- public interface --------------------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, x: torch.Tensor, cond=None) -> torch.Tensor:
        """x [B,3,H,H] -> planes [B,3,32,H/2,H/2] (img2plane_model.py:37-82)."""
        if cond is not None:
            raise NotImplementedError('Img2PlaneModel: cond is read only by the alpha / camera input modes, which are not built')
        out = self._run(self._check_image(x, 'Img2PlaneModel.forward'))
        return out.permute(0, 3, 4, 1, 2)                           # [B,H,W,3,C] -> [B,3,C,H,W] view (channels-last producer layout)

    @torch.no_grad()
    def planes_cl(self, img: torch.Tensor, out: Optional[torch.Tensor] = None) -> PlanesCL:
        """img [B,3,H,H] -> PlanesCL('hwpc') [B,H/2,H/2,3,32] fp32, the values forward(img) returns; written into `out` when given."""
        return PlanesCL(self._run(self._check_image(img, 'Img2PlaneModel.planes_cl'), out), 'hwpc')

    # ---- the launch sequence -----------------------------------------------------------------------------------------------------------
    def _run(self, x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        P, L, st, dev = self._prepared(), capi.lib(), capi.stream(), x.device
        B, _, H, _ = x.shape
        H2 = H // 2
        if out is None:
            out = torch.empty(B, H2, H2, 3, 32, device=dev)
        elif tuple(out.shape) != (B, H2, H2, 3, 32) or out.dtype != torch.float32 or not out.is_contiguous() or out.device != dev:
            raise ValueError(f'planes_cl: out must be a contiguous fp32 [{B},{H2},{H2},3,32] tensor on {dev}')
        ptr = capi.ptr

        def at(t, halves=0):                                        # a device pointer into an fp16 buffer, `halves` elements in
            return ctypes.c_void_p(t.data_ptr() + 2 * halves)

        def gemm(a, pk, relu=False, out_f32=False):                 # a [rows, K] fp16 -> [rows, cout]
            rows, K = a.shape
            y = torch.empty(rows, pk.cout, device=dev, dtype=torch.float32 if out_f32 else F16)
            conv3d.launch(pk, a, K, 0, K, (1, 1, rows, 1), (1, 1, 1), y, pk.cout, relu=int(relu), stream=st)
            return y

        def conv(xp, xs, h, cv, act=None, res=None, y=None, ys=None, yc0=0, out_f32=False, src=None):
            """cv on x [B,h,h,cv.cin] (pixel stride xs, at pointer xp; `src` the dense tensor itself for the patch rows) -> [B,ho,ho,cout].
            act: None, 'relu' or 'leaky' (nn.LeakyReLU(0.01), only into a tensor of its own)."""
            ho = cv.out_size(h)
            own = y is None
            if cv.tc is not None and xs == cv.cin and h % 128 == 0 and own and res is None and not out_f32:
                # r3dp_sr_tc_conv (tiles of 128-pixel rows) on the dense input; epilogue act 3 = ReLU, 2 = LeakyReLU(0.01)
                return sr_tc.conv_plain(src, (cv.tc, cv.pk.bias, 3), {None: 0, 'leaky': 2, 'relu': 3}[act]), ho
            if own:
                y = torch.empty(B, ho, ho, cv.cout, device=dev, dtype=torch.float32 if out_f32 else F16)
                ys = cv.cout
            assert act != 'leaky' or (own and not out_f32)
            relu = int(act == 'relu')
            if cv.box:
                conv3d.launch(cv.pk, xp, xs, 0, cv.cin, (B, 1, h, h), (1, 3, 3), y, ys, yc0, relu=relu, res=res, stream=st)
            elif cv.gemm:
                conv3d.launch(cv.pk, xp, xs, 0, cv.cin, (1, 1, B * h * h, 1), (1, 1, 1), y, ys, yc0, relu=relu, res=res, stream=st)
            else:
                assert src is not None and xs == src.shape[-1] == cv.cin
                pt = torch.empty(B * ho * ho, cv.ldy, device=dev, dtype=F16)
                capi.check(L.r3dp_sp_patches_dil(ptr(src, F16), B, h, h, cv.cin, cv.k, cv.s, cv.p, cv.d, ptr(pt, F16), cv.ldy, st))
                conv3d.launch(cv.pk, pt, cv.ldy, 0, cv.ldy, (1, 1, B * ho * ho, 1), (1, 1, 1), y, ys, yc0, relu=relu, res=res, stream=st)
            if act == 'leaky':
                capi.check(L.r3dp_sp_leaky(ptr(y, F16), y.numel(), 0.01, st))
            return y, ho

        def dense(t, cv, h, **kw):                                  # conv on a dense NHWC fp16 tensor
            return conv(ptr(t, F16), t.shape[-1], h, cv, src=t, **kw)

        def leaky(t, slope):
            capi.check(L.r3dp_sp_leaky(ptr(t, F16), t.numel(), slope, st))

        def layernorm(xv, t, R, p, xo=None, yf=None, yh=None):
            g, b, eps = p
            capi.check(L.r3dp_sp_layernorm(ptr(xv), ptr(t), R, DIM, ptr(g), ptr(b), eps, ptr(xo), ptr(yf), ptr(yh, F16), DIM, st))

        def vit(V, src, h, sr):
            """patch embed + Blocks on src [B,h,h,C] -> (xres, t, hv): the residual stream before the last block's MLP add, and that add."""
            t0, hv = dense(src, V['pe'], h, out_f32=True)
            R = B * hv * hv
            xres = torch.empty(R, DIM, device=dev)
            layernorm(t0, None, R, V['pe_norm'], yf=xres)
            del t0
            a = torch.empty(R, DIM, device=dev, dtype=F16)
            layernorm(xres, None, R, V['blocks'][0]['norm1'], yh=a)
            for bi, bw in enumerate(V['blocks']):
                q = gemm(a, bw['q'])
                if sr > 1:
                    r, hk = dense(a.view(B, hv, hv, DIM), bw['sr'], hv, out_f32=True)
                    a2 = torch.empty(B * hk * hk, DIM, device=dev, dtype=F16)
                    layernorm(r, None, B * hk * hk, bw['sr_norm'], yh=a2)
                    del r
                    kv, tk = gemm(a2, bw['kv']), hk * hk
                    del a2
                else:
                    kv, tk = gemm(a, bw['kv']), hv * hv
                o = torch.empty(R, DIM, device=dev, dtype=F16)
                with capi.region('img2plane.attention'):
                    capi.check(L.r3dp_ip_attention(ptr(q, F16), DIM, ptr(kv, F16), 2 * DIM, B, hv * hv, tk, HEADS, 1.0 / 16.0, ptr(o, F16), DIM, st))
                del q, kv
                t = gemm(o, bw['proj'], out_f32=True)
                del o
                layernorm(xres, t, R, bw['norm2'], xo=xres, yh=a)
                f1 = gemm(a, bw['fc1'])
                f2 = torch.empty_like(f1)
                capi.check(L.r3dp_sp_dwconv_gelu(ptr(f1, F16), B, hv, hv, MLP, ptr(bw['dw'][0]), ptr(bw['dw'][1]), ptr(f2, F16), st))
                del f1
                t = gemm(f2, bw['fc2'], out_f32=True)
                del f2
                if bi + 1 < len(V['blocks']):
                    layernorm(xres, t, R, V['blocks'][bi + 1]['norm1'], xo=xres, yh=a)
            return xres, t, hv

        with capi.region('img2plane'):
            xin = torch.empty(B, H, H, 8, device=dev, dtype=F16)
            capi.check(L.r3dp_ip_input(ptr(x), B, H, H, ptr(xin, F16), st))
            # the two 7x7/2 stems read the same patch rows
            with capi.region('img2plane.encoder'):
                cs = P['stem']
                h1 = cs.out_size(H)
                pt = torch.empty(B * h1 * h1, cs.ldy, device=dev, dtype=F16)
                capi.check(L.r3dp_sp_patches_dil(ptr(xin, F16), B, H, H, 8, 7, 2, 3, 1, ptr(pt, F16), cs.ldy, st))
                del xin
                e = gemm(pt, cs.pk, relu=True).view(B, h1, h1, 64)
                hi = gemm(pt, P['high_first'].pk).view(B, h1, h1, 64)
                del pt
                h = (h1 - 1) // 2 + 1
                y = torch.empty(B, h, h, 64, device=dev, dtype=F16)
                capi.check(L.r3dp_ip_maxpool(ptr(e, F16), B, h1, h1, 64, ptr(y, F16), st))
                del e
                for blocks in P['layers']:
                    for bw in blocks:
                        t, ho = dense(y, bw['c1'], h, act='relu')
                        res = dense(y, bw['down'], h)[0] if 'down' in bw else y
                        z, _ = dense(t, bw['c2'], ho, res=res)
                        leaky(z, 0.0)                               # BasicBlock's ReLU after the residual add
                        del t, res
                        y, h = z, ho
            with capi.region('img2plane.aspp'):
                h8 = h
                cat = torch.empty(B, h8, h8, 1280, device=dev, dtype=F16)
                dense(y, P['aspp0'], h8, act='relu', y=cat, ys=1280, yc0=0)
                for i, cv in enumerate(P['aspp_r']):
                    dense(y, cv, h8, act='relu', y=cat, ys=1280, yc0=256 * (i + 1))
                mean = torch.empty(B, 512, device=dev, dtype=F16)
                capi.check(L.r3dp_ip_channel_mean(ptr(y, F16), B, h8 * h8, 512, ptr(mean, F16), st))
                pooled = gemm(mean, P['aspp_pool'].pk, relu=True)
                capi.check(L.r3dp_ip_broadcast(ptr(pooled, F16), B, h8 * h8, 256, ptr(cat, F16), 1280, 1024, st))
                del y, mean, pooled
                proj, _ = dense(cat, P['aspp_proj'], h8, act='relu')
                del cat
                dec, _ = dense(proj, P['dec'], h8)
                del proj
            # cat448 = [pixel-shuffled tokens 256 | low 96 | high 96]: first_conv reads [256, 448), first_conv_after_cat [0, 352)
            cat = torch.empty(B, H2, H2, 448, device=dev, dtype=F16)
            with capi.region('img2plane.low_vit'):
                xres, t, hv = vit(P['low'], dec, h8, 1)
                del dec
                ps = torch.empty(B, 2 * hv, 2 * hv, 256, device=dev, dtype=F16)
                capi.check(L.r3dp_ip_pixel_shuffle(ptr(xres), ptr(t), B, hv, hv, 256, ptr(ps, F16), 256, 0, st))
                del xres, t
                hu = 2 * hv
                for cv in (P['low_c1'], P['low_c2']):
                    up = torch.empty(B, 2 * hu, 2 * hu, ps.shape[-1], device=dev, dtype=F16)
                    capi.check(L.r3dp_ip_upsample2(ptr(ps, F16), B, hu, hu, ps.shape[-1], ptr(up, F16), st))
                    hu *= 2
                    ps, _ = dense(up, cv, hu, act='relu')
                    del up
                dense(ps, P['low_final'], hu, y=cat, ys=448, yc0=256)
                del ps
            with capi.region('img2plane.high'):
                z = hi
                for cv in P['high'][:-1]:
                    z, _ = dense(z, cv, H2, act='leaky')
                dense(z, P['high'][-1], H2, y=cat, ys=448, yc0=352)
                del z, hi
            with capi.region('img2plane.tri_vit'):
                z, _ = conv(at(cat, 256), 448, H2, P['tri_pre'][0], act='leaky')
                z, _ = dense(z, P['tri_pre'][1], H2, act='leaky')
                xres, t, hv = vit(P['tri'], z, H2, 2)
                del z
                capi.check(L.r3dp_ip_pixel_shuffle(ptr(xres), ptr(t), B, hv, hv, 256, ptr(cat, F16), 448, 0, st))
                del xres, t
                z, _ = conv(at(cat), 448, H2, P['tri_post'][0], act='leaky')
                del cat
                for cv in P['tri_post'][1:]:
                    z, _ = dense(z, cv, H2, act='leaky')
                yf, _ = dense(z, P['tri_final'], H2, out_f32=True)
                del z
                capi.check(L.r3dp_ip_flip_hwpc(ptr(yf), B, H2, H2, ptr(out), st))
        return out
