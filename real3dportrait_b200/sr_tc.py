"""Tensor-core execution of SuperresolutionHybrid8XDC.forward (superresolution.py:348-359): the same layers as the
fp32 modules in superresolution.py, run as wgmma implicit GEMMs (csrc/sr_tc.cu) on NHWC fp16 activations with fp32
accumulation.  Weights are folded (modulated + demodulated) in fp32 per sample, exactly as the reference does, and only
then rounded to fp16.  Stated tolerance vs the fp32 reference: see tests/test_gpu_parity.py::test_sr_full_tc."""
from __future__ import annotations

from typing import Optional

import torch

from . import _capi as capi

F16 = torch.float16
#: the operations whose entry points are not named r3dp_sr_tc_<op> / r3dp_sr_tcx_<op>: op -> (fp16 operands, split operands)
_ENTRY = {'last_layer': ('r3dp_sr_tc_last_layer_ex', 'r3dp_sr_tcx_last_layer'), 'alpha_cat': ('r3dp_sr_alpha_cat_ex', 'r3dp_sr_tcx_alpha_cat_ex'),
          'cat3': ('r3dp_sr_cat3', 'r3dp_sr_tcx_cat3'), 'alpha_mix': ('r3dp_sr_alpha_mix', 'r3dp_sr_tcx_alpha_mix')}


def _fn(op: str, split: bool):
    """C entry point of operation `op` for fp16 operands, or for split [hi | lo] fp16 operands (sr_mode='tc_exact')."""
    return getattr(capi.lib(), _ENTRY.get(op, ('r3dp_sr_tc_' + op, 'r3dp_sr_tcx_' + op))[bool(split)])


def activation(N: int, H: int, W: int, C: int, split: bool, device) -> torch.Tensor:
    """An fp16 NHWC activation of C channels: [N,H,W,C], or [N,H,W,2C] = [hi | lo] halves when split."""
    return torch.empty(N, H, W, 2 * C if split else C, device=device, dtype=F16)


def _pack(layer, w_lat: torch.Tensor, split: bool = False) -> torch.Tensor:
    """SynthesisLayer -> packed fp16 weights [Nw,9,O,Ipad] ([Nw,9,O,2*Ipad] = [hi | lo] of w * 2^10 when split)."""
    wf = layer.folded_weight(w_lat)                                  # [Nw,O,I,3,3] fp32
    Nw, O, I = wf.shape[:3]
    Ip = (I + 63) // 64 * 64
    out = torch.empty(Nw, 9, O, Ip * (2 if split else 1), device=wf.device, dtype=torch.float16)
    capi.check(_fn('pack_weights', split)(capi.ptr(wf), Nw, O, I, capi.ptr(out, torch.float16), capi.stream()))
    return out


COMPOSE_MAX_CIN = 64      # up layers with at most this many input channels run through FIR-composed weights


def _pack_up_composed(layer_, w_lat: torch.Tensor, split: bool = False) -> torch.Tensor:
    """Up SynthesisLayer -> FIR-composed packed fp16 weights [Nw,36,O,Ipad] (4 output parities x 3x3 taps)."""
    wf = layer_.folded_weight(w_lat)
    Nw, O, I = wf.shape[:3]
    Ip = (I + 63) // 64 * 64
    out = torch.empty(Nw, 36, O, Ip * (2 if split else 1), device=wf.device, dtype=torch.float16)
    capi.check(_fn('pack_weights_up_composed', split)(capi.ptr(wf), Nw, O, I, capi.ptr(out, torch.float16), capi.stream()))
    return out


def pack_for(layer_, w_lat: torch.Tensor, split: bool = False) -> torch.Tensor:
    if layer_.up == 2 and layer_.in_channels <= COMPOSE_MAX_CIN:
        return _pack_up_composed(layer_, w_lat, split)
    return _pack(layer_, w_lat, split)


def layer(x16: torch.Tensor, lay, wp: torch.Tensor, up: int, split: bool = False) -> torch.Tensor:
    """x16 [N,H,W,Ipad] fp16 NHWC -> [N,H*up,W*up,O] fp16 NHWC (channel dims doubled = [hi | lo] halves when split)."""
    N, H, W, _ = x16.shape
    O, Nw = lay.out_channels, wp.shape[0]
    y = activation(N, H * up, W * up, O, split, x16.device)
    if up == 2 and wp.shape[1] == 36:                             # FIR-composed weights
        with capi.region('sr_conv'):
            capi.check(_fn('layer_up_composed', split)(capi.ptr(x16, torch.float16), capi.ptr(wp, torch.float16), capi.ptr(capi.f32(lay.bias)), N, Nw,
                                                       lay.in_channels, O, H, W, capi.ptr(y, torch.float16), capi.stream()))
        return y
    scratch = None
    if up == 2:
        scratch = torch.empty(_fn('scratch_bytes', split)(N, O, H, W), device=x16.device, dtype=torch.uint8)
    with capi.region('sr_conv'):
        capi.check(_fn('layer', split)(capi.ptr(x16, torch.float16), capi.ptr(wp, torch.float16), capi.ptr(capi.f32(lay.bias)), N, Nw,
                                       lay.in_channels, O, H, W, up, capi.ptr(y, torch.float16), capi.ptr(scratch, torch.uint8), capi.stream()))
    return y


def to_nhwc_f16(x: torch.Tensor, size: int, split: bool = False) -> torch.Tensor:
    """fp32 NCHW [N,C,h,w] -> (bilinear to size) -> NHWC fp16 [N,size,size,Cpad]."""
    x = capi.f32(x)
    N, Cc, h, w = x.shape
    y = activation(N, size, size, (Cc + 63) // 64 * 64, split, x.device)
    capi.check(_fn('input', split)(capi.ptr(x), N, Cc, h, w, size, capi.ptr(y, F16), capi.stream()))
    return y


def input_nhwc(x_nhwc: torch.Tensor, size: int, split: bool = False, rgb: bool = False):
    """to_nhwc_f16 of channels-last features [N,h,w,C] (the renderer's native output) -> (x, None); rgb: x_nhwc[..., :3] is the rgb
    image, its resize (fp32 NCHW [N,3,size,size]) rides in the same launch -> (x, rgb)."""
    xn = capi.f32(x_nhwc)
    N, h, w, Cc = xn.shape
    y = activation(N, size, size, (Cc + 63) // 64 * 64, split, xn.device)
    if not rgb:
        capi.check(_fn('input_nhwc', split)(capi.ptr(xn), N, Cc, h, w, size, capi.ptr(y, F16), capi.stream()))
        return y, None
    rgb0 = torch.empty(N, 3, size, size, device=xn.device)
    capi.check(capi.lib().r3dp_sr_tc_input_nhwc_rgb(capi.ptr(xn), N, Cc, h, w, size, capi.ptr(y, F16), capi.ptr(rgb0), int(split), capi.stream()))
    return y, rgb0


def layer_torgb(x16: torch.Tensor, blk, wp: torch.Tensor, wrgb: torch.Tensor, img: torch.Tensor, split: bool = False, noup: bool = False):
    """blk.conv1 + blk.torgb in one launch: x16 [N,H,W,Ipad] -> ([N,H,W,O], image fp32 [N,3,H,W] = ToRGB + img upsampled, or as is if noup)."""
    lay = blk.conv1
    N, H, W, _ = x16.shape
    y, out = activation(N, H, W, lay.out_channels, split, x16.device), torch.empty(N, 3, H, W, device=x16.device)
    with capi.region('sr_conv'):
        capi.check(_fn('layer_torgb_noup' if noup else 'layer_torgb', split)(
            capi.ptr(x16, F16), capi.ptr(wp, F16), capi.ptr(capi.f32(lay.bias)), capi.ptr(wrgb), capi.ptr(capi.f32(blk.torgb.bias)), capi.ptr(img),
            N, wp.shape[0], lay.in_channels, lay.out_channels, H, W, capi.ptr(y, F16), capi.ptr(out), capi.stream()))
    return y, out


def last_layer(x16: torch.Tensor, blk, wp: torch.Tensor, wrgb: torch.Tensor, img: Optional[torch.Tensor], clamp: bool = False,
               uint8: bool = False, split: bool = False) -> torch.Tensor:
    """layer_torgb without writing the activation: -> the image fp32 [N,3,H,W] (img None: no skip), clamped to [-1,1] with clamp; uint8:
    HWC frames [N,H,W,3] (the caller loop's conversion, inference/real3d_infer.py:515-519, fused)."""
    lay = blk.conv1
    N, H, W, _ = x16.shape
    out = torch.empty(N, H, W, 3, device=x16.device, dtype=torch.uint8) if uint8 else torch.empty(N, 3, H, W, device=x16.device)
    with capi.region('sr_conv'):
        capi.check(_fn('last_layer', split)(
            capi.ptr(x16, F16), capi.ptr(wp, F16), capi.ptr(capi.f32(lay.bias)), capi.ptr(wrgb), capi.ptr(capi.f32(blk.torgb.bias)), capi.ptr(img),
            N, wp.shape[0], lay.in_channels, H, W, None if uint8 else capi.ptr(out), capi.ptr(out, torch.uint8) if uint8 else None,
            int(clamp or uint8), capi.stream()))
    return out


def torgb(x16: torch.Tensor, wrgb: torch.Tensor, brgb: torch.Tensor, img: torch.Tensor, split: bool = False) -> torch.Tensor:
    """img + ToRGB(x16) at img's resolution: x16 [N,H,W,C], wrgb [Nw,3,C] and brgb [3] fp32, img fp32 [N,3,H,W] -> the same."""
    N, H, W, _ = x16.shape
    out = torch.empty(N, 3, H, W, device=x16.device)
    capi.check(_fn('torgb_ex', split)(capi.ptr(x16, F16), capi.ptr(wrgb), capi.ptr(brgb), capi.ptr(img), 1, N, wrgb.shape[0], wrgb.shape[2], H, W,
                                      capi.ptr(out), capi.stream()))
    return out


def alpha_cat(xa16: torch.Tensor, Ca: int, xb16: torch.Tensor, Cb: int, alpha: torch.Tensor, split: bool = False) -> torch.Tensor:
    """cat[xa*alpha, xb*(1-alpha)]; xb may hold ONE frame shared by the whole batch (per-clip constant features).  split: [hi | lo] inputs,
    output = the [hi | lo] layout of the (Ca + Cb)-channel result."""
    N, H, W, _ = xa16.shape
    out = activation(N, H, W, Ca + Cb, split, xa16.device)
    capi.check(_fn('alpha_cat', split)(capi.ptr(xa16, F16), Ca, xa16.shape[-1], capi.ptr(xb16, F16), Cb, xb16.shape[-1], int(xb16.shape[0] == 1 and N > 1),
                                       capi.ptr(alpha), N, H, W, capi.ptr(out, F16), capi.stream()))
    return out


def cat3(xa16: torch.Tensor, xb16: torch.Tensor, xc16: torch.Tensor, split: bool = False) -> torch.Tensor:
    """cat[xa, xb, xc] of three 256-channel NHWC fp16 tensors, unweighted; xc may hold ONE frame shared by the whole batch (per-clip constant
    features).  split: [hi | lo] inputs, output = the [hi | lo] layout of the 768-channel result."""
    N, H, W, _ = xa16.shape
    out = activation(N, H, W, 768, split, xa16.device)
    capi.check(_fn('cat3', split)(capi.ptr(xa16, F16), 256, xa16.shape[-1], capi.ptr(xb16, F16), 256, xb16.shape[-1], capi.ptr(xc16, F16), 256,
                                  xc16.shape[-1], int(xc16.shape[0] == 1 and N > 1), N, H, W, capi.ptr(out, F16), capi.stream()))
    return out


def alpha_mix(xa16: torch.Tensor, xb16: torch.Tensor, alpha: torch.Tensor, split: bool = False) -> torch.Tensor:
    """xa*alpha + xb*(1-alpha) of two NHWC fp16 tensors of C channels ([hi | lo] when split); alpha fp32 [N,1,H,W]."""
    N, H, W, Cs = xa16.shape
    C = Cs // 2 if split else Cs
    out = activation(N, H, W, C, split, xa16.device)
    capi.check(_fn('alpha_mix', split)(capi.ptr(xa16, F16), Cs, capi.ptr(xb16, F16), xb16.shape[-1], capi.ptr(alpha), C, N, H, W,
                                       capi.ptr(out, F16), capi.stream()))
    return out


def pack_plain_weights(w: torch.Tensor, b: torch.Tensor, in_tensor_channels: int, split: bool = False):
    """Conv weights [nw,O,I,k,k] (k = 1|3, float32 or float64, rounded to fp32 first) and bias [O] -> packed fp16 weights [nw,9,Opad,Ipad]
    (a 1x1 in tap 4) + fp32 bias [Opad] + k; output channels padded to a multiple of 128 with zero filters, input channels padded (zero
    weights) to the channel count of the activation tensor it reads."""
    w = w.detach()
    nw, O, I, k = w.shape[:4]
    Op = (O + 127) // 128 * 128
    w9 = torch.zeros(nw, Op, in_tensor_channels, 3, 3, device=w.device)
    if k == 3:
        w9[:, :O, :I] = w
    else:
        w9[:, :O, :I, 1, 1] = w[..., 0, 0]
    Ip = (in_tensor_channels + 63) // 64 * 64
    packed = torch.empty(nw, 9, Op, Ip * (2 if split else 1), device=w.device, dtype=torch.float16)
    capi.check(_fn('pack_weights', split)(capi.ptr(w9), nw, Op, in_tensor_channels, capi.ptr(packed, torch.float16), capi.stream()))
    bias = torch.zeros(Op, device=w.device)
    bias[:O] = b.detach()
    return packed, bias, k


def pack_plain(conv: torch.nn.Conv2d, in_tensor_channels: int, split: bool = False):
    """nn.Conv2d (k = 1|3) -> pack_plain_weights of its weight and bias."""
    return pack_plain_weights(conv.weight[None], conv.bias, in_tensor_channels, split)


def conv_plain(x16: torch.Tensor, packed, act: int, residual: Optional[torch.Tensor] = None, split: bool = False) -> torch.Tensor:
    """x16 [N,H,W,Ct] fp16 -> [N,H,W,Opad] fp16; act 0 linear, 2 nn.LeakyReLU(0.01), 3 ReLU; residual (same shape as the output) is added
    after the activation (ResBlock2d).  split: [hi | lo] tensors of twice the channels, weights from pack_plain(split=True).  No profiler
    region: the SR heads count it in 'sr_conv', the plane backbones in their own stages."""
    wp, bias, k = packed
    N, H, W, Ct = x16.shape
    y = activation(N, H, W, wp.shape[2], split, x16.device)
    args = (capi.ptr(x16, F16), capi.ptr(wp, F16), capi.ptr(bias), N, 1, Ct // 2 if split else Ct, wp.shape[2], H, W, k, act)
    if residual is None:
        capi.check(_fn('conv', split)(*args, capi.ptr(y, F16), capi.stream()))
    else:
        capi.check(_fn('conv_res', split)(*args, capi.ptr(residual, F16), capi.ptr(y, F16), capi.stream()))
    return y


def _sblocks(sr):
    """The two SynthesisBlocks (inside the LargeSynthesisBlocks when large_sr)."""
    return (sr.block0.block, sr.block1.block) if getattr(sr, 'large_sr', False) else (sr.block0, sr.block1)


class Prepared:
    """Folded + packed weights of the four conv layers and the two ToRGB layers for a given set of styles."""
    __slots__ = ('wp', 'wrgb0', 'wrgb1', 'Nw', 'split')

    def __init__(self, sr, wsel: torch.Tensor, split: bool = False):
        b0, b1 = _sblocks(sr)
        self.Nw, self.split = wsel.shape[0], bool(split)
        self.wp = [pack_for(b0.conv0, wsel[:, 0], split), pack_for(b0.conv1, wsel[:, 1], split), pack_for(b1.conv0, wsel[:, 0], split),
                   pack_for(b1.conv1, wsel[:, 1], split)]
        self.wrgb0, self.wrgb1 = b0.torgb.folded_weight(wsel[:, 2]), b1.torgb.folded_weight(wsel[:, 2])


def block0(b0, prep: Prepared, x0: torch.Tensor, rgb0: torch.Tensor):
    """SynthesisBlock b0: conv0 (up 2), then conv1 + ToRGB + the upsampled skip image rgb0 -> (activation, image)."""
    a0 = layer(x0, b0.conv0, prep.wp[0], 2, prep.split)
    return layer_torgb(a0, b0, prep.wp[1], prep.wrgb0, rgb0, prep.split)


def block1(b1, prep: Prepared, x: torch.Tensor, img: Optional[torch.Tensor], clamp: bool = False, uint8: bool = False) -> torch.Tensor:
    """SynthesisBlock b1: conv0 (up 2), then the fused last layer (conv1 + ToRGB + the upsampled skip image img, None: no skip) -> the image."""
    a2 = layer(x, b1.conv0, prep.wp[2], 2, prep.split)
    return last_layer(a2, b1, prep.wp[3], prep.wrgb1, img, clamp, uint8, prep.split)


def forward(sr, rgb: Optional[torch.Tensor], x: torch.Tensor, ws3: Optional[torch.Tensor], shared_styles: Optional[bool] = None,
            x_nhwc: Optional[torch.Tensor] = None, out_clamp: bool = False, out_uint8: bool = False, rgb_from_x: bool = False) -> torch.Tensor:
    """rgb [N,3,h,w], x [N,C,h,w] (fp32 NCHW, h <= 128), ws3 [N,3,512] -> [N,3,512,512] fp32.
    x_nhwc: the same features channels-last [N,h,w,C] (the renderer's native output) - skips a layout round trip.
    out_clamp: the image leaves the last epilogue clamped to [-1,1]; out_uint8: it leaves as uint8 HWC frames [N,512,512,3]
    (the caller loop's conversion, inference/real3d_infer.py:515-519, fused).
    With `sr.static_styles` (the caller guarantees constant styles, e.g. Real3D's ws == 1) the weight preparation
    (styles -> fold -> demod -> fp16 pack) is done once, by sr.prepared_styles()."""
    from .superresolution import SuperresolutionHybrid8XDC
    N, R = x.shape[0], sr.input_resolution
    split = getattr(sr, 'sr_mode', 'tc') == 'tc_exact'          # fp32-grade: split fp16 operands, three MMAs per product
    with capi.region('sr_prep'):
        prep = sr.prepared_styles()
        if prep is None:
            if shared_styles is None:
                shared_styles = N == 1 or getattr(sr, 'assume_shared_styles', False)
            prep = Prepared(sr, ws3[:1] if shared_styles else ws3, split)
        if x_nhwc is not None:                                 # rgb_from_x: rgb IS x[:, :3] (render head)
            x0, rgb0 = input_nhwc(x_nhwc, R, split, rgb=rgb_from_x)
        else:
            x0, rgb0 = to_nhwc_f16(x, R, split), None
        if rgb0 is None:
            rgb0 = SuperresolutionHybrid8XDC._resize(rgb, R) if rgb.shape[-1] != R else capi.f32(rgb)
    b0, b1 = _sblocks(sr)
    x1, img1 = block0(b0, prep, x0, rgb0)
    if getattr(sr, 'large_sr', False):
        return _forward_large_tail(sr, b1, x1, img1, prep, out_clamp, out_uint8)
    return block1(b1, prep, x1, img1, out_clamp, out_uint8)


def _large_packed(sr, split: bool = False):
    """Packed plain convolutions of the large_sr residual blocks / to_rgb layers (cached until the parameters are loaded or moved or the
    mode changes)."""
    def build():
        c = {}
        for name, blk, ch in (('b0', sr.block0, 256), ('b1', sr.block1, 128)):
            c[name] = [(pack_plain(rb.conv1, ch, split=split), pack_plain(rb.conv2, ch, split=split)) for rb in blk.resblocks]
            c[name + '_rgb'] = (blk.to_rgb.weight.detach().float().reshape(1, 3, ch).contiguous(), blk.to_rgb.bias.detach().float().contiguous())
        return c
    return sr.prepared('large', build, split)


def _forward_large_tail(sr, b1, a1, img1, prep, out_clamp, out_uint8):
    """LargeSynthesisBlock0/1.forward after the first SynthesisBlock (superresolution.py:296-329): residual blocks on the block output,
    `rgb = rgb + to_rgb(x)`, then the second block the same way.  x stays NHWC fp16 ([hi | lo] when split), rgb fp32 NCHW."""
    if out_uint8:
        raise NotImplementedError('uint8 frames are written by the standard SR\'s last epilogue; large_sr returns fp32')
    split = prep.split
    lp = _large_packed(sr, split)

    def tail(x16, img, key):
        with capi.region('sr_conv'):
            for c1, c2 in lp[key]:
                t = conv_plain(x16, c1, 3, split=split)
                x16 = conv_plain(t, c2, 3, residual=x16, split=split)
        return x16, torgb(x16, *lp[key + '_rgb'], img, split)

    x16, img1 = tail(a1, img1, 'b0')
    a2 = layer(x16, b1.conv0, prep.wp[2], 2, split)
    a3, img2 = layer_torgb(a2, b1, prep.wp[3], prep.wrgb1, img1, split)
    _, out = tail(a3, img2, 'b1')
    return out.clamp_(-1, 1) if out_clamp else out
