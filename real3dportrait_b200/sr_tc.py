"""Tensor-core execution of SuperresolutionHybrid8XDC.forward (superresolution.py:348-359): the same layers as the
fp32 modules in superresolution.py, run as wgmma implicit GEMMs (csrc/sr_tc.cu) on NHWC fp16 activations with fp32
accumulation.  Weights are folded (modulated + demodulated) in fp32 per sample, exactly as the reference does, and only
then rounded to fp16.  Stated tolerance vs the fp32 reference: see tests/test_gpu_parity.py::test_sr_full_tc."""
from __future__ import annotations

from typing import Optional

import torch

from . import _capi as capi


def available() -> bool:
    return hasattr(capi.lib(), 'r3dp_sr_tc_layer')


def _fn(name: str, split: bool):
    """C entry point `r3dp_sr_tc_<name>` or its split-operand twin `r3dp_sr_tcx_<name>` (sr_mode='tc_exact')."""
    return getattr(capi.lib(), ('r3dp_sr_tcx_' if split else 'r3dp_sr_tc_') + name)


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
    y = torch.empty(N, H * up, W * up, O * (2 if split else 1), device=x16.device, dtype=torch.float16)
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
    Cp = (Cc + 63) // 64 * 64
    y = torch.empty(N, size, size, Cp * (2 if split else 1), device=x.device, dtype=torch.float16)
    capi.check(_fn('input', split)(capi.ptr(x), N, Cc, h, w, size, capi.ptr(y, torch.float16), capi.stream()))
    return y


def pack_plain(conv: torch.nn.Conv2d, in_tensor_channels: int, out_pad: int = 128, split: bool = False):
    """nn.Conv2d (k = 1|3) -> packed fp16 weights [1,9,Opad,Ipad] + fp32 bias [Opad]; output channels padded to a multiple of
    `out_pad` with zero filters, input channels padded (zero weights) to the channel count of the activation tensor it reads."""
    w = conv.weight.detach().float()
    O, I, k, _ = w.shape
    Op = (O + out_pad - 1) // out_pad * out_pad
    w9 = torch.zeros(1, Op, in_tensor_channels, 3, 3, device=w.device)
    if k == 3:
        w9[0, :O, :I] = w
    else:
        w9[0, :O, :I, 1, 1] = w[:, :, 0, 0]
    Ip = (in_tensor_channels + 63) // 64 * 64
    packed = torch.empty(1, 9, Op, Ip * (2 if split else 1), device=w.device, dtype=torch.float16)
    capi.check(_fn('pack_weights', split)(capi.ptr(w9), 1, Op, in_tensor_channels, capi.ptr(packed, torch.float16), capi.stream()))
    bias = torch.zeros(Op, device=w.device)
    bias[:O] = conv.bias.detach().float()
    return packed, bias, k


def conv_plain(x16: torch.Tensor, packed, act: int, residual: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x16 [N,H,W,Ct] fp16 -> [N,H,W,Opad] fp16; act 0 linear, 2 nn.LeakyReLU(0.01), 3 ReLU; residual (same shape as the output) is added
    after the activation (ResBlock2d)."""
    wp, bias, k = packed
    N, H, W, Ct = x16.shape
    y = torch.empty(N, H, W, wp.shape[2], device=x16.device, dtype=torch.float16)
    with capi.region('sr_conv'):
        capi.check(capi.lib().r3dp_sr_tc_conv_res(capi.ptr(x16, torch.float16), capi.ptr(wp, torch.float16), capi.ptr(bias), N, 1, Ct, wp.shape[2], H, W, k, act,
                                                  capi.ptr(residual, torch.float16), capi.ptr(y, torch.float16), capi.stream()))
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


def forward(sr, rgb: Optional[torch.Tensor], x: torch.Tensor, ws3: Optional[torch.Tensor], shared_styles: Optional[bool] = None,
            x_nhwc: Optional[torch.Tensor] = None, out_clamp: bool = False, out_uint8: bool = False, rgb_from_x: bool = False) -> torch.Tensor:
    """rgb [N,3,h,w], x [N,C,h,w] (fp32 NCHW, h <= 128), ws3 [N,3,512] -> [N,3,512,512] fp32.
    x_nhwc: the same features channels-last [N,h,w,C] (the renderer's native output) - skips a layout round trip.
    out_clamp: the image leaves the last epilogue clamped to [-1,1]; out_uint8: it leaves as uint8 HWC frames [N,512,512,3]
    (the caller loop's conversion, inference/real3d_infer.py:515-519, fused).
    If `sr.static_prepared` is set (caller guarantees constant styles, e.g. Real3D's ws == 1) the weight preparation
    (styles -> fold -> demod -> fp16 pack) is skipped."""
    from .superresolution import SuperresolutionHybrid8XDC
    L = capi.lib()
    N = x.shape[0]
    split = getattr(sr, 'sr_mode', 'tc') == 'tc_exact'          # fp32-grade: split fp16 operands, three MMAs per product
    wide = 2 if split else 1
    if split and getattr(sr, 'large_sr', False):
        raise NotImplementedError("large_sr runs with sr_mode='tc' (its residual epilogue is not built for split operands)")
    prep = getattr(sr, 'static_prepared', None)
    if prep is not None and prep.split != split:
        prep = None
    with capi.region('sr_prep'):
        if prep is None:
            if shared_styles is None:
                shared_styles = N == 1 or getattr(sr, 'assume_shared_styles', False)
            prep = Prepared(sr, ws3[:1] if shared_styles else ws3, split)
        if x_nhwc is not None:
            xn = capi.f32(x_nhwc)
            _, h, w, Cc = xn.shape
            x0 = torch.empty(N, sr.input_resolution, sr.input_resolution, (Cc + 63) // 64 * 64 * wide, device=xn.device, dtype=torch.float16)
            if rgb_from_x:                                     # rgb IS x[:, :3] (render head): its resize rides in the same launch
                rgb0 = torch.empty(N, 3, sr.input_resolution, sr.input_resolution, device=xn.device)
                capi.check(L.r3dp_sr_tc_input_nhwc_rgb(capi.ptr(xn), N, Cc, h, w, sr.input_resolution, capi.ptr(x0, torch.float16), capi.ptr(rgb0), int(split),
                                                       capi.stream()))
            else:
                capi.check(_fn('input_nhwc', split)(capi.ptr(xn), N, Cc, h, w, sr.input_resolution, capi.ptr(x0, torch.float16), capi.stream()))
        else:
            x0 = to_nhwc_f16(x, sr.input_resolution, split)
        if not (rgb_from_x and x_nhwc is not None):
            rgb0 = SuperresolutionHybrid8XDC._resize(rgb, sr.input_resolution) if rgb.shape[-1] != sr.input_resolution else capi.f32(rgb)
    (b0, b1), Nw, wp = _sblocks(sr), prep.Nw, prep.wp
    a0 = layer(x0, b0.conv0, wp[0], 2, split)
    a1 = torch.empty(N, 256, 256, 256 * wide, device=x.device, dtype=torch.float16)
    img1 = torch.empty(N, 3, 256, 256, device=x.device)
    with capi.region('sr_conv'):                               # block0.conv1 + block0.torgb (+ upsampled skip) in one kernel
        capi.check(_fn('layer_torgb', split)(capi.ptr(a0, torch.float16), capi.ptr(wp[1], torch.float16), capi.ptr(capi.f32(b0.conv1.bias)),
                                            capi.ptr(prep.wrgb0), capi.ptr(capi.f32(b0.torgb.bias)), capi.ptr(rgb0), N, Nw, 256, 256, 256, 256,
                                            capi.ptr(a1, torch.float16), capi.ptr(img1), capi.stream()))
    if getattr(sr, 'large_sr', False):
        return _forward_large_tail(sr, a1, img1, prep, out_clamp, out_uint8)
    a2 = layer(a1, b1.conv0, wp[2], 2, split)
    out = torch.empty(N, 512, 512, 3, device=x.device, dtype=torch.uint8) if out_uint8 else torch.empty(N, 3, 512, 512, device=x.device)
    with capi.region('sr_conv'):                               # block1.conv1 + block1.torgb: the 128-channel activation is never written
        capi.check((L.r3dp_sr_tcx_last_layer if split else L.r3dp_sr_tc_last_layer_ex)(capi.ptr(a2, torch.float16), capi.ptr(wp[3], torch.float16), capi.ptr(capi.f32(b1.conv1.bias)),
                                              capi.ptr(prep.wrgb1), capi.ptr(capi.f32(b1.torgb.bias)), capi.ptr(img1), N, Nw, 128, 512, 512,
                                              None if out_uint8 else capi.ptr(out), capi.ptr(out, torch.uint8) if out_uint8 else None,
                                              int(out_clamp or out_uint8), capi.stream()))
    return out


def _large_packed(sr):
    """Packed plain convolutions of the large_sr residual blocks / to_rgb layers (cached until the parameters are reloaded)."""
    c = getattr(sr, '_large_cache', None)
    if c is None:
        c = {}
        for name, blk, ch in (('b0', sr.block0, 256), ('b1', sr.block1, 128)):
            c[name] = [(pack_plain(rb.conv1, ch), pack_plain(rb.conv2, ch)) for rb in blk.resblocks]
            c[name + '_rgb'] = (blk.to_rgb.weight.detach().float().reshape(1, 3, ch).contiguous(), blk.to_rgb.bias.detach().float().contiguous())
        sr._large_cache = c
    return c


def _forward_large_tail(sr, a1, img1, prep, out_clamp, out_uint8):
    """LargeSynthesisBlock0/1.forward after the first SynthesisBlock (superresolution.py:296-329): residual blocks on the block output,
    `rgb = rgb + to_rgb(x)`, then the second block the same way.  x stays NHWC fp16, rgb fp32 NCHW."""
    if out_uint8:
        raise NotImplementedError('uint8 frames are written by the standard SR\'s last epilogue; large_sr returns fp32')
    L = capi.lib()
    lp = _large_packed(sr)
    _, b1 = _sblocks(sr)
    N, Nw, wp = a1.shape[0], prep.Nw, prep.wp

    def tail(x16, img, key, ch, res):
        for c1, c2 in lp[key]:
            t = conv_plain(x16, c1, 3)
            x16 = conv_plain(t, c2, 3, residual=x16)
        wrgb, brgb = lp[key + '_rgb']
        out = torch.empty(N, 3, res, res, device=x16.device)
        capi.check(L.r3dp_sr_tc_torgb_ex(capi.ptr(x16, torch.float16), capi.ptr(wrgb), capi.ptr(brgb), capi.ptr(img), 1, N, 1, ch, res, res, capi.ptr(out),
                                         capi.stream()))
        return x16, out

    x16, img1 = tail(a1, img1, 'b0', 256, 256)
    a2 = layer(x16, b1.conv0, wp[2], 2)
    a3 = torch.empty(N, 512, 512, 128, device=a1.device, dtype=torch.float16)
    img2 = torch.empty(N, 3, 512, 512, device=a1.device)
    with capi.region('sr_conv'):
        capi.check(L.r3dp_sr_tc_layer_torgb(capi.ptr(a2, torch.float16), capi.ptr(wp[3], torch.float16), capi.ptr(capi.f32(b1.conv1.bias)),
                                            capi.ptr(prep.wrgb1), capi.ptr(capi.f32(b1.torgb.bias)), capi.ptr(img1), N, Nw, 128, 128, 512, 512,
                                            capi.ptr(a3, torch.float16), capi.ptr(img2), capi.stream()))
    _, out = tail(a3, img2, 'b1', 128, 512)
    return out.clamp_(-1, 1) if out_clamp else out
