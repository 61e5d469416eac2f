"""SuperresolutionHybrid8XDC and its StyleGAN2 blocks — host mirror of
modules/eg3ds/models/superresolution.py:331-359 and modules/eg3ds/models/networks_stylegan2.py:286-473.

Module / parameter / buffer names equal the reference's, so `load_state_dict(strict=True)` of released checkpoints
works.  forward() orchestrates libr3dp_b200 calls; two arithmetic modes (`sr_mode`):
  'fp32'  exact CUDA-core path (parity anchor, matches the reference to fp32 re-association noise),
  'tc'    tensor-core path (wgmma, fp16 operands, fp32 accumulate) — the fast path, own stated tolerance,
  'tc_exact'  the same kernels with split fp16 operands (hi + lo) — fp32-grade results (also for large_sr and the torso head).
Inference only: noise_mode must be 'none' (as in img2plane_baseline.py:113,144), fp32 parameters."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _capi as capi
from .decoder import FullyConnectedLayer
from .prepared import PreparedMixin


def setup_filter(f=(1, 3, 3, 1)) -> torch.Tensor:
    """upfirdn2d.setup_filter (torch_utils/ops/upfirdn2d.py:72-116): separable taps -> normalised 2-D filter."""
    f = torch.as_tensor(f, dtype=torch.float32)
    f = torch.outer(f, f)
    return f / f.sum()


def _styles(affine: FullyConnectedLayer, w: torch.Tensor, post_scale: float = 1.0) -> torch.Tensor:
    w = capi.f32(w)
    s = torch.empty(w.shape[0], affine.out_features, device=w.device)
    capi.check(capi.lib().r3dp_sr_styles(capi.ptr(w), capi.ptr(capi.f32(affine.weight)), capi.ptr(capi.f32(affine.bias)), w.shape[0],
                                         affine.in_features, affine.out_features, C.c_float(post_scale), capi.ptr(s), capi.stream()))
    return s


def _fold(weight: torch.Tensor, styles: torch.Tensor, demodulate: bool) -> torch.Tensor:
    O, I, k, _ = weight.shape
    N = styles.shape[0]
    wf = torch.empty(N, O, I, k, k, device=styles.device)
    capi.check(capi.lib().r3dp_sr_fold_weights(capi.ptr(capi.f32(weight)), capi.ptr(styles), N, O, I, k, int(demodulate), capi.ptr(wf),
                                               capi.stream()))
    return wf


class SynthesisLayer(torch.nn.Module):
    def __init__(self, in_channels, out_channels, w_dim, resolution, kernel_size=3, up=1, use_noise=True, activation='lrelu',
                 resample_filter=(1, 3, 3, 1), conv_clamp=None, channels_last=False, **other_args):
        super().__init__()
        assert kernel_size == 3 and activation == 'lrelu' and up in (1, 2)
        self.in_channels, self.out_channels, self.w_dim = in_channels, out_channels, w_dim
        self.resolution, self.up, self.use_noise, self.activation, self.conv_clamp = resolution, up, use_noise, activation, conv_clamp
        self.register_buffer('resample_filter', setup_filter(resample_filter))
        self.padding = kernel_size // 2
        self.act_gain = float(np.sqrt(2))
        self.affine = FullyConnectedLayer(w_dim, in_channels, bias_init=1)
        self.weight = torch.nn.Parameter(torch.randn([out_channels, in_channels, kernel_size, kernel_size]))
        if use_noise:
            self.register_buffer('noise_const', torch.randn([resolution, resolution]))
            self.noise_strength = torch.nn.Parameter(torch.zeros([]))
        self.bias = torch.nn.Parameter(torch.zeros([out_channels]))

    def folded_weight(self, w: torch.Tensor) -> torch.Tensor:
        """Per-sample modulated + demodulated weights [N,O,I,3,3] (modulated_conv2d, networks_stylegan2.py:63-70)."""
        return _fold(self.weight, _styles(self.affine, w), True)

    def forward(self, x, w, noise_mode='random', fused_modconv=True, gain=1, **kwargs):
        """x [N,Cin,r/up,r/up], w [N,w_dim] -> [N,Cout,r,r]  (exact fp32 path)."""
        assert noise_mode in ['random', 'const', 'none']
        if noise_mode != 'none' and self.use_noise and float(self.noise_strength) != 0.0:
            raise NotImplementedError("only noise_mode='none' is on the inference path (img2plane_baseline.py:113)")
        if gain != 1 or self.conv_clamp is not None:
            raise NotImplementedError('gain != 1 / conv_clamp are fp16-training options outside the inference path')
        in_res = self.resolution // self.up
        x = capi.f32(x)
        N = x.shape[0]
        assert tuple(x.shape[1:]) == (self.in_channels, in_res, in_res), (x.shape, self.in_channels, in_res)
        wf = self.folded_weight(w)
        y = torch.empty(N, self.out_channels, self.resolution, self.resolution, device=x.device)
        L = capi.lib()
        scratch = None
        if self.up == 2:
            scratch = torch.empty(L.r3dp_sr_layer_scratch_bytes(N, self.out_channels, in_res, in_res), device=x.device, dtype=torch.uint8)
        with capi.region('sr_conv'):
            capi.check(L.r3dp_sr_layer_fp32(capi.ptr(x), capi.ptr(wf), capi.ptr(capi.f32(self.bias)), N, self.in_channels,
                                            self.out_channels, in_res, in_res, self.up, capi.ptr(y), capi.ptr(scratch, torch.uint8),
                                            capi.stream()))
        return y

    def extra_repr(self):
        return (f'in_channels={self.in_channels:d}, out_channels={self.out_channels:d}, w_dim={self.w_dim:d}, '
                f'resolution={self.resolution:d}, up={self.up}, activation={self.activation:s}')


class ToRGBLayer(torch.nn.Module):
    def __init__(self, in_channels, out_channels, w_dim, kernel_size=1, conv_clamp=None, channels_last=False):
        super().__init__()
        assert kernel_size == 1 and out_channels == 3
        self.in_channels, self.out_channels, self.w_dim, self.conv_clamp = in_channels, out_channels, w_dim, conv_clamp
        self.affine = FullyConnectedLayer(w_dim, in_channels, bias_init=1)
        self.weight = torch.nn.Parameter(torch.randn([out_channels, in_channels, kernel_size, kernel_size]))
        self.bias = torch.nn.Parameter(torch.zeros([out_channels]))
        self.weight_gain = 1 / np.sqrt(in_channels * (kernel_size ** 2))

    def folded_weight(self, w: torch.Tensor) -> torch.Tensor:
        """[N,3,Cin]: weight * styles * 1/sqrt(Cin), no demodulation (networks_stylegan2.py:366-368)."""
        return _fold(self.weight, _styles(self.affine, w, float(self.weight_gain)), False).reshape(-1, 3, self.in_channels)

    def forward(self, x, w, fused_modconv=True, skip=None):
        """x [N,Cin,H,W] -> [N,3,H,W]; if `skip` [N,3,H/2,W/2] is given, adds upsample2d(skip) (SynthesisBlock :465-469)."""
        x = capi.f32(x)
        N, I, H, W = x.shape
        out = torch.empty(N, 3, H, W, device=x.device)
        capi.check(capi.lib().r3dp_sr_torgb_fp32(capi.ptr(x), capi.ptr(self.folded_weight(w)), capi.ptr(capi.f32(self.bias)),
                                                 capi.ptr(None if skip is None else capi.f32(skip)), N, I, H, W, capi.ptr(out),
                                                 capi.stream()))
        return out


class SynthesisBlock(torch.nn.Module):
    def __init__(self, in_channels, out_channels, w_dim, resolution, img_channels, is_last, architecture='skip',
                 resample_filter=(1, 3, 3, 1), conv_clamp=256, use_fp16=False, fp16_channels_last=False,
                 fused_modconv_default=True, **layer_kwargs):
        super().__init__()
        assert architecture == 'skip' and in_channels != 0 and not use_fp16, 'SR blocks of Real3D-Portrait: skip arch, fp32'
        self.in_channels, self.w_dim, self.resolution, self.img_channels = in_channels, w_dim, resolution, img_channels
        self.is_last, self.architecture = is_last, architecture
        self.register_buffer('resample_filter', setup_filter(resample_filter))
        layer_kwargs = {k: v for k, v in layer_kwargs.items() if k not in ('channel_base', 'channel_max')}
        self.conv0 = SynthesisLayer(in_channels, out_channels, w_dim=w_dim, resolution=resolution, up=2,
                                    resample_filter=resample_filter, conv_clamp=conv_clamp, **layer_kwargs)
        self.conv1 = SynthesisLayer(out_channels, out_channels, w_dim=w_dim, resolution=resolution, conv_clamp=conv_clamp, **layer_kwargs)
        self.torgb = ToRGBLayer(out_channels, img_channels, w_dim=w_dim, conv_clamp=conv_clamp)
        self.num_conv, self.num_torgb = 2, 1

    def forward(self, x, img, ws, force_fp32=False, fused_modconv=None, update_emas=False, **layer_kwargs):
        """x [N,Cin,r/2,r/2], img [N,3,r/2,r/2] | None, ws [N,3,w_dim] -> (x [N,Cout,r,r], img [N,3,r,r])."""
        assert ws.ndim == 3 and ws.shape[1] == self.num_conv + self.num_torgb and ws.shape[2] == self.w_dim, ws.shape
        w0, w1, w2 = ws.unbind(dim=1)
        x = self.conv0(x, w0, **layer_kwargs)
        x = self.conv1(x, w1, **layer_kwargs)
        img = self.torgb(x, w2, skip=img)
        return x, img


class ResBlock2d(torch.nn.Module):
    """Parameter container of superresolution.py:263-288: out = relu(conv2(relu(conv1(x)))) + x (runs inside sr_tc.forward)."""

    def __init__(self, in_features, kernel_size, padding):
        super().__init__()
        self.conv1 = torch.nn.Conv2d(in_features, in_features, kernel_size=kernel_size, padding=padding)
        self.conv2 = torch.nn.Conv2d(in_features, in_features, kernel_size=kernel_size, padding=padding)
        self.act = torch.nn.ReLU(inplace=False)


class LargeSynthesisBlock0(torch.nn.Module):
    """superresolution.py:296-312: SynthesisBlock(channels -> 256 @256) + residual blocks + `rgb = rgb + to_rgb(x)`."""

    def __init__(self, channels, use_fp16, resblocks, **block_kwargs):
        super().__init__()
        self.block = SynthesisBlock(channels, 256, w_dim=512, resolution=256, img_channels=3, is_last=False, use_fp16=use_fp16, conv_clamp=None,
                                    **block_kwargs)
        self.resblocks = torch.nn.Sequential(*[ResBlock2d(256, kernel_size=3, padding=1) for _ in range(resblocks)])
        self.to_rgb = torch.nn.Conv2d(256, 3, kernel_size=1)


class LargeSynthesisBlock1(torch.nn.Module):
    """superresolution.py:314-329: SynthesisBlock(256 -> 128 @512) + residual blocks + `rgb = rgb + to_rgb(x)`."""

    def __init__(self, use_fp16, resblocks, **block_kwargs):
        super().__init__()
        self.block = SynthesisBlock(256, 128, w_dim=512, resolution=512, img_channels=3, is_last=True, use_fp16=use_fp16, conv_clamp=None,
                                    **block_kwargs)
        self.resblocks = torch.nn.Sequential(*[ResBlock2d(128, kernel_size=3, padding=1) for _ in range(resblocks)])
        self.to_rgb = torch.nn.Conv2d(128, 3, kernel_size=1)


class SuperresolutionHybrid8XDC(PreparedMixin, torch.nn.Module):
    def __init__(self, channels, img_resolution, sr_num_fp16_res, sr_antialias, large_sr=False, sr_mode='fp32', resblocks_in_large_sr=None,
                 **block_kwargs):
        """large_sr=True (superresolution.py:263-345) needs `resblocks_in_large_sr` (the reference reads hparams['resblocks_in_large_sr']) and
        runs on the tensor-core path only (sr_mode 'tc' or 'tc_exact')."""
        super().__init__()
        assert img_resolution == 512
        if sr_num_fp16_res > 0:
            raise NotImplementedError('Real3D-Portrait runs the SR with sr_num_fp16_res=0 (img2plane_baseline.py:102)')
        assert sr_mode in ('fp32', 'tc', 'tc_exact')      # tc_exact: tensor cores with split fp16 operands, fp32-grade results
        self.sr_mode = sr_mode
        self.large_sr = bool(large_sr)
        self.input_resolution = 128
        self.sr_antialias = sr_antialias
        if self.large_sr:
            if sr_mode not in ('tc', 'tc_exact') or resblocks_in_large_sr is None:
                raise NotImplementedError("large_sr is built on the tensor-core path (sr_mode='tc' | 'tc_exact') and needs resblocks_in_large_sr")
            self.block0 = LargeSynthesisBlock0(channels, False, int(resblocks_in_large_sr), **block_kwargs)
            self.block1 = LargeSynthesisBlock1(False, int(resblocks_in_large_sr), **block_kwargs)
        else:
            self.block0 = SynthesisBlock(channels, 256, w_dim=512, resolution=256, img_channels=3, is_last=False, use_fp16=False,
                                         conv_clamp=None, **block_kwargs)
            self.block1 = SynthesisBlock(256, 128, w_dim=512, resolution=512, img_channels=3, is_last=True, use_fp16=False,
                                         conv_clamp=None, **block_kwargs)
        self.static_styles = False       # the caller passes constant styles (Real3D's ws == 1): the tensor-core path prepares them once

    def prepare_styles(self, wsel: torch.Tensor):
        """Folded + packed weights of the tensor-core path for styles wsel [Nw,3,512]."""
        from . import sr_tc
        return sr_tc.Prepared(self, wsel, self.sr_mode == 'tc_exact')

    def prepared_styles(self):
        """With static_styles on the tensor-core path: prepare_styles() of the all-ones styles, cached until the parameters are loaded or
        moved; None otherwise (the styles are then prepared per call)."""
        if not self.static_styles or self.sr_mode not in ('tc', 'tc_exact'):
            return None

        def build():
            with torch.no_grad():
                return self.prepare_styles(torch.ones(1, 3, 512, device=next(self.parameters()).device))
        return self.prepared('styles', build, self.sr_mode == 'tc_exact')

    @staticmethod
    def _resize(x: torch.Tensor, size: int) -> torch.Tensor:
        x = capi.f32(x)
        N, Cc, h, w = x.shape
        y = torch.empty(N, Cc, size, size, device=x.device)
        capi.check(capi.lib().r3dp_sr_resize_bilinear(capi.ptr(x), N, Cc, h, w, size, capi.ptr(y), capi.stream()))
        return y

    def forward(self, rgb, x, ws, **block_kwargs):
        """rgb [N,3,h,w], x [N,channels,h,w], ws [N,>=1,512] -> [N,3,512,512]   (superresolution.py:348-359)."""
        x_nhwc = block_kwargs.pop('x_nhwc', None)          # optional: the same features channels-last (tensor-core path only)
        out_clamp, out_uint8 = bool(block_kwargs.pop('out_clamp', False)), bool(block_kwargs.pop('out_uint8', False))
        if (out_clamp or out_uint8) and self.sr_mode not in ('tc', 'tc_exact'):
            raise NotImplementedError('fused clamp / uint8 output is an option of the tensor-core SR path')
        rgb_from_x = bool(block_kwargs.pop('rgb_from_x', False))   # tensor-core path: the caller states rgb == x[:, :3] (one fused input launch)
        block_kwargs = {k: v for k, v in block_kwargs.items() if k != 'sr_mode'}
        if not (self.sr_mode in ('tc', 'tc_exact') and self.static_styles):     # prepared weights: the styles are not read again
            ws = ws[:, -1:, :].repeat(1, 3, 1)
        if x.shape[-1] > self.input_resolution:
            raise NotImplementedError('down-scaling inputs (antialiased) is not on the Real3D path')
        if self.sr_mode in ('tc', 'tc_exact'):
            from . import sr_tc
            return sr_tc.forward(self, rgb, x, ws, x_nhwc=x_nhwc, out_clamp=out_clamp, out_uint8=out_uint8, rgb_from_x=rgb_from_x)
        if x.shape[-1] != self.input_resolution:
            x = self._resize(x, self.input_resolution)
            rgb = self._resize(rgb, self.input_resolution)
        x, rgb = self.block0(x, rgb, ws, **block_kwargs)
        x, rgb = self.block1(x, rgb, ws, **block_kwargs)
        return rgb
