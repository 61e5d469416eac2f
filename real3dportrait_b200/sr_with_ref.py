"""SuperresolutionHybrid8XDC_Warp — host mirror of modules/real3d/super_resolution/sr_with_ref.py:16-162 (the torso/background
fusing SR head of OSAvatarSECC_Img2plane_Torso, BASELINE config 5).

Same constructor arguments, child-module names (`block0/1`, `torso_encoder`, `bg_encoder`, `head_torso_alpha_predictor`,
`fuse_head_torso_convs`, `head_torso_block`, `fuse_fg_bg_convs`, `torso_model`) and `forward` signature/return as the reference, so
released checkpoints load with strict=True.  The conv stack (782 GFLOP/frame, SURVEY.md §8d) runs on the tensor-core kernels of
csrc/sr_tc.cu; the torso warper `torso_model` (WarpBasedTorsoModelMediaPipe, SURVEY.md §2 #11: out of scope) stays the caller's
PyTorch module and is called as an opaque child exactly where the reference calls it.  Supported configuration = the released one
(egs/os_avatar/real3d_orig/secc_img2plane_torso_orig.yaml:26-30): torso_model_version v2, htbsr_head_weight_fuse_mode v2."""
from __future__ import annotations

from typing import Dict, Optional

import torch

from . import _capi as capi
from . import sr_tc
from .superresolution import SuperresolutionHybrid8XDC, SynthesisLayer, ToRGBLayer, setup_filter


class SynthesisBlockNoUp(torch.nn.Module):
    """Parameter container + tensor-core forward of superresolution.py:159-258 (architecture 'skip', in_channels != 0, fp32)."""

    def __init__(self, in_channels, out_channels, w_dim, resolution, img_channels, is_last, architecture='skip',
                 resample_filter=(1, 3, 3, 1), conv_clamp=256, use_fp16=False, fp16_channels_last=False, fused_modconv_default=True,
                 **layer_kwargs):
        super().__init__()
        assert architecture == 'skip' and in_channels != 0 and not use_fp16
        self.in_channels, self.w_dim, self.resolution, self.img_channels, self.is_last = in_channels, w_dim, resolution, img_channels, is_last
        self.register_buffer('resample_filter', setup_filter(resample_filter))
        layer_kwargs = {k: v for k, v in layer_kwargs.items() if k not in ('channel_base', 'channel_max')}
        self.conv0 = SynthesisLayer(in_channels, out_channels, w_dim=w_dim, resolution=resolution, conv_clamp=conv_clamp, **layer_kwargs)
        self.conv1 = SynthesisLayer(out_channels, out_channels, w_dim=w_dim, resolution=resolution, conv_clamp=conv_clamp, **layer_kwargs)
        self.torgb = ToRGBLayer(out_channels, img_channels, w_dim=w_dim, conv_clamp=conv_clamp)
        self.num_conv, self.num_torgb = 2, 1


_pack_plain = sr_tc.pack_plain


class SuperresolutionHybrid8XDC_Warp(SuperresolutionHybrid8XDC):
    def __init__(self, channels, img_resolution, sr_num_fp16_res, sr_antialias, hp: Optional[dict] = None, torso_model: Optional[torch.nn.Module] = None,
                 **block_kwargs):
        block_kwargs.setdefault('sr_mode', 'tc')
        super().__init__(channels, img_resolution, sr_num_fp16_res, sr_antialias, **block_kwargs)
        if self.sr_mode != 'tc':
            raise NotImplementedError('the torso head is built on the tensor-core path only (sr_mode="tc")')
        hp = dict(hp or {})
        self.hparams = {'torso_model_version': hp.get('torso_model_version', 'v2'), 'htbsr_head_weight_fuse_mode': hp.get('htbsr_head_weight_fuse_mode', 'v2'),
                        'htbsr_head_threshold': float(hp.get('htbsr_head_threshold', 0.9)), 'weight_fuse': hp.get('weight_fuse', True)}
        self.fuse_mode = self.hparams['htbsr_head_weight_fuse_mode']
        if self.hparams['torso_model_version'] != 'v2' or self.fuse_mode not in ('v1', 'v2', 'v3') or not self.hparams['weight_fuse']:
            raise NotImplementedError('built: torso_model_version=v2 with htbsr_head_weight_fuse_mode v1 | v2 (the released Real3D torso config) | v3, weight_fuse=True')
        if torso_model is not None:
            self.torso_model = torso_model                      # the reference's WarpBasedTorsoModelMediaPipe('standard'), supplied by the caller
        nn = torch.nn
        self.torso_encoder = nn.Sequential(nn.Conv2d(64, 256, 1, 1, padding=0))
        self.bg_encoder = nn.Sequential(nn.Conv2d(3, 64, 3, 1, padding=1), nn.LeakyReLU(), nn.Conv2d(64, 256, 3, 1, padding=1), nn.LeakyReLU(),
                                        nn.Conv2d(256, 256, 3, 1, padding=1))
        if self.fuse_mode != 'v1':                              # the reference builds these children for every mode but v1 (sr_with_ref.py:36-55)
            self.head_torso_alpha_predictor = nn.Sequential(nn.Conv2d(7, 32, 3, 1, padding=1), nn.LeakyReLU(), nn.Conv2d(32, 32, 3, 1, padding=1),
                                                            nn.LeakyReLU(), nn.Conv2d(32, 1, 3, 1, padding=1), nn.Sigmoid())   # used by v3 only
            self.fuse_head_torso_convs = nn.Sequential(nn.Conv2d(512, 256, 3, 1, padding=1), nn.LeakyReLU(), nn.Conv2d(256, 256, 3, 1, padding=1))
            bk = {k: v for k, v in block_kwargs.items() if k not in ('sr_mode', 'channel_base', 'channel_max')}
            self.head_torso_block = SynthesisBlockNoUp(256, 256, w_dim=512, resolution=256, img_channels=3, is_last=False, use_fp16=False,
                                                       conv_clamp=None, **bk)
        self.fuse_fg_bg_convs = nn.Sequential(nn.Conv2d(512, 64, 1, 1, padding=0), nn.LeakyReLU(), nn.Conv2d(64, 256, 3, 1, padding=1),
                                              nn.LeakyReLU(), nn.Conv2d(256, 256, 3, 1, padding=1))
        self._plain_cache = None
        self._clip_cache = None
        self.static_prepared_warp = None

    # ---- weight preparation ------------------------------------------------------------------------------------------------
    def _plain(self) -> Dict[str, tuple]:
        if self._plain_cache is None:
            te, bg, ff = self.torso_encoder, self.bg_encoder, self.fuse_fg_bg_convs
            self._plain_cache = {
                'te': _pack_plain(te[0], 64), 'bg0': _pack_plain(bg[0], 64), 'bg2': _pack_plain(bg[2], 128), 'bg4': _pack_plain(bg[4], 256),
                'ff0': _pack_plain(ff[0], 512), 'ff2': _pack_plain(ff[2], 128), 'ff4': _pack_plain(ff[4], 256),
            }
            if self.fuse_mode != 'v1':
                fh = self.fuse_head_torso_convs
                self._plain_cache.update({'fh0': _pack_plain(fh[0], 512), 'fh2': _pack_plain(fh[2], 256)})
            if self.fuse_mode == 'v3':                             # the mask predictor runs with split fp16 operands (its output is thresholded)
                ap = self.head_torso_alpha_predictor
                self._plain_cache.update({'ap0': sr_tc.pack_plain(ap[0], 64, split=True), 'ap2': sr_tc.pack_plain(ap[2], 128, split=True),
                                          'ap4': sr_tc.pack_plain(ap[4], 128, split=True)})
        return self._plain_cache

    def _load_from_state_dict(self, *a, **k):
        # runs for THIS module whenever it or any parent (RenderHead, FrameEngine.load_params) loads a state_dict: every cache that was
        # derived from the parameters is dropped (packed fp16 conv weights, per-clip constants, prepared styles)
        self._plain_cache = None
        self._clip_cache = None
        self.static_prepared_warp = None
        return super()._load_from_state_dict(*a, **k)

    @staticmethod
    def _conv(x16: torch.Tensor, packed, act: int, split: bool = False) -> torch.Tensor:
        """x16 [N,H,W,Ct] fp16 -> [N,H,W,Opad] fp16; act 0 linear, 2 nn.LeakyReLU(0.01).  split: [hi | lo] tensors of twice the channels (fp32-grade)."""
        wp, bias, k = packed
        N, H, W, Ct = x16.shape
        wide = 2 if split else 1
        y = torch.empty(N, H, W, wp.shape[2] * wide, device=x16.device, dtype=torch.float16)
        fn = capi.lib().r3dp_sr_tcx_conv if split else capi.lib().r3dp_sr_tc_conv
        with capi.region('sr_conv'):
            capi.check(fn(capi.ptr(x16, torch.float16), capi.ptr(wp, torch.float16), capi.ptr(bias), N, 1, Ct // wide, wp.shape[2], H, W, k, act,
                          capi.ptr(y, torch.float16), capi.stream()))
        return y

    @staticmethod
    def _alpha_cat(xa16, Ca, xb16, Cb, alpha) -> torch.Tensor:
        """cat[xa*alpha, xb*(1-alpha)]; xb may hold ONE frame shared by the whole batch (per-clip constant features)."""
        N, H, W, _ = xa16.shape
        out = torch.empty(N, H, W, Ca + Cb, device=xa16.device, dtype=torch.float16)
        capi.check(capi.lib().r3dp_sr_alpha_cat_ex(capi.ptr(xa16, torch.float16), Ca, xa16.shape[-1], capi.ptr(xb16, torch.float16), Cb, xb16.shape[-1],
                                                   int(xb16.shape[0] == 1 and N > 1), capi.ptr(alpha), N, H, W, capi.ptr(out, torch.float16), capi.stream()))
        return out

    # ---- per-clip constants (SURVEY.md §8f #2) -------------------------------------------------------------------------------------------
    @torch.no_grad()
    def begin_clip(self, ref_torso_rgb: torch.Tensor, ref_bg_rgb: torch.Tensor) -> None:
        """Hoist what the reference recomputes for every frame although it only depends on the clip's reference images
        (sr_with_ref.py:77-90): the two antialiased 512->256 resizes and bg_encoder(ref_bg) (96.9 GFLOP/frame).  ref_* [1,3,512,512].
        Until end_clip(), forward() ignores its ref_torso_rgb / ref_bg_rgb arguments and uses these."""
        assert ref_torso_rgb.shape[0] == 1 and ref_bg_rgb.shape[0] == 1, 'one reference image per clip'
        plain = self._plain()
        t256, b256 = self._aa_down2(ref_torso_rgb), self._aa_down2(ref_bg_rgb)
        x_bg = self._conv(self._conv(self._conv(sr_tc.to_nhwc_f16(b256, 256), plain['bg0'], 2), plain['bg2'], 2), plain['bg4'], 0)
        self._clip_cache = {'ref_torso_256': t256, 'ref_bg_256': b256, 'x_bg': x_bg}

    def end_clip(self) -> None:
        self._clip_cache = None

    @staticmethod
    def _blend(a, b, alpha) -> torch.Tensor:
        a, b = capi.f32(a), capi.f32(b)
        N, Cc, H, W = a.shape
        out = torch.empty_like(a)
        capi.check(capi.lib().r3dp_sr_blend(capi.ptr(a), capi.ptr(b), capi.ptr(alpha), N, Cc, H, W, capi.ptr(out), capi.stream()))
        return out

    @staticmethod
    def _aa_down2(x) -> torch.Tensor:
        x = capi.f32(x)
        N, Cc, H2, W2 = x.shape
        y = torch.empty(N, Cc, H2 // 2, W2 // 2, device=x.device)
        capi.check(capi.lib().r3dp_sr_resize_aa_down2(capi.ptr(x), N, Cc, H2 // 2, W2 // 2, capi.ptr(y), capi.stream()))
        return y

    # ---- forward -------------------------------------------------------------------------------------------------------------
    def forward(self, rgb, x, ws, ref_torso_rgb, ref_bg_rgb, weights_img, segmap, kp_s, kp_d, target_torso_mask=None, **block_kwargs):
        """rgb [N,3,h,w], x [N,32,h,w], ws [N,>=1,512], ref_torso_rgb/ref_bg_rgb [N,3,512,512], weights_img [N,1,h,w], segmap [N,6,512,512],
        kp_s/kp_d [N,68,3] -> (rgb [N,3,512,512], facev2v_ret)   (sr_with_ref.py:67-162)."""
        if getattr(self, 'torso_model', None) is None:
            raise RuntimeError('SuperresolutionHybrid8XDC_Warp needs its torso_model child (the reference WarpBasedTorsoModelMediaPipe); '
                               'pass torso_model=... to the constructor')
        if block_kwargs.get('noise_mode', 'none') != 'none':
            raise NotImplementedError("only noise_mode='none' is on the inference path")
        L = capi.lib()
        N = rgb.shape[0]
        if ref_torso_rgb.shape[-1] != 512 or ref_bg_rgb.shape[-1] != 512:
            raise NotImplementedError('reference images must be 512x512 (antialiased 1/2 resize is the only down-scaling built)')
        ws3 = ws[:, -1:, :].expand(N, 3, -1)
        prep = getattr(self, 'static_prepared_warp', None)
        with capi.region('sr_prep'):
            if prep is None:
                shared = N == 1 or getattr(self, 'assume_shared_styles', False)
                wsel = ws3[:1] if shared else ws3
                prep = {'main': sr_tc.Prepared(self, wsel)}
                if self.fuse_mode != 'v1':
                    prep.update({'ht0': sr_tc.pack_for(self.head_torso_block.conv0, wsel[:, 0]), 'ht1': sr_tc.pack_for(self.head_torso_block.conv1, wsel[:, 1]),
                                 'htrgb': self.head_torso_block.torgb.folded_weight(wsel[:, 2])})
            plain = self._plain()
            x0 = sr_tc.to_nhwc_f16(x, self.input_resolution)
            rgb0 = self._resize(rgb, self.input_resolution) if rgb.shape[-1] != self.input_resolution else capi.f32(rgb)
            rgb_256 = self._resize(rgb0, 256)
            weights_256 = self._resize(weights_img.detach(), 256)
            cc = self._clip_cache
            if cc is None:
                ref_torso_256, ref_bg_256 = self._aa_down2(ref_torso_rgb), self._aa_down2(ref_bg_rgb)
            else:                                                        # per-clip constants, one frame broadcast over the batch (0.8 MB copies)
                ref_torso_256, ref_bg_256 = cc['ref_torso_256'].expand(N, -1, -1, -1).contiguous(), cc['ref_bg_256'].expand(N, -1, -1, -1).contiguous()
        main, Nw = prep['main'], prep['main'].Nw
        b0, b1, hb = self.block0, self.block1, getattr(self, 'head_torso_block', None)
        # block0: 128^2 -> 256^2 head features + head rgb
        a0 = sr_tc.layer(x0, b0.conv0, main.wp[0], 2)
        xh = torch.empty(N, 256, 256, 256, device=x.device, dtype=torch.float16)
        rgb_h = torch.empty(N, 3, 256, 256, device=x.device)
        with capi.region('sr_conv'):
            capi.check(L.r3dp_sr_tc_layer_torgb(capi.ptr(a0, torch.float16), capi.ptr(main.wp[1], torch.float16), capi.ptr(capi.f32(b0.conv1.bias)),
                                                capi.ptr(main.wrgb0), capi.ptr(capi.f32(b0.torgb.bias)), capi.ptr(rgb0), N, Nw, 256, 256, 256, 256,
                                                capi.ptr(xh, torch.float16), capi.ptr(rgb_h), capi.stream()))
        # torso warper: the caller's PyTorch module (opaque child, sr_with_ref.py:84-87)
        with capi.region('torso_model'):
            rgb_torso, facev2v_ret = self.torso_model(ref_torso_256, segmap, kp_s, kp_d, rgb_256.detach(), weights_256.detach(), cal_loss=True,
                                                      target_torso_mask=target_torso_mask)
        x_torso = self._conv(sr_tc.to_nhwc_f16(facev2v_ret['deformed_torso_hid'], 256), plain['te'], 0)               # 1x1, 64 -> 256
        if cc is None:
            x_bg = self._conv(self._conv(self._conv(sr_tc.to_nhwc_f16(ref_bg_256, 256), plain['bg0'], 2), plain['bg2'], 2), plain['bg4'], 0)
        else:
            x_bg = cc['x_bg']                                            # [1,256,256,256] fp16, read by every frame of the batch
        thr = float(self.hparams['htbsr_head_threshold'])
        if self.fuse_mode == 'v1':
            # head/torso fusion v1 (sr_with_ref.py:96-98): plain alpha blend of the rgb images AND of the feature maps; no fusing convs, no head_torso_block
            alpha = weights_256
            rgb_p2 = self._blend(rgb_h, rgb_torso, alpha)
            xp = torch.empty(N, 256, 256, 256, device=x.device, dtype=torch.float16)
            capi.check(L.r3dp_sr_alpha_mix(capi.ptr(xh, torch.float16), xh.shape[-1], capi.ptr(x_torso, torch.float16), x_torso.shape[-1], capi.ptr(alpha), 256,
                                           N, 256, 256, capi.ptr(xp, torch.float16), capi.stream()))
        else:
            if self.fuse_mode == 'v3':
                # sr_with_ref.py:129-132: a 3-conv net post-processes the head mask from (head rgb, weights, torso rgb); capped by the weights.  The net runs
                # on the tensor cores with SPLIT fp16 operands (fp32-grade): its output is compared with thresholds below, fp16 noise would flip pixels
                inp7 = torch.cat([rgb_h.clamp(-1, 1) / 2 + 0.5, weights_256, capi.f32(rgb_torso).clamp(-1, 1) / 2 + 0.5], dim=1)
                t = sr_tc.to_nhwc_f16(inp7, 256, split=True)
                t = self._conv(self._conv(self._conv(t, plain['ap0'], 2, split=True), plain['ap2'], 2, split=True), plain['ap4'], 0, split=True)
                alpha = torch.empty(N, 1, 256, 256, device=x.device)
                capi.check(L.r3dp_sr_alpha_gate(capi.ptr(t, torch.float16), t.shape[-1], t.shape[-1] // 2, capi.ptr(weights_256), N, 256, 256, capi.ptr(alpha),
                                                capi.stream()))
                if not self.training:                              # :141-143: batch-wide 5 % quantile of the mask values above 0.05 (a host-side scalar, as in the reference)
                    sel = alpha[alpha > 0.05]
                    if sel.numel() > 0:
                        thr = max(float(sel.quantile(0.05)), thr)
            else:
                alpha = weights_256                                 # v2, sr_with_ref.py:108-109 (the masked assignment is a no-op)
            # alpha-cat fusion of the head and torso features (sr_with_ref.py:110-113 | 133-136)
            rgb_p = self._blend(rgb_h, rgb_torso, alpha)
            xf = self._conv(self._conv(self._alpha_cat(xh, 256, x_torso, 256, alpha), plain['fh0'], 2), plain['fh2'], 0)
            c0 = sr_tc.layer(xf, hb.conv0, prep['ht0'], 1)
            xp = torch.empty(N, 256, 256, 256, device=x.device, dtype=torch.float16)
            rgb_p2 = torch.empty(N, 3, 256, 256, device=x.device)
            with capi.region('sr_conv'):
                capi.check(L.r3dp_sr_tc_layer_torgb_noup(capi.ptr(c0, torch.float16), capi.ptr(prep['ht1'], torch.float16), capi.ptr(capi.f32(hb.conv1.bias)),
                                                         capi.ptr(prep['htrgb']), capi.ptr(capi.f32(hb.torgb.bias)), capi.ptr(rgb_p), N, Nw, 256, 256, 256, 256,
                                                         capi.ptr(xp, torch.float16), capi.ptr(rgb_p2), capi.stream()))
        # person / background fusion, sr_with_ref.py:115-124
        occ = capi.f32(facev2v_ret['occlusion_2'])
        torso_occ = occ if occ.shape[-1] == 256 else self._resize(occ, 256)
        person = torch.empty(N, 1, 256, 256, device=x.device)
        capi.check(L.r3dp_sr_person_occlusion(capi.ptr(alpha), capi.ptr(torso_occ), thr, N, 256, 256,
                                              capi.ptr(person), capi.stream()))
        rgb_f = self._blend(rgb_p2, ref_bg_256, person)
        xg = self._conv(self._conv(self._conv(self._alpha_cat(xp, 256, x_bg, 256, person), plain['ff0'], 2), plain['ff2'], 2), plain['ff4'], 0)
        # block1: 256^2 -> 512^2
        a2 = sr_tc.layer(xg, b1.conv0, main.wp[2], 2)
        out = torch.empty(N, 3, 512, 512, device=x.device)
        with capi.region('sr_conv'):
            capi.check(L.r3dp_sr_tc_last_layer(capi.ptr(a2, torch.float16), capi.ptr(main.wp[3], torch.float16), capi.ptr(capi.f32(b1.conv1.bias)),
                                               capi.ptr(main.wrgb1), capi.ptr(capi.f32(b1.torgb.bias)), capi.ptr(rgb_f), N, Nw, 128, 512, 512,
                                               capi.ptr(out), capi.stream()))
        return out, facev2v_ret
