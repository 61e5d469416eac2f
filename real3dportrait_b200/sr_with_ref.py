"""SuperresolutionHybrid8XDC_Warp — host mirror of modules/real3d/super_resolution/sr_with_ref.py:16-162 (the torso/background
fusing SR head of OSAvatarSECC_Img2plane_Torso, BASELINE config 5).

Same constructor arguments, child-module names (`block0/1`, `torso_encoder`, `bg_encoder`, `head_torso_alpha_predictor`,
`fuse_head_torso_convs`, `head_torso_block`, `fuse_fg_bg_convs`, `torso_model`) and `forward` signature/return as the reference, so
released checkpoints load with strict=True.  The conv stack (782 GFLOP/frame, SURVEY.md §8d) runs on the tensor-core kernels of
csrc/sr_tc.cu; the torso warper `torso_model` (WarpBasedTorsoModelMediaPipe, SURVEY.md §2 #11: out of scope) stays the caller's
PyTorch module and is called as an opaque child exactly where the reference calls it.  Every configuration of the reference class is built:
torso_model_version v1 | v2, weight_fuse True (htbsr_head_weight_fuse_mode v1 | v2 | v3) | False.  The released one
(egs/os_avatar/real3d_orig/secc_img2plane_torso_orig.yaml:26-30) is torso_model_version v2, htbsr_head_weight_fuse_mode v2."""
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
                 torso_stage2: str = 'torch', torso_motion: str = 'torch', **block_kwargs):
        block_kwargs.setdefault('sr_mode', 'tc')
        super().__init__(channels, img_resolution, sr_num_fp16_res, sr_antialias, **block_kwargs)
        if self.sr_mode not in ('tc', 'tc_exact'):
            raise NotImplementedError('the torso head is built on the tensor-core path only (sr_mode="tc" | "tc_exact")')
        if not sr_antialias:
            # sr_with_ref.py:79-82 would down-sample the 512^2 reference images with plain bilinear; _aa_down2 is the antialiased filter
            # (the head's other resizes are up-samplings, where antialias changes nothing)
            raise NotImplementedError('the torso head is built with sr_antialias=True only (its 512 -> 256 resizes are antialiased)')
        hp = dict(hp or {})
        self.hparams = {'torso_model_version': hp.get('torso_model_version', 'v2'), 'htbsr_head_weight_fuse_mode': hp.get('htbsr_head_weight_fuse_mode', 'v2'),
                        'htbsr_head_threshold': float(hp.get('htbsr_head_threshold', 0.9)), 'weight_fuse': hp.get('weight_fuse', True)}
        self.weight_fuse = bool(self.hparams['weight_fuse'])
        # weight_fuse=False concatenates the head, torso and background features unweighted and ignores the fuse mode (sr_with_ref.py:36,158-161)
        self.fuse_mode = self.hparams['htbsr_head_weight_fuse_mode'] if self.weight_fuse else None
        if self.hparams['torso_model_version'] not in ('v1', 'v2') or (self.weight_fuse and self.fuse_mode not in ('v1', 'v2', 'v3')):
            raise NotImplementedError('built: torso_model_version v1 | v2 with weight_fuse=False or htbsr_head_weight_fuse_mode v1 | v2 | v3')
        if torso_model is not None:
            self.torso_model = torso_model                      # the reference's WarpBasedTorsoModelMediaPipe('standard') (model.py for v1, model2.py for v2)
        nn = torch.nn
        self.torso_encoder = nn.Sequential(nn.Conv2d(64, 256, 1, 1, padding=0))
        self.bg_encoder = nn.Sequential(nn.Conv2d(3, 64, 3, 1, padding=1), nn.LeakyReLU(), nn.Conv2d(64, 256, 3, 1, padding=1), nn.LeakyReLU(),
                                        nn.Conv2d(256, 256, 3, 1, padding=1))
        if self.fuse_mode in ('v2', 'v3'):                      # the reference builds these children for every weighted mode but v1 (sr_with_ref.py:36-55)
            self.head_torso_alpha_predictor = nn.Sequential(nn.Conv2d(7, 32, 3, 1, padding=1), nn.LeakyReLU(), nn.Conv2d(32, 32, 3, 1, padding=1),
                                                            nn.LeakyReLU(), nn.Conv2d(32, 1, 3, 1, padding=1), nn.Sigmoid())   # used by v3 only
            self.fuse_head_torso_convs = nn.Sequential(nn.Conv2d(512, 256, 3, 1, padding=1), nn.LeakyReLU(), nn.Conv2d(256, 256, 3, 1, padding=1))
            bk = {k: v for k, v in block_kwargs.items() if k not in ('sr_mode', 'channel_base', 'channel_max')}
            self.head_torso_block = SynthesisBlockNoUp(256, 256, w_dim=512, resolution=256, img_channels=3, is_last=False, use_fp16=False,
                                                       conv_clamp=None, **bk)
        self.fuse_in_dim = 512 if self.weight_fuse else 768      # weight_fuse=False: cat[x, x_torso, x_bg] (sr_with_ref.py:57-58)
        self.fuse_fg_bg_convs = nn.Sequential(nn.Conv2d(self.fuse_in_dim, 64, 1, 1, padding=0), nn.LeakyReLU(), nn.Conv2d(64, 256, 3, 1, padding=1),
                                              nn.LeakyReLU(), nn.Conv2d(256, 256, 3, 1, padding=1))
        self._warper = None
        self.torso_motion = 'torch'
        self.set_torso_stage2(torso_stage2)
        self.set_torso_motion(torso_motion)

    def set_torso_stage2(self, mode: str) -> None:
        """'torch': the caller's torso_model(...) call (the reference's path).  'cuda': the warper's stage 2 (Generator + occlusion_2_predictor)
        on this library's kernels, stage 1 restated in torso_warp.py around the caller's appearance_extractor and motion_field_estimator;
        built for torso_model_version v2 (model2.py) only."""
        if mode not in ('torch', 'cuda'):
            raise ValueError(f"torso_stage2 is 'torch' or 'cuda', got {mode!r}")
        if mode == 'cuda' and self.hparams['torso_model_version'] != 'v2':
            raise NotImplementedError("torso_stage2='cuda' is built for torso_model_version v2 (facev2v_warp/model2.py) only")
        if mode == 'torch' and getattr(self, 'torso_motion', 'torch') == 'cuda':
            raise ValueError("torso_motion='cuda' needs torso_stage2='cuda': call set_torso_motion('torch') first")
        self.torso_stage2 = mode
        self.forget('stage2')

    def set_torso_motion(self, mode: str) -> None:
        """'torch': the warper calls the caller's motion_field_estimator.  'cuda': the estimator (network2.py:162-244) runs on this library's
        3-D convolutions (torso_warp.motion), its compressed source volume cached per clip by begin_clip(segmap=...).  Needs torso_stage2='cuda'
        (the restated stage 1 is where the call is replaced) and MotionFieldEstimator('standard') with torso_kp_num 4 or 9."""
        if mode not in ('torch', 'cuda'):
            raise ValueError(f"torso_motion is 'torch' or 'cuda', got {mode!r}")
        if mode == 'cuda':
            if self.hparams['torso_model_version'] != 'v2':
                raise NotImplementedError("torso_motion='cuda' is built for torso_model_version v2 (facev2v_warp/model2.py) only")
            if self.torso_stage2 != 'cuda':
                raise ValueError("torso_motion='cuda' needs torso_stage2='cuda'")
            tm = getattr(self, 'torso_model', None)
            if tm is not None:
                from . import torso_warp
                err = torso_warp.estimator_shape_error(tm.motion_field_estimator)
                if err is not None:
                    raise NotImplementedError(f"torso_motion='cuda' is built for MotionFieldEstimator('standard'): {err}")
        self.torso_motion = mode
        self.forget('motion')

    def _motion_weights(self):
        """Folded + packed estimator weights (torso_warp.MotionWeights), keyed like _stage2_weights(); None unless torso_motion='cuda'."""
        if self.torso_motion != 'cuda':
            return None
        from . import torso_warp
        sp, mfe = self._split, self.torso_model.motion_field_estimator
        return self.prepared('motion', lambda: torso_warp.MotionWeights(mfe, sp), sp, watch=(mfe,))

    def _stage2_weights(self):
        """Folded + packed stage-2 weights, rebuilt when the mode, the device or any of the warper's parameters / buffers changed (a
        load_state_dict of the head or of torso_model alone, an optimizer step, .to(device)).  The per-clip appearance cache is not re-keyed:
        it holds until the next begin_clip(), like the head's other clip constants."""
        from . import torso_warp
        sp, tm = self._split, self.torso_model
        mods = (tm.deform_based_generator, tm.occlusion_2_predictor)
        return self.prepared('stage2', lambda: torso_warp.Stage2Weights(*mods, sp), sp, watch=mods)

    @property
    def _split(self) -> bool:
        """sr_mode='tc_exact': every activation of the head is a [hi | lo] pair of fp16 tensors, every conv runs with split operands."""
        return self.sr_mode == 'tc_exact'

    # ---- weight preparation ------------------------------------------------------------------------------------------------
    def _plain(self) -> Dict[str, tuple]:
        return self.prepared('plain', self._build_plain, self._split)

    def _build_plain(self) -> Dict[str, tuple]:
        sp = self._split
        te, bg, ff = self.torso_encoder, self.bg_encoder, self.fuse_fg_bg_convs
        P = {
            'te': _pack_plain(te[0], 64, split=sp), 'bg0': _pack_plain(bg[0], 64, split=sp), 'bg2': _pack_plain(bg[2], 128, split=sp),
            'bg4': _pack_plain(bg[4], 256, split=sp),
            'ff0': _pack_plain(ff[0], self.fuse_in_dim, split=sp), 'ff2': _pack_plain(ff[2], 128, split=sp), 'ff4': _pack_plain(ff[4], 256, split=sp),
        }
        if self.fuse_mode in ('v2', 'v3'):
            fh = self.fuse_head_torso_convs
            P.update({'fh0': _pack_plain(fh[0], 512, split=sp), 'fh2': _pack_plain(fh[2], 256, split=sp)})
        if self.fuse_mode == 'v3':                             # the mask predictor runs with split fp16 operands (its output is thresholded)
            ap = self.head_torso_alpha_predictor
            P.update({'ap0': sr_tc.pack_plain(ap[0], 64, split=True), 'ap2': sr_tc.pack_plain(ap[2], 128, split=True),
                      'ap4': sr_tc.pack_plain(ap[4], 128, split=True)})
        return P

    def prepare_styles(self, wsel: torch.Tensor) -> Dict:
        """Folded + packed weights of block0/1 and head_torso_block for styles wsel [Nw,3,512] (with static_styles, prepared_styles()
        keeps those of the all-ones styles)."""
        sp = self._split
        prep = {'main': sr_tc.Prepared(self, wsel, sp)}
        if self.fuse_mode in ('v2', 'v3'):
            prep.update({'ht0': sr_tc.pack_for(self.head_torso_block.conv0, wsel[:, 0], sp), 'ht1': sr_tc.pack_for(self.head_torso_block.conv1, wsel[:, 1], sp),
                         'htrgb': self.head_torso_block.torgb.folded_weight(wsel[:, 2])})
        return prep

    @staticmethod
    def _conv(x16: torch.Tensor, packed, act: int, split: bool = False) -> torch.Tensor:
        """sr_tc.conv_plain (no residual), timed in the 'sr_conv' profiler stage."""
        with capi.region('sr_conv'):
            return sr_tc.conv_plain(x16, packed, act, split=split)

    # ---- per-clip constants (SURVEY.md §8f #2) -------------------------------------------------------------------------------------------
    @torch.no_grad()
    def begin_clip(self, ref_torso_rgb: torch.Tensor, ref_bg_rgb: torch.Tensor, batch: Optional[int] = None, in_place: bool = False,
                   segmap: Optional[torch.Tensor] = None) -> bool:
        """Hoist what the reference recomputes for every frame although it only depends on the clip's reference images
        (sr_with_ref.py:77-90): the two antialiased 512->256 resizes and bg_encoder(ref_bg) (96.9 GFLOP/frame).  ref_* [1,3,512,512].
        Until end_clip(), forward() ignores its ref_torso_rgb / ref_bg_rgb arguments and uses these.
        batch: also keep the [batch,3,256,256] broadcasts of the two resized images, read by every call with that batch instead of
        copies made per call.  in_place: when a clip with the same mode and batch is already begun, write the new constants into its
        tensors (CUDA graphs captured against them then render the new clip).  Returns True when the constants were refilled in place.
        segmap [1,6,512,512] with torso_stage2='cuda': also keep the warper's per-clip part (torso_warp.appearance: appearance_extractor of
        the reference torso image, the dilated torso mask, the 64^2 segmap, the volume in NDHWC; with torso_motion='cuda' the estimator's
        compressed source volume too); forward() then ignores its segmap argument."""
        assert ref_torso_rgb.shape[0] == 1 and ref_bg_rgb.shape[0] == 1, 'one reference image per clip'
        plain, sp = self._plain(), self._split
        t256, b256 = self._aa_down2(ref_torso_rgb), self._aa_down2(ref_bg_rgb)
        cc = {'ref_torso_256': t256, 'ref_bg_256': b256, 'x_bg': self._bg_features(b256, plain, sp), 'batch': None, 'torso_app': None}
        if segmap is not None and self.torso_stage2 == 'cuda':
            from . import torso_warp
            assert segmap.shape[0] == 1, 'one segmap per clip'
            cc['torso_app'] = torso_warp.appearance(self.torso_model, t256, segmap, self._motion_weights())
        if batch is not None:
            cc['batch'] = (t256.expand(batch, -1, -1, -1).contiguous(), b256.expand(batch, -1, -1, -1).contiguous())
        old = self._clip_cache
        if in_place and old is not None and (old['batch'] is None) == (batch is None) and \
                (batch is None or old['batch'][0].shape[0] == batch) and (old['torso_app'] is None) == (cc['torso_app'] is None) and \
                (cc['torso_app'] is None or old['torso_app'].keys() == cc['torso_app'].keys()):
            for k in ('ref_torso_256', 'ref_bg_256', 'x_bg'):
                old[k].copy_(cc[k])
            if cc['torso_app'] is not None:                         # a graph that captured the warper reads these tensors by address
                for k, v in cc['torso_app'].items():
                    old['torso_app'][k].copy_(v)
            if batch is not None:
                for dst, src in zip(old['batch'], cc['batch']):
                    dst.copy_(src)
            return True
        self.store('clip', cc, sp)
        return False

    def end_clip(self) -> None:
        self.forget('clip')

    @property
    def _clip_cache(self) -> Optional[Dict]:
        """The constants of the clip begun in the current sr_mode (None outside a clip)."""
        return self.cached('clip', self._split)

    def _bg_features(self, ref_bg_256, plain, split: bool) -> torch.Tensor:
        """bg_encoder(ref_bg) on the tensor cores: [N,256,256,256] fp16 ([N,256,256,512] = [hi | lo] when split)."""
        x = sr_tc.to_nhwc_f16(ref_bg_256, 256, split)
        return self._conv(self._conv(self._conv(x, plain['bg0'], 2, split), plain['bg2'], 2, split), plain['bg4'], 0, split)

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
        kp_s/kp_d [N,68,3] -> (rgb [N,3,512,512], facev2v_ret)   (sr_with_ref.py:67-162).
        Optional, as for the plain head (tensor-core path): x_nhwc = the renderer's channels-last features [N,h,w,C] with rgb_from_x=True
        (rgb == x[:, :3]) and wsum = its channels-last weights [N,h*w,1] - the inputs are then read in place by one launch;
        out_clamp: the image leaves the last epilogue clamped to [-1,1]; out_uint8: it leaves as uint8 HWC frames [N,512,512,3]."""
        st = self.forward_pre(rgb, x, ws, ref_torso_rgb, ref_bg_rgb, weights_img, segmap, kp_s, kp_d, target_torso_mask, **block_kwargs)
        rgb_torso, facev2v_ret = self.run_torso(st)
        return self.forward_post(st, rgb_torso, facev2v_ret), facev2v_ret

    def forward_pre(self, rgb, x, ws, ref_torso_rgb, ref_bg_rgb, weights_img, segmap, kp_s, kp_d, target_torso_mask=None, **block_kwargs) -> Dict:
        """First half of forward(), up to the torso_model call: input preparation, block0 and the warper's inputs.  Returns the state that
        run_torso() and forward_post() take; every tensor in it is written on the current stream (a CUDA graph may capture this half)."""
        if getattr(self, 'torso_model', None) is None:
            raise RuntimeError('SuperresolutionHybrid8XDC_Warp needs its torso_model child (the reference WarpBasedTorsoModelMediaPipe); '
                               'pass torso_model=... to the constructor')
        if block_kwargs.get('noise_mode', 'none') != 'none':
            raise NotImplementedError("only noise_mode='none' is on the inference path")
        x_nhwc, wsum = block_kwargs.pop('x_nhwc', None), block_kwargs.pop('wsum', None)
        rgb_from_x = bool(block_kwargs.pop('rgb_from_x', False))
        if x_nhwc is not None and not (rgb_from_x and wsum is not None):
            raise NotImplementedError('x_nhwc is the lean hand-off from the renderer: it needs rgb_from_x=True and wsum (the channels-last weights)')
        N = rgb.shape[0]
        if ref_torso_rgb.shape[-1] != 512 or ref_bg_rgb.shape[-1] != 512:
            raise NotImplementedError('reference images must be 512x512 (antialiased 1/2 resize is the only down-scaling built)')
        ws3 = ws[:, -1:, :].expand(N, 3, -1)
        sp = self._split
        with capi.region('sr_prep'):
            prep = self.prepared_styles()
            if prep is None:
                shared = N == 1 or getattr(self, 'assume_shared_styles', False)
                prep = self.prepare_styles(ws3[:1] if shared else ws3)
            plain = self._plain()
            R = self.input_resolution
            if x_nhwc is not None:                                       # one launch, bit-identical to the three below
                xn = capi.f32(x_nhwc)
                _, h, w, Cc = xn.shape
                x0 = sr_tc.activation(N, R, R, (Cc + 63) // 64 * 64, sp, xn.device)
                rgb0 = torch.empty(N, 3, R, R, device=xn.device)
                rgb_256 = torch.empty(N, 3, 256, 256, device=xn.device)
                weights_256 = torch.empty(N, 1, 256, 256, device=xn.device)
                capi.check(capi.lib().r3dp_sr_warp_input(capi.ptr(xn), capi.ptr(capi.f32(wsum)), N, Cc, h, w, R, capi.ptr(x0, torch.float16), capi.ptr(rgb0),
                                                         capi.ptr(rgb_256), capi.ptr(weights_256), int(sp), capi.stream()))
            else:
                x0 = sr_tc.to_nhwc_f16(x, R, sp)
                rgb0 = self._resize(rgb, R) if rgb.shape[-1] != R else capi.f32(rgb)
                rgb_256 = self._resize(rgb0, 256)
                weights_256 = self._resize(weights_img.detach(), 256)
            cc = self._clip_cache                                        # None when begun in another sr_mode: run uncached
            if cc is None:
                ref_torso_256, ref_bg_256 = self._aa_down2(ref_torso_rgb), self._aa_down2(ref_bg_rgb)
            elif cc['batch'] is not None and cc['batch'][0].shape[0] == N:  # per-clip constants, broadcast over the batch once per clip
                ref_torso_256, ref_bg_256 = cc['batch']
            else:                                                        # per-clip constants, one frame broadcast over the batch (0.8 MB copies)
                ref_torso_256, ref_bg_256 = cc['ref_torso_256'].expand(N, -1, -1, -1).contiguous(), cc['ref_bg_256'].expand(N, -1, -1, -1).contiguous()
        xh, rgb_h = sr_tc.block0(self.block0, prep['main'], x0, rgb0)   # 128^2 -> 256^2 head features + head rgb
        return {'N': N, 'split': sp, 'prep': prep, 'plain': plain, 'cc': cc, 'device': x.device, 'xh': xh, 'rgb_h': rgb_h, 'ref_bg_256': ref_bg_256,
                'weights_256': weights_256, 'out_clamp': bool(block_kwargs.pop('out_clamp', False)), 'out_uint8': bool(block_kwargs.pop('out_uint8', False)),
                'torso_args': (ref_torso_256, segmap, kp_s, kp_d, rgb_256, weights_256), 'target_torso_mask': target_torso_mask}

    def run_torso(self, st: Dict):
        """The torso warper: the caller's PyTorch module (opaque child, sr_with_ref.py:84-87) -> (rgb_torso, facev2v_ret).
        torso_model_version v1 (model.py) takes no head weights image; v2 (model2.py) does."""
        ref_torso_256, segmap, kp_s, kp_d, rgb_256, weights_256 = st['torso_args']
        if self.torso_stage2 == 'cuda':
            from . import torso_warp
            if self._warper is None or self._warper.tm is not self.torso_model:
                self._warper = torso_warp.TorsoWarper(self.torso_model)
            cc = st['cc']
            with capi.region('torso_model'):
                return self._warper(self._stage2_weights(), ref_torso_256, segmap, kp_s, kp_d, rgb_256.detach(), weights_256.detach(),
                                    app=cc.get('torso_app') if cc is not None else None, motion_wts=self._motion_weights())
        with capi.region('torso_model'):
            if self.hparams['torso_model_version'] == 'v1':
                return self.torso_model(ref_torso_256, segmap, kp_s, kp_d, rgb_256.detach(), cal_loss=True, target_torso_mask=st['target_torso_mask'])
            return self.torso_model(ref_torso_256, segmap, kp_s, kp_d, rgb_256.detach(), weights_256.detach(), cal_loss=True,
                                    target_torso_mask=st['target_torso_mask'])

    def forward_post(self, st: Dict, rgb_torso: torch.Tensor, facev2v_ret: Dict) -> torch.Tensor:
        """Second half of forward(), after the torso_model call: torso encoder, background features, head / torso / background fusion
        and block1 -> the image (fp32 [N,3,512,512], or uint8 [N,512,512,3] when forward_pre() got out_uint8).  weight_fuse=False reads neither
        rgb_torso nor facev2v_ret['occlusion_2']."""
        L = capi.lib()
        N, sp, prep, plain, cc, dev = st['N'], st['split'], st['prep'], st['plain'], st['cc'], st['device']
        xh, rgb_h, weights_256 = st['xh'], st['rgb_h'], st['weights_256']
        hb = getattr(self, 'head_torso_block', None)
        x_torso = self._conv(sr_tc.to_nhwc_f16(facev2v_ret['deformed_torso_hid'], 256, sp), plain['te'], 0, sp)       # 1x1, 64 -> 256
        if cc is None:
            x_bg = self._bg_features(st['ref_bg_256'], plain, sp)
        else:
            x_bg = cc['x_bg']                                            # [1,256,256,256 (x2 split)] fp16, read by every frame of the batch
        if not self.weight_fuse:
            # sr_with_ref.py:159-161: cat[x, x_torso, x_bg] unweighted, and block1 without a skip image
            return self._fg_bg_block1(st, sr_tc.cat3(xh, x_torso, x_bg, sp), None)
        thr = float(self.hparams['htbsr_head_threshold'])
        if self.fuse_mode == 'v1':
            # head/torso fusion v1 (sr_with_ref.py:96-98): plain alpha blend of the rgb images AND of the feature maps; no fusing convs, no head_torso_block
            alpha = weights_256
            rgb_p2 = self._blend(rgb_h, rgb_torso, alpha)
            xp = sr_tc.alpha_mix(xh, x_torso, alpha, sp)
        else:
            if self.fuse_mode == 'v3':
                # sr_with_ref.py:129-132: a 3-conv net post-processes the head mask from (head rgb, weights, torso rgb); capped by the weights.  The net runs
                # on the tensor cores with SPLIT fp16 operands (fp32-grade): its output is compared with thresholds below, fp16 noise would flip pixels
                inp7 = torch.cat([rgb_h.clamp(-1, 1) / 2 + 0.5, weights_256, capi.f32(rgb_torso).clamp(-1, 1) / 2 + 0.5], dim=1)
                t = sr_tc.to_nhwc_f16(inp7, 256, split=True)
                t = self._conv(self._conv(self._conv(t, plain['ap0'], 2, split=True), plain['ap2'], 2, split=True), plain['ap4'], 0, split=True)
                alpha = torch.empty(N, 1, 256, 256, device=dev)
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
            xf = self._conv(self._conv(sr_tc.alpha_cat(xh, 256, x_torso, 256, alpha, sp), plain['fh0'], 2, sp), plain['fh2'], 0, sp)
            c0 = sr_tc.layer(xf, hb.conv0, prep['ht0'], 1, sp)
            xp, rgb_p2 = sr_tc.layer_torgb(c0, hb, prep['ht1'], prep['htrgb'], rgb_p, sp, noup=True)
        # person / background fusion, sr_with_ref.py:115-124
        occ = capi.f32(facev2v_ret['occlusion_2'])
        torso_occ = occ if occ.shape[-1] == 256 else self._resize(occ, 256)
        person = torch.empty(N, 1, 256, 256, device=dev)
        capi.check(L.r3dp_sr_person_occlusion(capi.ptr(alpha), capi.ptr(torso_occ), thr, N, 256, 256,
                                              capi.ptr(person), capi.stream()))
        rgb_f = self._blend(rgb_p2, st['ref_bg_256'], person)
        return self._fg_bg_block1(st, sr_tc.alpha_cat(xp, 256, x_bg, 256, person, sp), rgb_f)

    def _fg_bg_block1(self, st: Dict, xg: torch.Tensor, rgb_f: Optional[torch.Tensor]) -> torch.Tensor:
        """fuse_fg_bg_convs and block1 on the fused features xg; rgb_f = block1's skip image (None: no skip, the image is ToRGB alone)."""
        sp, plain = st['split'], st['plain']
        xg = self._conv(self._conv(self._conv(xg, plain['ff0'], 2, sp), plain['ff2'], 2, sp), plain['ff4'], 0, sp)
        # block1: 256^2 -> 512^2; with out_uint8 the last epilogue writes the video frames (real3d_infer.py:515-519)
        return sr_tc.block1(self.block1, st['prep']['main'], xg, rgb_f, st['out_clamp'], st['out_uint8'])
