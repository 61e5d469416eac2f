"""RenderHead — the part of OSAvatarSECC_Img2plane.synthesis() that follows plane production
(modules/real3d/secc_img2plane.py:93-137 with _forward_sr from img2plane_baseline.py:140-147): cameras + tri-planes ->
rays -> fused render -> feature image -> super-resolution -> the reference's `ret` dict."""
from __future__ import annotations

from typing import Dict, Optional

import torch

from .decoder import OSGDecoder
from .ray_sampler import RaySampler
from .renderer import ImportanceRenderer
from .superresolution import SuperresolutionHybrid8XDC
from .sr_with_ref import SuperresolutionHybrid8XDC_Warp

# defaults follow the reference configs (egs/egs_bases/eg3d/base.yaml:39-40: 48 coarse + 48 importance samples); BASELINE.json's
# configs 1-4 are quoted at 48 samples/ray, so bench.py / the fixtures pass num_samples_fine=0 explicitly
DEFAULT_HPARAMS = {
    'neural_rendering_resolution': 64, 'w_dim': 512, 'final_resolution': 512, 'triplane_hid_dim': 32,
    'num_samples_coarse': 48, 'num_samples_fine': 48, 'box_warp': 1.0, 'base_channel': 32768, 'max_channel': 512,
    'enable_rescale_plane_regulation': False, 'triplane_feature_type': 'triplane', 'mask_invalid_rays': False,
}


class RenderHead(torch.nn.Module):
    """Child module names (`decoder`, `superresolution`, `renderer`, `ray_sampler`) match the reference model, so the
    corresponding slices of a released checkpoint load unchanged."""

    def __init__(self, hp: Optional[dict] = None, sr_mode: str = 'fp32', torso_model: Optional[torch.nn.Module] = None):
        """torso_model given (or hp['torso'] true) -> the OSAvatarSECC_Img2plane_Torso head (secc_img2plane_torso.py:7-18): the SR module is
        SuperresolutionHybrid8XDC_Warp and synthesis() needs `cond` with ref_torso_img, bg_img, segmap, kp_s, kp_d."""
        super().__init__()
        self.hparams = dict(DEFAULT_HPARAMS, **(hp or {}))
        hp = self.hparams
        self.torso = torso_model is not None or bool(hp.get('torso', False))
        self.neural_rendering_resolution = hp['neural_rendering_resolution']
        c = hp['triplane_hid_dim']
        self.decoder = OSGDecoder(c, {'decoder_lr_mul': 1, 'decoder_output_dim': c})
        sr_kwargs = dict(channels=c, img_resolution=hp['final_resolution'], sr_num_fp16_res=0, sr_antialias=True, channel_base=hp['base_channel'],
                         channel_max=hp['max_channel'], fused_modconv_default='inference_only')
        if self.torso:                                               # tensor-core only: 'tc_exact' is kept, every other mode runs as 'tc'
            torso_mode = 'tc_exact' if sr_mode == 'tc_exact' else 'tc'
            self.superresolution = SuperresolutionHybrid8XDC_Warp(hp=hp, torso_model=torso_model, sr_mode=torso_mode, **sr_kwargs)
        else:
            self.superresolution = SuperresolutionHybrid8XDC(sr_mode=sr_mode, **sr_kwargs)
        self.renderer = ImportanceRenderer(hp=hp)
        self.ray_sampler = RaySampler()
        self.rendering_kwargs = {
            'image_resolution': hp['final_resolution'], 'disparity_space_sampling': False, 'clamp_mode': 'softplus',
            'superresolution_noise_mode': 'none', 'sr_antialias': True, 'depth_resolution': hp['num_samples_coarse'],
            'depth_resolution_importance': hp['num_samples_fine'], 'ray_start': 'auto', 'ray_end': 'auto',
            'box_warp': hp.get('box_warp', 1.0), 'white_back': False,
        }

    def _render(self, planes, camera: torch.Tensor, render_overrides: Dict):
        cam2world = camera[:, :16].reshape(-1, 4, 4)
        intrinsics = camera[:, 16:25].reshape(-1, 3, 3)
        ray_o, ray_d = self.ray_sampler(cam2world, intrinsics, self.neural_rendering_resolution)
        opts = dict(self.rendering_kwargs, **render_overrides)
        return self.renderer(planes, self.decoder, ray_o, ray_d, opts)

    def _lean(self) -> bool:
        return self.superresolution.sr_mode in ('tc', 'tc_exact') and not self.hparams.get('mask_invalid_rays', False)

    def _lean_sr_inputs(self, feat: torch.Tensor):
        """The renderer's channels-last output as the SR's lean inputs: (rgb view, feature view, x_nhwc, ones_ws) - no NCHW copies, and
        ones_ws is allocated once per batch size."""
        res = self.neural_rendering_resolution
        N = feat.shape[0]
        x_nhwc = feat.view(N, res, res, feat.shape[-1])
        if getattr(self, '_ones_ws', None) is None or self._ones_ws.shape[0] != N or self._ones_ws.device != feat.device:
            self._ones_ws = torch.ones(N, 14, self.hparams['w_dim'], device=feat.device)
        return x_nhwc[..., :3].permute(0, 3, 1, 2), x_nhwc.permute(0, 3, 1, 2), x_nhwc, self._ones_ws

    def _torso_pre_from(self, feat, wsum, cond: Dict, out_uint8: bool) -> Dict:
        rgb, x, x_nhwc, ones_ws = self._lean_sr_inputs(feat)
        res = self.neural_rendering_resolution
        return self.superresolution.forward_pre(rgb, x, ones_ws, cond['ref_torso_img'], cond['bg_img'], wsum.view(feat.shape[0], 1, res, res), cond['segmap'],
                                                cond['kp_s'], cond['kp_d'], cond.get('target_torso_mask'), noise_mode='none', x_nhwc=x_nhwc, wsum=wsum,
                                                rgb_from_x=True, out_clamp=True, out_uint8=out_uint8)

    @torch.no_grad()
    def torso_pre(self, planes, camera: torch.Tensor, cond: Dict, out_uint8: bool = False, keep_render: bool = False, **render_overrides) -> Dict:
        """Lean torso step up to the torso_model call: render, then the first half of the torso SR head (forward_pre) on the renderer's
        channels-last output.  Continue with superresolution.run_torso(state) and superresolution.forward_post(state, ...) -> the image,
        clamped to [-1,1] (uint8 HWC frames with out_uint8).  keep_render: the state also holds the render's channels-last features
        'render_feat' [N,4096,C] and depths 'render_depth' [N,4096,1]."""
        feat, depth, wsum, _ = self._render(planes, camera, render_overrides)
        st = self._torso_pre_from(feat, wsum, cond, out_uint8)
        if keep_render:
            st['render_feat'], st['render_depth'] = feat, depth
        return st

    @torch.no_grad()
    def synthesis(self, planes, camera: torch.Tensor, ret: Optional[Dict] = None, cond: Optional[Dict] = None, **render_overrides) -> Dict[str, torch.Tensor]:
        """planes [N,3,C,H,W], camera [N,25] -> ret dict with the reference's keys (secc_img2plane.py:134-136).
        lean=True (tensor-core SR, no mask_invalid_rays): the frame-loop fast path of FrameEngine; only ret['image'] (plus ret['is_ray_valid']
        for the plain head) is filled, clamped to [-1,1], or as uint8 HWC frames [N,512,512,3] with out_uint8=True; keep_render=True adds the
        render's channels-last features ret['render_feat'] [N,4096,C] and depths ret['render_depth'] [N,4096,1] (no copies)."""
        if ret is None:
            ret = {}
        res = self.neural_rendering_resolution
        lean = bool(render_overrides.pop('lean', False))
        out_uint8 = bool(render_overrides.pop('out_uint8', False))
        keep_render = bool(render_overrides.pop('keep_render', False))
        feat, depth, wsum, valid = self._render(planes, camera, render_overrides)
        N = feat.shape[0]
        if lean and self._lean():
            if keep_render:
                ret['render_feat'], ret['render_depth'] = feat, depth
            # frame-loop fast path (FrameEngine): only ret['image'] is wanted, so the NCHW copies of the feature / weight images, the
            # clamped raw image and the per-call ones_ws are not materialised; the SR reads the renderer's channels-last output directly.
            # The clamp (and, if asked, the uint8 HWC conversion of real3d_infer.py:519) happen in the last SR epilogue
            if self.torso:
                sr = self.superresolution
                st = self._torso_pre_from(feat, wsum, cond, out_uint8)
                rgb_torso, facev2v_ret = sr.run_torso(st)
                ret['image'] = sr.forward_post(st, rgb_torso, facev2v_ret)
                return ret
            rgb, x, x_nhwc, ones_ws = self._lean_sr_inputs(feat)
            sr_image = self.superresolution(rgb, x, ones_ws, noise_mode='none', x_nhwc=x_nhwc, out_clamp=True, out_uint8=out_uint8, rgb_from_x=True)
            ret.update({'image': sr_image, 'is_ray_valid': valid})
            return ret
        if out_uint8:
            raise NotImplementedError('uint8 frames come from the lean tensor-core path (FrameEngine); the full ret dict is fp32 like the reference')
        feature_image = feat.permute(0, 2, 1).reshape(N, feat.shape[-1], res, res).contiguous()
        weights_image = wsum.permute(0, 2, 1).reshape(N, 1, res, res).contiguous()
        depth_image = depth.permute(0, 2, 1).reshape(N, 1, res, res)
        if self.hparams.get('mask_invalid_rays', False):
            mask = valid.reshape(N, 1, res, res)
            feature_image = torch.where(mask, feature_image, torch.full_like(feature_image, -1.0))
            depth_image = torch.where(mask, depth_image, depth_image[mask].min())
        rgb_image = feature_image[:, :3]
        ret['weights_img'] = weights_image
        ones_ws = torch.ones(N, 14, self.hparams['w_dim'], device=feature_image.device)
        if self.torso:                                               # secc_img2plane_torso.py:13-18
            sr_image, facev2v_ret = self.superresolution(rgb_image, feature_image, ones_ws, cond['ref_torso_img'], cond['bg_img'], weights_image,
                                                         cond['segmap'], cond['kp_s'], cond['kp_d'], cond.get('target_torso_mask'), noise_mode='none')
            ret.update(facev2v_ret)
        else:
            extra = {'x_nhwc': feat.view(N, res, res, feat.shape[-1])} if self.superresolution.sr_mode in ('tc', 'tc_exact') else {}
            sr_image = self.superresolution(rgb_image, feature_image, ones_ws, noise_mode='none', **extra)
        ret.update({'image_raw': rgb_image.clamp(-1, 1), 'image_depth': depth_image, 'image': sr_image.clamp(-1, 1),
                    'image_feature': feature_image[:, 3:], 'plane': planes, 'is_ray_valid': valid})
        return ret

    forward = synthesis
