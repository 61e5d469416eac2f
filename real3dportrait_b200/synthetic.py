"""Deterministic synthetic inputs for the render + SR path (SURVEY.md §8d): tri-planes, look-at cameras, jitter
uniforms and random-init decoder / SR parameters.  Everything is drawn on the CPU from seeded generators so the
CPU oracle, the golden fixtures and the GPU path see identical bits; callers upload with `.cuda()`.

Camera convention follows the reference's pose sampler (modules/eg3ds/camera_utils/pose_sampler.py:28-36,
94-131,174-204): camera on a sphere of radius 2.7 around `lookat`, y up, 25-vector = row-major c2w (16) +
row-major normalised intrinsics (9) with focal 4.2647 and principal point 0.5."""
from __future__ import annotations

import math
from typing import Dict, Tuple

import torch

FOCAL = 4.2647
SR_CHANNELS = {'block0': (32, 256), 'block1': (256, 128)}


def lookat_camera(pitch: torch.Tensor, yaw: torch.Tensor, lookat=(0.0, 0.0, 0.2), radius: float = 2.7) -> torch.Tensor:
    """pitch[N], yaw[N] (radians) -> camera[N,25]."""
    pitch = pitch.float().reshape(-1)
    yaw = yaw.float().reshape(-1)
    n = pitch.shape[0]
    theta = yaw + math.pi / 2
    v = (pitch + math.pi / 2).clamp(1e-5, math.pi - 1e-5) / math.pi
    phi = torch.arccos(1 - 2 * v)
    origin = torch.stack([radius * torch.sin(phi) * torch.cos(math.pi - theta),
                          radius * torch.cos(phi),
                          radius * torch.sin(phi) * torch.sin(math.pi - theta)], dim=1)
    look = torch.tensor(lookat, dtype=torch.float32).expand(n, 3)
    fwd = torch.nn.functional.normalize(look - origin, dim=1)
    up0 = torch.tensor([0.0, 1.0, 0.0]).expand(n, 3)
    right = -torch.nn.functional.normalize(torch.cross(up0, fwd, dim=1), dim=1)
    up = torch.nn.functional.normalize(torch.cross(fwd, right, dim=1), dim=1)
    c2w = torch.eye(4).repeat(n, 1, 1)
    c2w[:, :3, 0], c2w[:, :3, 1], c2w[:, :3, 2], c2w[:, :3, 3] = right, up, fwd, origin
    K = torch.tensor([[FOCAL, 0, 0.5], [0, FOCAL, 0.5], [0, 0, 1.0]]).reshape(1, 9).repeat(n, 1)
    return torch.cat([c2w.reshape(n, 16), K], dim=1)


def make_cameras(n: int, seed: int = 1) -> torch.Tensor:
    """pitch ~ U[-0.2,0.4], yaw ~ U[-0.6,0.6] (SURVEY.md §8d: all 64^2 rays hit the box for this range)."""
    g = torch.Generator().manual_seed(seed)
    pitch = torch.rand(n, generator=g) * 0.6 - 0.2
    yaw = torch.rand(n, generator=g) * 1.2 - 0.6
    return lookat_camera(pitch, yaw)


def split_camera(camera: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    return camera[:, :16].reshape(-1, 4, 4), camera[:, 16:25].reshape(-1, 3, 3)


def make_planes(n: int, c: int = 32, h: int = 256, w: int = 256, seed: int = 0) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, 3, c, h, w, generator=g)


def make_jitter(n: int, m: int, s: int, s_imp: int = 0, seed: int = 2):
    g = torch.Generator().manual_seed(seed)
    u_c = torch.rand(n, m, s, 1, generator=g)
    u_f = torch.rand(n * m, s_imp, generator=torch.Generator().manual_seed(seed + 1)) if s_imp > 0 else None
    return u_c, u_f


def make_decoder_params(seed: int = 4, n_features: int = 32, hidden: int = 64, out_dim: int = 32) -> Dict[str, torch.Tensor]:
    """OSGDecoder state_dict (modules/img2plane/triplane.py:123-131): N(0,1) weights, small random biases."""
    g = torch.Generator().manual_seed(seed)
    return {
        'net.0.weight': torch.randn(hidden, n_features, generator=g),
        'net.0.bias': 0.1 * torch.randn(hidden, generator=g),
        'net.2.weight': torch.randn(1 + out_dim, hidden, generator=g),
        'net.2.bias': 0.1 * torch.randn(1 + out_dim, generator=g),
    }


def make_sr_params(seed: int = 5, channels: int = 32, w_dim: int = 512) -> Dict[str, torch.Tensor]:
    """SuperresolutionHybrid8XDC state_dict incl. buffers (networks_stylegan2.py:286-321,352-363,377-427)."""
    g = torch.Generator().manual_seed(seed)
    f = torch.tensor([1.0, 3.0, 3.0, 1.0])
    f = torch.outer(f, f)
    f = f / f.sum()
    p: Dict[str, torch.Tensor] = {}
    for blk, res in (('block0', 256), ('block1', 512)):
        cin, cout = SR_CHANNELS[blk]
        if blk == 'block0':
            cin = channels
        p[f'{blk}.resample_filter'] = f.clone()
        for name, ci in (('conv0', cin), ('conv1', cout)):
            pre = f'{blk}.{name}.'
            p[pre + 'weight'] = torch.randn(cout, ci, 3, 3, generator=g)
            p[pre + 'bias'] = 0.1 * torch.randn(cout, generator=g)
            p[pre + 'affine.weight'] = torch.randn(ci, w_dim, generator=g)
            p[pre + 'affine.bias'] = 1.0 + 0.1 * torch.randn(ci, generator=g)
            p[pre + 'noise_strength'] = torch.zeros([])
            p[pre + 'noise_const'] = torch.randn(res, res, generator=g)
            p[pre + 'resample_filter'] = f.clone()
        pre = f'{blk}.torgb.'
        p[pre + 'weight'] = torch.randn(3, cout, 1, 1, generator=g)
        p[pre + 'bias'] = 0.1 * torch.randn(3, generator=g)
        p[pre + 'affine.weight'] = torch.randn(cout, w_dim, generator=g)
        p[pre + 'affine.bias'] = 1.0 + 0.1 * torch.randn(cout, generator=g)
    return p


def make_sr_large_params(seed: int = 8, n_res: int = 2) -> Dict[str, torch.Tensor]:
    """state_dict of SuperresolutionHybrid8XDC(large_sr=True) (superresolution.py:263-345): the two SynthesisBlocks move under `.block`,
    plus `resblocks.{i}.conv{1,2}` and `to_rgb` per LargeSynthesisBlock."""
    base = make_sr_params(seed=seed)
    p = {k.replace('block0.', 'block0.block.', 1).replace('block1.', 'block1.block.', 1): v for k, v in base.items()}
    g = torch.Generator().manual_seed(seed + 200)
    for blk, ch in (('block0', 256), ('block1', 128)):
        for i in range(n_res):
            for c in ('conv1', 'conv2'):
                p[f'{blk}.resblocks.{i}.{c}.weight'] = torch.randn(ch, ch, 3, 3, generator=g) / math.sqrt(ch * 9) * 1.2
                p[f'{blk}.resblocks.{i}.{c}.bias'] = 0.1 * torch.randn(ch, generator=g)
        p[f'{blk}.to_rgb.weight'] = torch.randn(3, ch, 1, 1, generator=g) / math.sqrt(ch)
        p[f'{blk}.to_rgb.bias'] = 0.1 * torch.randn(3, generator=g)
    return p


RENDERING_OPTIONS = {
    'ray_start': 'auto', 'ray_end': 'auto', 'box_warp': 1.0, 'depth_resolution': 48,
    'depth_resolution_importance': 0, 'disparity_space_sampling': False, 'clamp_mode': 'softplus',
    'white_back': False,
}


# ---- torso head (config 5) ------------------------------------------------------------------------------------------------------
class StubTorsoModel(torch.nn.Module):
    """Parameter-free stand-in for the reference's WarpBasedTorsoModelMediaPipe (modules/real3d/facev2v_warp/model2.py:199-336) with the
    same forward signature and the two outputs the SR head consumes.  The real torso warper is an opaque PyTorch child of
    SuperresolutionHybrid8XDC_Warp (out of scope, SURVEY.md §2 #11); parity of the head is tested with THIS module plugged into
    both the reference and our implementation."""

    def forward(self, torso_src_img, segmap, kp_s, kp_d, tgt_head_img, tgt_head_weights, cal_loss=False, target_torso_mask=None):
        rgb_torso = (0.6 * torso_src_img + 0.4 * tgt_head_img.flip(-1)).clamp(-1, 1)
        hid = 0.5 * torch.cat([torso_src_img.repeat(1, 21, 1, 1), tgt_head_weights], dim=1)            # [N,64,256,256]
        seg = torch.nn.functional.avg_pool2d(segmap[:, 2:3].float(), 2)                                # [N,1,256,256]
        occ = torch.sigmoid(6.0 * seg - 3.0 + 0.1 * (kp_d[:, :1, :1] - kp_s[:, :1, :1]).unsqueeze(-1))
        return rgb_torso, {'deformed_torso_hid': hid, 'occlusion_2': occ}


class StubTorsoModelV1(StubTorsoModel):
    """The same stand-in with the forward signature of torso_model_version 'v1' (modules/real3d/facev2v_warp/model.py:216), which takes no head
    weights image; the weights channel of its hidden features is zero.  `calls` counts the forward calls.  Called with the v2 argument list it
    raises TypeError (cal_loss given twice)."""

    def __init__(self):
        super().__init__()
        self.calls = 0

    def forward(self, torso_src_img, segmap, kp_s, kp_d, tgt_head_img, cal_loss=False, target_torso_mask=None):
        self.calls += 1
        return super().forward(torso_src_img, segmap, kp_s, kp_d, tgt_head_img, torch.zeros_like(tgt_head_img[:, :1]), cal_loss, target_torso_mask)


def make_sr_warp_params(seed: int = 6, fuse_mode: str = 'v2', weight_fuse: bool = True) -> Dict[str, torch.Tensor]:
    """state_dict of SuperresolutionHybrid8XDC_Warp WITHOUT its torso_model child (sr_with_ref.py:16-66).  The same random values for every fuse mode;
    mode 'v1' has no head_torso_alpha_predictor / fuse_head_torso_convs / head_torso_block children (sr_with_ref.py:36-55), so their keys are dropped.
    weight_fuse=False has none of them either, whatever the mode, and fuse_fg_bg_convs.0 takes 768 inputs: that weight and bias are drawn from a
    generator of their own (seed + 300), so every other key keeps its weight_fuse=True value."""
    p = make_sr_params(seed=seed)
    g = torch.Generator().manual_seed(seed + 100)
    f = p['block0.resample_filter']

    def conv(name, o, i, k):
        p[name + '.weight'] = torch.randn(o, i, k, k, generator=g) / math.sqrt(i * k * k)
        p[name + '.bias'] = 0.1 * torch.randn(o, generator=g)

    conv('torso_encoder.0', 256, 64, 1)
    conv('bg_encoder.0', 64, 3, 3); conv('bg_encoder.2', 256, 64, 3); conv('bg_encoder.4', 256, 256, 3)
    conv('head_torso_alpha_predictor.0', 32, 7, 3); conv('head_torso_alpha_predictor.2', 32, 32, 3); conv('head_torso_alpha_predictor.4', 1, 32, 3)
    conv('fuse_head_torso_convs.0', 256, 512, 3); conv('fuse_head_torso_convs.2', 256, 256, 3)
    conv('fuse_fg_bg_convs.0', 64, 512, 1); conv('fuse_fg_bg_convs.2', 256, 64, 3); conv('fuse_fg_bg_convs.4', 256, 256, 3)
    blk = 'head_torso_block'
    p[f'{blk}.resample_filter'] = f.clone()
    for name in ('conv0', 'conv1'):
        pre = f'{blk}.{name}.'
        p[pre + 'weight'] = torch.randn(256, 256, 3, 3, generator=g)
        p[pre + 'bias'] = 0.1 * torch.randn(256, generator=g)
        p[pre + 'affine.weight'] = torch.randn(256, 512, generator=g)
        p[pre + 'affine.bias'] = 1.0 + 0.1 * torch.randn(256, generator=g)
        p[pre + 'noise_strength'] = torch.zeros([])
        p[pre + 'noise_const'] = torch.randn(256, 256, generator=g)
        p[pre + 'resample_filter'] = f.clone()
    pre = f'{blk}.torgb.'
    p[pre + 'weight'] = torch.randn(3, 256, 1, 1, generator=g)
    p[pre + 'bias'] = 0.1 * torch.randn(3, generator=g)
    p[pre + 'affine.weight'] = torch.randn(256, 512, generator=g)
    p[pre + 'affine.bias'] = 1.0 + 0.1 * torch.randn(256, generator=g)
    if fuse_mode == 'v1' or not weight_fuse:
        p = {k: v for k, v in p.items() if not k.startswith(('head_torso_alpha_predictor.', 'fuse_head_torso_convs.', 'head_torso_block.'))}
    if not weight_fuse:
        g = torch.Generator().manual_seed(seed + 300)          # conv() draws from g
        conv('fuse_fg_bg_convs.0', 64, 768, 1)
    return p


def make_warp_inputs(n: int, seed: int = 7) -> Dict[str, torch.Tensor]:
    """ref_torso / ref_bg / segmap / key points of SURVEY.md §8d (config 5)."""
    g = torch.Generator().manual_seed(seed)
    return {
        'ref_torso_rgb': torch.randn(n, 3, 512, 512, generator=g).clamp(-1, 1),
        'ref_bg_rgb': torch.randn(n, 3, 512, 512, generator=g).clamp(-1, 1),
        'segmap': torch.rand(n, 6, 512, 512, generator=g),
        'kp_s': torch.rand(n, 68, 3, generator=g) * 2 - 1,
        'kp_d': torch.rand(n, 68, 3, generator=g) * 2 - 1,
    }


WARP_HPARAMS = {'torso_model_version': 'v2', 'htbsr_head_weight_fuse_mode': 'v2', 'htbsr_head_threshold': 0.9, 'torso_kp_num': 4,
                'torso_inp_mode': 'rgb_alpha', 'weight_fuse': True}
