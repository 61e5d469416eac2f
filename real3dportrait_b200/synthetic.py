"""Deterministic synthetic inputs for the render + SR path (SURVEY.md §8d): tri-planes, look-at cameras, jitter
uniforms and random-init decoder / SR parameters.  Everything is drawn on the CPU from seeded generators so the
CPU oracle, the golden fixtures and the GPU path see identical bits; callers upload with `.cuda()`.

Camera convention follows the reference's pose sampler (modules/eg3ds/camera_utils/pose_sampler.py:28-36,
94-131,174-204): camera on a sphere of radius 2.7 around `lookat`, y up, 25-vector = row-major c2w (16) +
row-major normalised intrinsics (9) with focal 4.2647 and principal point 0.5."""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

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


# ---- SECC renderer: a synthetic BFM (the real BFM_model_front.mat is licensed and not shipped) ----------------------------------
BFM_ID, BFM_EXP = 80, 64


def make_bfm(seed: int = 0, rows: int = 150, cols: int = 238) -> Dict[str, 'np.ndarray']:
    """A head-like mesh at BFM scale with the BFM's file contents (float64 numpy; the loader casts like the reference):
    meanshape [1, 3N] (xyz interleaved, not centred: the loader recentres it), idBase [3N, 80], exBase [3N, 64], tri [F, 3] 1-based,
    ncc [3, N] in [0, 1], right_eye / left_eye: disjoint 1-based face lists.  Default size 150 x 238 = 35 700 vertices, 70 626 faces.

    The surface is a grid on an ellipsoidal shell (semi-axes 0.75 / 0.9 / 0.7, facing +z, i.e. the camera after to_camera) over 0.15-0.85 pi
    of polar angle and +-0.8 pi of azimuth, so part of the back is meshed too, with a nose bump that occludes the cheek under yaw.  The id and exp
    bases are smooth low-frequency fields: N(0,1) coefficients move a vertex by a few hundredths.  Face 0 sits on the forehead, where every
    image with |yaw| <= 0.6 sees it."""
    import numpy as np
    rng = np.random.default_rng(seed)
    th = np.linspace(0.15 * np.pi, 0.85 * np.pi, rows)[:, None]
    ph = np.linspace(-0.8 * np.pi, 0.8 * np.pi, cols)[None, :]
    nose = 0.22 * np.exp(-((th - 0.56 * np.pi) ** 2 / 0.02 + ph ** 2 / 0.012))
    rad = 1.0 + nose
    P = np.stack([0.75 * rad * np.sin(th) * np.sin(ph), 0.9 * np.cos(th) * np.ones_like(ph), 0.7 * rad * np.sin(th) * np.cos(ph)], -1)
    P = P.reshape(-1, 3) + np.array([0.02, 0.05, -0.03])             # off-centre: recentring at load moves it back
    n = P.shape[0]
    u, w = (th[:, 0] - th.min()) / np.ptp(th), (ph[0] - ph.min()) / np.ptp(ph)

    def basis(k, amp):                                                 # separable fields a cos(pi f u + p) cos(pi g w + q) per column and axis
        f = rng.integers(1, 4, size=(k, 3, 2))
        p = rng.uniform(0, 2 * np.pi, size=(k, 3, 2))
        a = rng.normal(size=(k, 3, 1)) * amp
        fu = a * np.cos(np.pi * f[..., :1] * u + p[..., :1])           # [k, 3, rows]
        fw = np.cos(np.pi * f[..., 1:] * w + p[..., 1:])               # [k, 3, cols]
        return np.einsum('kar,kac->rcak', fu, fw).reshape(3 * n, k)   # rows 3v + axis, v = row * cols + col
    id_base, ex_base = basis(BFM_ID, 0.006), basis(BFM_EXP, 0.004)
    idx = np.arange(n).reshape(rows, cols)
    q0, q1, q2, q3 = idx[:-1, :-1].reshape(-1), idx[:-1, 1:].reshape(-1), idx[1:, :-1].reshape(-1), idx[1:, 1:].reshape(-1)
    tri = np.concatenate([np.stack([q0, q2, q1], 1), np.stack([q1, q2, q3], 1)], 0)
    cen = P[tri].mean(1)
    front = np.argmin(np.abs(cen[:, 0]) + np.abs(cen[:, 1] - 0.45) + np.abs(cen[:, 2] - cen[:, 2].max()) * 0.1)
    tri[[0, front]] = tri[[front, 0]]                                  # face 0: the forehead
    cen = P[tri].mean(1)
    eyes = []
    for sx in (-1, 1):                                                 # right eye (image left), then left eye
        d = (cen[:, 0] - sx * 0.28) ** 2 + (cen[:, 1] - 0.18) ** 2
        sel = np.nonzero((d < 0.06 ** 2) & (cen[:, 2] > 0))[0]
        eyes.append(sel[sel != 0] + 1)
    ncc = ((P - P.min(0)) / np.ptp(P, 0)).T
    return {'meanshape': P.reshape(1, -1), 'idBase': id_base, 'exBase': ex_base, 'tri': (tri + 1).astype(np.float64), 'ncc': ncc,
            'right_eye': eyes[0].astype(np.int64), 'left_eye': eyes[1].astype(np.int64)}


def make_keypoints(bfm: dict, seed: int = 0, rows: int = 150, cols: int = 238) -> 'np.ndarray':
    """68 landmark vertices of make_bfm's head as BFM_model_front.mat stores them: [68, 1] float64, 1-based.  The layout follows the 68-point
    scheme (jaw 17, brows 10, nose 9, eyes 12, mouth 20) on the front of the head; the jaw reaches x = +-0.7 and the chin y = -0.75, so
    translations of a few tenths push key points past +-1 in NDC.  Each target is jittered by a generator of its own (seed + 1000), not
    make_bfm's: the bases and every output drawn from them stay as they are."""
    import numpy as np
    rng = np.random.default_rng(seed + 1000)
    P = np.asarray(bfm['meanshape'], np.float64).reshape(-1, 3)
    jaw = [(0.7 * np.sin(a), 0.15 - 0.9 * np.cos(a)) for a in np.linspace(-1.45, 1.45, 17)]
    brows = [(sx * x, 0.3 + 0.04 * np.sin(np.pi * (x - 0.12) / 0.3)) for sx in (-1, 1) for x in np.linspace(0.12, 0.42, 5)]
    nose = [(0.0, y) for y in np.linspace(0.12, -0.12, 4)] + [(x, -0.2) for x in np.linspace(-0.1, 0.1, 5)]
    eyes = [(sx * (0.28 + 0.08 * np.cos(a)), 0.18 + 0.035 * np.sin(a)) for sx in (-1, 1) for a in np.linspace(0, 2 * np.pi, 7)[:-1]]
    outer = [(0.2 * np.cos(a), -0.42 + 0.09 * np.sin(a)) for a in np.linspace(0, 2 * np.pi, 13)[:-1]]
    inner = [(0.12 * np.cos(a), -0.42 + 0.04 * np.sin(a)) for a in np.linspace(0, 2 * np.pi, 9)[:-1]]
    tgt = np.array(jaw + brows + nose + eyes + outer + inner) + rng.normal(scale=0.01, size=(68, 2))
    front = np.nonzero(P[:, 2] > P[:, 2].mean())[0]
    d = ((P[front, None, :2] - tgt[None]) ** 2).sum(-1)
    v = front[np.argmin(d, 0)]
    assert v.max() + 1 < P.shape[0]                                   # the reference reads vertex v + 1 (no - 1): it must exist
    return (v + 1).astype(np.float64).reshape(68, 1)


#: the 8 mediapipe points without a BFM vertex (index -1 in index_mp468_from_mesh35709.npy; weight 0 in the fit's landmark loss)
MP_UNMATCHED = (93, 127, 132, 234, 323, 356, 361, 454)


def make_mp468_index(bfm: dict, seed: int = 0) -> 'np.ndarray':
    """index_mp468_from_mesh35709.npy for make_bfm's head: int64 [468], 0-based vertex indices of 468 distinct vertices spread over the front
    of the face (|x| < 0.6, -0.8 < y < 0.55), -1 at MP_UNMATCHED.  A generator of its own (seed + 2000), so make_bfm's outputs stay as they are."""
    import numpy as np
    rng = np.random.default_rng(seed + 2000)
    P = np.asarray(bfm['meanshape'], np.float64).reshape(-1, 3)
    front = np.nonzero((P[:, 2] > P[:, 2].mean()) & (np.abs(P[:, 0]) < 0.6) & (P[:, 1] > -0.8) & (P[:, 1] < 0.55))[0]
    idx = rng.choice(front, size=468, replace=False).astype(np.int64)
    idx[list(MP_UNMATCHED)] = -1
    return idx


def write_bfm_folder(path: str, bfm: Optional[dict] = None, seed: int = 0, keypoints: bool = False, mp468: bool = False) -> Dict[str, object]:
    """Write a BFM in the reference's file layout under `path` (BFM/BFM_model_front.mat with 1-based tri, ncc_code.npy [3,N],
    bfm_{right,left}_eye_faces.npy 1-based) and return the SECC_Renderer keyword arguments that read it.  keypoints=True also writes the
    68 key points (make_keypoints) and zero placeholders for the other keys Face3DHelper loads (meantex, texBase, point_buf).  mp468=True
    writes BFM/index_mp468_from_mesh35709.npy (make_mp468_index) and placeholders for every key ParametricFaceModel(is_train=True) loads."""
    import numpy as np
    import os
    import scipy.io
    bfm = make_bfm(seed) if bfm is None else bfm
    os.makedirs(os.path.join(path, 'BFM'), exist_ok=True)
    mat = {k: bfm[k] for k in ('meanshape', 'idBase', 'exBase', 'tri')}
    if keypoints:
        n = bfm['meanshape'].size // 3
        mat.update({'keypoints': make_keypoints(bfm, seed), 'meantex': np.zeros((1, 3 * n)), 'texBase': np.zeros((3 * n, 1)),
                    'point_buf': np.zeros((n, 8))})
    if mp468:
        n = bfm['meanshape'].size // 3
        mat.setdefault('keypoints', make_keypoints(bfm, seed))
        for k, v in (('meantex', np.zeros((1, 3 * n))), ('texBase', np.zeros((3 * n, 1))), ('point_buf', np.ones((n, 8))),
                     ('frontmask2_idx', np.ones((n, 1))), ('tri_mask2', bfm['tri'][:16]), ('skinmask', np.ones((1, n)))):
            mat.setdefault(k, v)
        np.save(os.path.join(path, 'BFM', 'index_mp468_from_mesh35709.npy'), make_mp468_index(bfm, seed))
    scipy.io.savemat(os.path.join(path, 'BFM', 'BFM_model_front.mat'), mat)
    np.save(os.path.join(path, 'ncc_code.npy'), bfm['ncc'].astype(np.float32))
    eyes = (os.path.join(path, 'bfm_right_eye_faces.npy'), os.path.join(path, 'bfm_left_eye_faces.npy'))
    np.save(eyes[0], bfm['right_eye'])
    np.save(eyes[1], bfm['left_eye'])
    return {'bfm_folder': os.path.join(path, 'BFM'), 'ncc_path': os.path.join(path, 'ncc_code.npy'), 'eye_faces': eyes}


def make_coeffs(n: int, seed: int = 0, yaw: float = 0.0) -> Dict[str, torch.Tensor]:
    """id [n,80], exp [n,64] ~ N(0,1); euler [n,3] with yaw ~ U[-yaw, yaw] and pitch / roll a fifth of it; trans [n,3] ~ 0.02 N(0,1) when yaw > 0
    (zero otherwise, as real3d_infer.py:392-393 drives the renderer)."""
    g = torch.Generator().manual_seed(seed)
    c = {'id': torch.randn(n, BFM_ID, generator=g), 'exp': torch.randn(n, BFM_EXP, generator=g)}
    e = (torch.rand(n, 3, generator=g) * 2 - 1) * yaw * torch.tensor([0.2, 1.0, 0.2])
    t = 0.02 * torch.randn(n, 3, generator=g) * (1.0 if yaw > 0 else 0.0)
    c.update({'euler': e, 'trans': t})
    return c


# ---- source images: a portrait-like segmap and a smooth image (the segmap itself comes from mediapipe and is not shipped) ---------------
SEG_BG, SEG_HAIR, SEG_BODY, SEG_FACE, SEG_CLOTHES, SEG_OTHERS = range(6)


def make_segmap(H: int = 512, W: int = 512, seed: int = 0, *, center: float = 0.5, torso_top: float = 0.72, torso: bool = True,
                neck_width: float = 0.09, neck_gaps: int = 0, roll: int = 0, fractional: bool = False) -> 'np.ndarray':
    """A [6,H,W] float32 one-hot map in _cal_seg_map's channel order: a head ellipse (face skin, hair on top, an 'others' band for glasses)
    centred on column center * W, a neck (body skin) from inside the head down to the torso, clothes from row torso_top * H to the bottom
    (torso=False: none) widening downward, background elsewhere; every boundary wobbles per column with the seed.  neck_width: the neck's
    half width / W (wider than the head's bottom gives neck columns without head above them).  neck_gaps: that many 10-row background gaps
    cut into random neck columns (a neck that is not contiguous within a column).  roll: np.roll of the rows (a negative roll of the torso's
    top puts the torso on row 0 and the head on the last rows).  fractional: soft values, so that (s1 + s3 + s5) != 0 and > 0.5 disagree on
    part of the image and s0 is fractional but nonzero on the background."""
    import numpy as np
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    wob = lambda amp: amp * np.sin(x[0] / W * rng.uniform(4, 12) + rng.uniform(0, 6.3))[None, :]   # noqa: E731  per-column wobble
    cy, cx, ry, rx = 0.36 * H, center * W, 0.2 * H, 0.16 * W
    cls = np.full((H, W), SEG_BG, np.int64)
    t0 = torso_top * H + wob(0.02 * H)
    if torso:
        cls[(y >= t0) & (np.abs(x - cx) <= 0.22 * W + 0.5 * (y - t0) + wob(0.01 * W))] = SEG_CLOTHES
    neck = (y >= cy) & (y < t0) & (np.abs(x - cx) <= neck_width * W + wob(0.01 * W))
    cls[neck] = SEG_BODY
    head = ((y - cy) / ry) ** 2 + ((x - cx) / rx) ** 2 <= 1 + wob(0.05)
    cls[head] = SEG_FACE
    cls[head & (y < cy - 0.45 * ry + wob(0.04 * H))] = SEG_HAIR
    cls[head & (np.abs(y - (cy - 0.1 * ry)) < 0.04 * H) & (np.abs(x - cx) < 0.7 * rx)] = SEG_OTHERS
    cols = np.nonzero(neck.any(0))[0]
    for _ in range(neck_gaps):
        if cols.size:
            c = rng.choice(cols)
            r = np.nonzero(cls[:, c] == SEG_BODY)[0]
            if r.size > 16:
                r0 = rng.integers(r[0] + 2, r[-1] - 12)
                cls[r0:r0 + 10, c] = SEG_BG
    seg = (np.arange(6)[:, None, None] == cls[None]).astype(np.float32)
    if fractional:
        u = rng.uniform(0.0, 1.0, (H, W)).astype(np.float32)
        soft = rng.uniform(0.0, 1.0, (H, W)) < 0.3
        seg[SEG_HAIR][soft & (cls != SEG_HAIR)] = 0.4 * u[soft & (cls != SEG_HAIR)]       # head sum in (0, 0.4]: != 0 yet not > 0.5
        seg[SEG_FACE][soft & (cls == SEG_FACE)] = 0.2 + 0.6 * u[soft & (cls == SEG_FACE)]
        seg[SEG_BG][soft & (cls == SEG_BG)] = 0.25 + 0.5 * u[soft & (cls == SEG_BG)]
    if roll:
        seg = np.roll(seg, roll, axis=1)
    return np.ascontiguousarray(seg)


def make_source_image(H: int = 512, W: int = 512, seed: int = 0) -> 'np.ndarray':
    """A smooth uint8 [H,W,3] RGB image: a few seeded low-frequency waves per channel."""
    import numpy as np
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    img = np.empty((H, W, 3))
    for ch in range(3):
        v = rng.uniform(60, 190) + np.zeros((H, W))
        for _ in range(3):
            fy, fx, ph = rng.uniform(0.5, 4, 2).tolist() + [rng.uniform(0, 6.3)]
            v += rng.uniform(20, 40) * np.sin(2 * np.pi * (fy * y / H + fx * x / W) + ph)
        img[..., ch] = v
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)
