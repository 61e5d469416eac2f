"""CPU restatement of the reference's 'concat_debug' video frames (real3d_infer.py:494-521), with the reference's dtypes and promotion,
and the synthetic inputs the debug-frame tests and tests/golden/make_golden_debug.py share.

The reference concatenates four float32 panels with the SECC panel, which comes back from numpy as float64 (:510-511), so torch.cat promotes
and the clamp (:517) and the ((x + 1) / 2 * 255).int() conversion (:521) of every panel run in float64.  `float32_only=True` and
`copy_bytes=True` are two plausible but wrong readings; the CPU tests show that the fixture tells them apart from the reference."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

S, RES = 512, 64


def to_u8(x: torch.Tensor) -> torch.Tensor:
    """((x + 1) / 2 * 255).int() -> numpy astype(uint8) (:521): int32 wraps modulo 256, so NaN (INT_MIN) gives 0."""
    return torch.from_numpy(((x + 1) / 2 * 255).int().numpy().astype(np.uint8))


def concat_debug_reference(ref_gt_img, drv_secc, image_raw, image_depth, image, float32_only: bool = False, copy_bytes: bool = False,
                           ref_bytes=None) -> torch.Tensor:
    """ref_gt_img [1,3,512,512], drv_secc [N,3,H,W], image_raw [N,3,64,64], image_depth [N,1,64,64], image [N,3,512,512] (CPU, float32)
    -> uint8 [N,512,2560,3].  float32_only: convert every panel in float32 (as out_mode='final' does the final frame); copy_bytes: panel 0 =
    the source bytes ref_bytes [512,512,3] and panel 1 = q, the naive reading of :502."""
    N = image.shape[0]
    secc_img = torch.cat([F.interpolate(drv_secc[i:i + 1], (S, S)) for i in range(N)])
    q = ((secc_img + 1) * 127.5).permute(0, 2, 3, 1).int()                                   # float32, truncated toward zero (:502)
    depth_img = F.interpolate(image_depth, (S, S)).repeat([1, 3, 1, 1])
    depth_img = (depth_img - depth_img.min()) / (depth_img.max() - depth_img.min())           # float32 (:506)
    depth_img = (depth_img * 2 - 1).clamp(-1, 1)
    if float32_only:
        secc = (q.float() / 127.5 - 1).permute(0, 3, 1, 2)
    else:
        secc = torch.from_numpy(q.numpy() / 127.5 - 1).permute(0, 3, 1, 2)                     # numpy: int32 / float -> float64 (:510-511)
    imgs = torch.cat([ref_gt_img.repeat([N, 1, 1, 1]), secc, F.interpolate(image_raw, (S, S)), depth_img, image], dim=-1)
    out = to_u8(imgs.clamp(-1, 1).permute(0, 2, 3, 1))
    if copy_bytes:
        out[:, :, :S] = torch.as_tensor(ref_bytes)
        out[:, :, S:2 * S] = q.to(torch.uint8)
    return out


# ---- synthetic inputs -----------------------------------------------------------------------------------------------------------------
def up8(x: torch.Tensor) -> torch.Tensor:
    """[..., 64, 64] -> [..., 512, 512] by nearest replication (the fixture stores the 64^2 fields)."""
    return x.repeat_interleave(8, -2).repeat_interleave(8, -1)


def ref_gt_from_bytes(b) -> torch.Tensor:
    """load_img_to_normalized_512_bchw_tensor (infer_utils.py:21): (b - 127.5) / 127.5 in float32, [1,3,H,W]."""
    return ((torch.as_tensor(b) - 127.5) / 127.5).float().unsqueeze(0).permute(0, 3, 1, 2).contiguous()


def _f32(x) -> np.ndarray:
    return np.asarray(x, np.float64).astype(np.float32)


def byte_boundaries() -> np.ndarray:
    """The float32 values nearest to the 255 byte boundaries x = 2k / 255 - 1 of ((x + 1) / 2 * 255).int(), and their two neighbours."""
    b = _f32(2 * np.arange(1, 256) / 255 - 1)
    return np.concatenate([np.nextafter(b, np.float32(-2)), b, np.nextafter(b, np.float32(2))]).astype(np.float32)


def secc_boundaries() -> np.ndarray:
    """SECC values at the q = ((s + 1) * 127.5).int() boundaries s = k / 127.5 - 1 and their float32 neighbours, and values below -1."""
    b = _f32(np.arange(0, 256) / 127.5 - 1)
    below = _f32([-1.0000001, -1.001, -1.25, -1.5, -2.0, -3.7, -1.0078125, -1.0078126])
    return np.concatenate([np.nextafter(b, np.float32(-2)), b, np.nextafter(b, np.float32(2)), below, _f32([1.0, 1.0001, 1.5])])


def quirk_inputs(N: int, seed: int, constant_depth: bool = False):
    """64^2 fields (fp32) that exercise the quirks: every source byte, the SECC q boundaries, the float32 neighbours of the byte boundaries
    in image and image_raw (image_raw also outside [-1, 1]), and depths whose min and max sit in different frames.
    -> dict of numpy arrays: ref_bytes [64,64,3] uint8, secc [N,3,64,64], image_raw [N,3,64,64], image_depth [N,1,64,64], image [N,3,64,64]."""
    g = np.random.default_rng(seed)
    n = RES * RES * 3
    ref_bytes = np.concatenate([np.arange(256), g.integers(0, 256, n - 256)]).astype(np.uint8)
    g.shuffle(ref_bytes)

    def field(special, lo, hi):
        out = np.empty((N, 3 * RES * RES), np.float32)
        for i in range(N):
            v = g.uniform(lo, hi, 3 * RES * RES).astype(np.float32)
            v[:len(special)] = special
            g.shuffle(v)
            out[i] = v
        return out.reshape(N, 3, RES, RES)

    edges = byte_boundaries()
    raw_special = np.concatenate([edges, _f32([-1.0, 1.0, 1.5, -1.25, 3.0, -7.0])])
    if constant_depth:                                                 # the tiny case: every field constant, panel 3 is 0 / 0
        c = lambda v, C: np.full((N, C, RES, RES), v, np.float32)     # noqa: E731
        return {'ref_bytes': np.full((RES, RES, 3), 77, np.uint8), 'secc': c(0.1, 3), 'image_raw': c(0.3, 3), 'image_depth': c(2.5, 1),
                'image': c(-0.2, 3)}
    depth = g.uniform(2.2, 2.8, (N, 1, RES, RES)).astype(np.float32)
    depth[0, 0, 5, 7] = np.float32(2.0)                                # the clip's min in frame 0 ...
    depth[N - 1, 0, 60, 3] = np.float32(3.0)                           # ... and its max in the last frame
    return {'ref_bytes': ref_bytes.reshape(RES, RES, 3), 'secc': field(secc_boundaries(), -1.0, 1.0),
            'image_raw': field(raw_special, -1.1, 1.1), 'image_depth': depth, 'image': field(_f32(np.append(edges, [-1.0, 1.0])), -1.0, 1.0)}


def full_inputs(fields: dict):
    """The stored 64^2 fields -> the reference's tensors: ref_gt_img [1,3,512,512], drv_secc [N,3,512,512], image_raw [N,3,64,64],
    image_depth [N,1,64,64], image [N,3,512,512]; also the source bytes [512,512,3]."""
    rb = np.repeat(np.repeat(np.asarray(fields['ref_bytes']), 8, 0), 8, 1)
    return {'ref_gt_img': ref_gt_from_bytes(rb), 'drv_secc': up8(torch.as_tensor(fields['secc'])),
            'image_raw': torch.as_tensor(fields['image_raw']).clone(), 'image_depth': torch.as_tensor(fields['image_depth']).clone(),
            'image': up8(torch.as_tensor(fields['image'])), 'ref_bytes': rb}
