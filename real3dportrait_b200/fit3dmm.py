"""3DMM landmark fit on libr3dp_b200: the source image's and a driving video's coefficients (id, exp, euler, trans) from mediapipe's
landmarks, as fit_3dmm_for_a_image (data_gen/utils/process_image/fit_3dmm_landmark.py:85-236) and fit_3dmm_for_a_video with
id_mode='global' (data_gen/utils/process_video/fit_3dmm_landmark.py:131-360) compute them.  Both run the reference's two Adam stages
(200 steps on the pose, then 200 on everything) as 800 launches on the caller's stream (DESIGN.md, "3DMM fit"):

  r3dp_fit_grad  the landmark loss's gradient: key shapes, projection, residual and the chain rule back to the coefficients
  r3dp_fit_adam  the chunk partials summed, the regulariser and Laplacian terms, Adam's step

The reference's fine stage (50-iteration batches at lr 0.005) writes its results into temporary copies, so its returned coefficients are
the second stage's; it is not run here."""
from __future__ import annotations

import os
from typing import Dict, Optional

import numpy as np
import torch
import torch.nn as nn

from . import _capi as capi
from .motion import load_bfm

N_KP, N_ID, N_EXP = 468, 80, 64
CHUNK, CHUNKS = 64, 8                     # key points per chunk; 8 chunks hold the 468 (the last 44 rows padded, weight 0)
ROW = N_EXP + 6                           # per-frame parameters: exp, euler, trans
MAX_CTAS = 16                             # frame-tile CTAs per chunk of r3dp_fit_grad (its part_id rows)
ITERS = 200                               # Adam steps per stage
_UNMATCHED = [93, 127, 132, 234, 323, 356, 361, 454]
_UPPER_EYE = [161, 160, 159, 158, 157, 388, 387, 386, 385, 384]
_EYE = [33, 246, 161, 160, 159, 158, 157, 173, 133, 155, 154, 153, 145, 144, 163, 7,
        263, 466, 388, 387, 386, 385, 384, 398, 362, 382, 381, 380, 374, 373, 390, 249]
_INNER_LIP = [78, 191, 80, 81, 82, 13, 312, 311, 310, 415, 308, 324, 318, 402, 317, 14, 87, 178, 88, 95]
_OUTER_LIP = [61, 185, 40, 39, 37, 0, 267, 269, 270, 409, 291, 375, 321, 405, 314, 17, 84, 181, 91, 146]
#: (lambda_id, lambda_exp, lambda_lap): the image file's module constants and the video file's id_mode='global' ones
_LAMBDAS = {False: (0.3, 0.05, 0.0), True: (0.2, 0.6, 1.0)}
_NAMES = ('id', 'exp', 'euler', 'trans')


def _weights(video: bool) -> np.ndarray:
    """cal_lan_loss_mp's per-point weights: image eye 5, lips 2; video eye 3, upper eye 20, lips 5; the 8 unmatched points 0."""
    w = np.ones(CHUNK * CHUNKS, np.float32)
    w[N_KP:] = 0
    w[_EYE] = 3 if video else 5
    if video:
        w[_UPPER_EYE] = 20
    w[_INNER_LIP] = 5 if video else 2
    w[_OUTER_LIP] = 5 if video else 2
    w[_UNMATCHED] = 0
    return w


def load_mp468_index(bfm_folder: str, n_vertices: int) -> np.ndarray:
    """index_mp468_from_mesh35709.npy -> int64 [468] as ParametricFaceModel(keypoint_mode='mediapipe') uses it: 0-based, negative entries
    (the points without a vertex) replaced by vertex 0 (bfm.py:60-63)."""
    path = os.path.join(bfm_folder, 'index_mp468_from_mesh35709.npy')
    if not os.path.isfile(path):
        raise FileNotFoundError(f'Fit3DMM: index_mp468_from_mesh35709.npy not found at {path!r}')
    idx = np.load(path).astype(np.int64).reshape(-1)
    if idx.size != N_KP:
        raise ValueError(f'Fit3DMM: index_mp468_from_mesh35709.npy holds {idx.size} entries, not {N_KP}')
    idx[idx < 0] = 0
    if idx.max() >= n_vertices:
        raise ValueError(f'Fit3DMM: index_mp468_from_mesh35709.npy indexes vertex {idx.max()}, the BFM has {n_vertices}')
    return idx


class Fit3DMM(nn.Module):
    """The reference's mediapipe 3DMM fit on the GPU (CUDA tensors, fp32).

    Fit3DMM(bfm_folder) reads BFM_model_front.mat (meanshape, idBase, exBase) and index_mp468_from_mesh35709.npy, and keeps the 468 key
    points' mean and [id | exp] basis on the device.  fit_image(lms) and fit_video(lms) return {'id' [1,80], 'exp' [T,64], 'euler' [T,3],
    'trans' [T,3]}.  A call does no host sync and allocates its workspace before its launches, so it can be captured in a CUDA graph."""

    def __init__(self, bfm_folder: str = 'deep_3drecon/BFM', device='cuda'):
        super().__init__()
        m = load_bfm(bfm_folder, 'Fit3DMM')
        if m['id_base'].shape[1] != N_ID or m['exp_base'].shape[1] != N_EXP:
            raise ValueError(f'Fit3DMM: the fit takes {N_ID} id and {N_EXP} exp coefficients, the BFM has '
                             f'{m["id_base"].shape[1]} and {m["exp_base"].shape[1]}')
        n = m['mean'].shape[0]
        idx = load_mp468_index(bfm_folder, n)
        basis = np.concatenate([m['id_base'].reshape(n, 3, N_ID)[idx], m['exp_base'].reshape(n, 3, N_EXP)[idx]], -1)   # [468,3,144]
        pad = CHUNK * CHUNKS - N_KP
        basis = np.concatenate([basis, np.zeros((pad, 3, N_ID + N_EXP), np.float32)])
        mean = np.concatenate([m['mean'][idx], np.zeros((pad, 3), np.float32)])
        # per chunk: rows [x of its 64 points | y | z]
        basis = basis.reshape(CHUNKS, CHUNK, 3, -1).transpose(0, 2, 1, 3).reshape(CHUNKS, 3 * CHUNK, -1)
        mean = mean.reshape(CHUNKS, CHUNK, 3).transpose(0, 2, 1).reshape(CHUNKS, 3 * CHUNK)
        self.register_buffer('basis', torch.from_numpy(np.ascontiguousarray(basis)), persistent=False)
        self.register_buffer('mean_shape', torch.from_numpy(np.ascontiguousarray(mean)), persistent=False)
        self.register_buffer('w_image', torch.from_numpy(_weights(False)), persistent=False)
        self.register_buffer('w_video', torch.from_numpy(_weights(True)), persistent=False)
        self.register_buffer('index', torch.from_numpy(idx), persistent=False)
        self.to(device)

    @torch.no_grad()
    def fit_image(self, lms: torch.Tensor, img_size: int = 512, out: Optional[Dict[str, torch.Tensor]] = None) -> Dict[str, torch.Tensor]:
        """fit_3dmm_for_a_image: lms [468|478, 2] or [1, 468|478, 2], mediapipe's pixels (y down) in an img_size^2 image -> {'id' [1,80],
        'exp' [1,64], 'euler' [1,3], 'trans' [1,3]}.  out: a dict of those four fp32 CUDA tensors, written in place (any strides)."""
        if isinstance(lms, torch.Tensor) and lms.ndim == 2:
            lms = lms.unsqueeze(0)
        if not isinstance(lms, torch.Tensor) or lms.ndim != 3 or lms.shape[0] != 1:
            raise ValueError(f'Fit3DMM.fit_image: lms must be a tensor [468|478, 2] or [1, 468|478, 2], got {tuple(getattr(lms, "shape", ()))}')
        return self._fit(lms, img_size, False, out, 'fit_image')

    @torch.no_grad()
    def fit_video(self, lms: torch.Tensor, img_size: int = 512, out: Optional[Dict[str, torch.Tensor]] = None) -> Dict[str, torch.Tensor]:
        """fit_3dmm_for_a_video (id_mode='global'): lms [T, 468|478, 2], T >= 1, mediapipe's pixels (y down) in img_size^2 frames ->
        {'id' [1,80], 'exp' [T,64], 'euler' [T,3], 'trans' [T,3]}.  out: a dict of those four fp32 CUDA tensors, written in place; exp may
        be strided, e.g. the column slice rows[:, 80:144] of the engine's [id | exp | ...] rows."""
        return self._fit(lms, img_size, True, out, 'fit_video')

    def _fit(self, lms, img_size, video, out, what):
        if not isinstance(lms, torch.Tensor) or lms.ndim != 3 or lms.shape[0] < 1 or lms.shape[1] not in (N_KP, 478) or lms.shape[2] != 2:
            raise ValueError(f'Fit3DMM.{what}: lms must be a tensor [T, 468|478, 2] with T >= 1, got {tuple(getattr(lms, "shape", ()))}')
        if isinstance(img_size, bool) or not isinstance(img_size, (int, np.integer)) or img_size < 1:
            raise ValueError(f'Fit3DMM.{what}: img_size must be a positive int, got {img_size!r}')
        T, L = lms.shape[0], lms.shape[1]
        shapes = {'id': (1, N_ID), 'exp': (T, N_EXP), 'euler': (T, 3), 'trans': (T, 3)}
        if out is not None:
            if not isinstance(out, dict) or set(out) != set(_NAMES):
                raise ValueError(f'Fit3DMM.{what}: out must be a dict with the keys {list(_NAMES)}')
            for k in _NAMES:
                t = out[k]
                if not isinstance(t, torch.Tensor) or tuple(t.shape) != shapes[k] or t.dtype != torch.float32:
                    raise ValueError(f'Fit3DMM.{what}: out[{k!r}] must be an fp32 tensor {list(shapes[k])}')
        dev = self.basis.device
        for name, t in [('lms', lms)] + ([] if out is None else [(f'out[{k!r}]', out[k]) for k in _NAMES]):
            if not t.is_cuda:
                raise RuntimeError(f'real3dportrait_b200 runs on CUDA tensors only (no CPU fallback); {name} is not a CUDA tensor')
            if t.device != dev:
                raise ValueError(f'Fit3DMM.{what}: {name} is on {t.device}, the BFM on {dev}')
        lms = capi.f32(lms)
        n = N_ID + ROW * T
        # fp64: the parameters and Adam's moments (ping-pong x pair, m, v) and the per-frame and id partials; fp32: the exp partials
        sizes = (n, n, n, n, CHUNKS * T * 12, CHUNKS * MAX_CTAS * N_ID)
        ws = torch.empty(sum(sizes), device=dev, dtype=torch.float64)
        xa, xb, m, v, part_frame, part_id = ws.split(sizes)
        part_exp = torch.empty(CHUNKS * T * N_EXP, device=dev)
        ws[:4 * n].zero_()                                         # parameters and Adam's moments start at zero
        lam_id, lam_exp, lam_lap = _LAMBDAS[video]
        weight = self.w_video if video else self.w_image
        L_, p, st = capi.lib(), capi.ptr, capi.stream()
        basis, mean, w, lp, pe = (p(t) for t in (self.basis, self.mean_shape, weight, lms, part_exp))
        pf, pi, pm, pv = (p(t, torch.float64) for t in (part_frame, part_id, m, v))
        d = lambda t: p(t, torch.float64)                          # noqa: E731
        with capi.region('fit3dmm'):
            for stage in (1, 2):
                for s in range(1, ITERS + 1):
                    capi.check(L_.r3dp_fit_grad(basis, mean, w, lp, T, L, int(img_size), d(xa), stage, pf, pe, pi, st))
                    step_frame, step_idexp = (s, 0) if stage == 1 else (ITERS + s, s)
                    capi.check(L_.r3dp_fit_adam(pf, pe, pi, T, step_frame, step_idexp, 0.1, lam_id, lam_exp, lam_lap, d(xa), d(xb), pm, pv,
                                                None, st))
                    xa, xb = xb, xa
        rows = xa[N_ID:].view(T, ROW)
        res = {'id': xa[:N_ID].view(1, N_ID), 'exp': rows[:, :N_EXP], 'euler': rows[:, N_EXP:N_EXP + 3], 'trans': rows[:, N_EXP + 3:]}
        if out is None:
            return {k: r.float().contiguous() for k, r in res.items()}
        for k in _NAMES:
            out[k].copy_(res[k])
        return out
