"""Clip motion on libr3dp_b200: each frame's camera [T,25] and the torso head's key points kp_s [1,68,3] / kp_d [T,68,3] from the source
frame's 3DMM fit, the clip's expression rows and a driving pose, as real3d_infer.py builds them on the host (:271-321, :428-452) with
Face3DHelper, get_eg3d_convention_camera_pose_intrinsic, smooth_camera_sequence and smooth_features_xd.  Four launches, no host sync
after validation (DESIGN.md, "Clip motion"):

  r3dp_motion_camera     the frames' poses and their smoothed cameras
  r3dp_secc_vertices     x2: the source frame and the clip's frames at the 68 key points (the SECC renderer's vertex pass on a gathered basis)
  r3dp_motion_keypoints  clamp, 7-frame smoothing of kp_d, z = 0

The outputs feed FrameEngine(torso_model=...): begin_clip(..., kp_s) once, then step / prepare with cameras[i:i+B] and kp_d[i:i+B]."""
from __future__ import annotations

import ctypes
import os
from typing import Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn as nn

from . import _capi as capi
from .secc_render import CAMERA_DISTANCE, CENTER, FOCAL

def load_bfm(bfm_folder: str, who: str, keys=()):
    """BFM_model_front.mat -> float32 numpy: mean [N,3] recentred (bfm.py:78-81), id_base [3N,n_id], exp_base [3N,n_exp], and the raw
    entries `keys` (which must be present too).  who names the caller in error messages."""
    from scipy.io import loadmat
    path = os.path.join(bfm_folder, 'BFM_model_front.mat')
    if not os.path.isfile(path):
        raise FileNotFoundError(f'{who}: BFM_model_front.mat not found at {path!r}')
    mat = loadmat(path)
    missing = [k for k in ('meanshape', 'idBase', 'exBase') + tuple(keys) if k not in mat]
    if missing:
        raise KeyError(f'{who}: BFM_model_front.mat lacks {missing}')
    mean = mat['meanshape'].astype(np.float32).reshape(-1, 3)
    mean = mean - np.mean(mean, axis=0, keepdims=True)
    id_base, exp_base = mat['idBase'].astype(np.float32), mat['exBase'].astype(np.float32)
    n = mean.shape[0]
    if id_base.shape[0] != 3 * n or exp_base.shape[0] != 3 * n:
        raise ValueError(f'{who}: idBase {id_base.shape} / exBase {exp_base.shape} do not match {n} vertices')
    out = {'mean': mean, 'id_base': id_base, 'exp_base': exp_base}
    out.update({k: mat[k] for k in keys})
    return out


def load_keypoint_bfm(bfm_folder: str):
    """BFM_model_front.mat -> load_bfm's arrays and keypoints int64 [68] as stored (1-based in the file; read without the - 1, see
    ClipMotion)."""
    m = load_bfm(bfm_folder, 'ClipMotion', ('keypoints',))
    n = m['mean'].shape[0]
    kp = np.squeeze(m['keypoints']).astype(np.int64).reshape(-1)
    if kp.size == 0 or kp.min() < 0 or kp.max() >= n:
        raise ValueError(f'ClipMotion: keypoints must index the {n} vertices as stored (the reference gathers them without - 1)')
    m['keypoints'] = kp
    return m


class ClipMotion(nn.Module):
    """A clip's cameras and torso key points on the GPU (CUDA tensors, fp32).

    The key points are Face3DHelper(keypoint_mode='lm68')'s: the mean, id and exp basis rows at model['keypoints'] AS STORED.  The file
    holds 1-based indices and ParametricFaceModel subtracts 1 (bfm.py:65), but Face3DHelper does not, so the reference's torso key points sit
    one vertex after the 68 landmarks; the torso model was trained on exactly those points, so they are reproduced here.

    reconstruct_lm2d(id, exp, euler, trans) is Face3DHelper.reconstruct_lm2d; clip(...) is the whole per-clip motion (see its docstring)."""

    def __init__(self, bfm_folder: str = 'deep_3drecon/BFM', device='cuda'):
        super().__init__()
        m = load_keypoint_bfm(bfm_folder)
        self.n_id, self.n_exp = m['id_base'].shape[1], m['exp_base'].shape[1]
        if (self.n_id + self.n_exp) % 4 or self.n_id + self.n_exp > 256:
            raise NotImplementedError('ClipMotion: id + exp coefficients must be a multiple of 4, at most 256')
        kp = m['keypoints']
        self.n_kp = kp.size
        rows = (3 * kp[:, None] + np.arange(3)[None]).reshape(-1)                      # rows 3v + axis of the gathered vertices
        basis = np.ascontiguousarray(np.concatenate([m['id_base'][rows], m['exp_base'][rows]], 1))
        self.tan_half = CENTER / FOCAL                                                 # tan(fov / 2) of the reference's projection
        self.register_buffer('basis', torch.from_numpy(basis), persistent=False)       # [3 K, n_id + n_exp]
        self.register_buffer('mean_shape', torch.from_numpy(np.ascontiguousarray(m['mean'][kp].reshape(-1))), persistent=False)
        self.register_buffer('keypoints', torch.from_numpy(kp), persistent=False)
        self.to(device)

    # ---- validation ----------------------------------------------------------------------------------------------------------------------
    def _rows(self, x: torch.Tensor, n: int, what: str, T: Optional[int] = None, shape_only: bool = False) -> Tuple[torch.Tensor, int]:
        """[T, n] (or wider rows) fp32 CUDA -> (tensor read in place, row stride); a [1, n] row broadcasts with stride 0 when T is given."""
        if not isinstance(x, torch.Tensor) or x.ndim != 2 or x.shape[1] != n or (T is not None and x.shape[0] not in (1, T)) or x.shape[0] < 1:
            want = f'[{T},{n}] or [1,{n}]' if T is not None else f'[T,{n}]'
            raise ValueError(f'ClipMotion: {what} must be a tensor {want}, got {tuple(getattr(x, "shape", ()))}')
        if shape_only:
            return x, 0
        if not x.is_cuda:
            raise RuntimeError(f'real3dportrait_b200 runs on CUDA tensors only (no CPU fallback); {what} is not a CUDA tensor')
        if x.device != self.basis.device:
            raise ValueError(f'ClipMotion: {what} is on {x.device}, the BFM on {self.basis.device}')
        if x.dtype != torch.float32 or x.stride(1) != 1 or (x.shape[0] > 1 and x.stride(0) < n):
            x = x.detach().float().contiguous()                                        # plumbing copy; fp32 unit-stride rows are read in place
        stride = 0 if x.shape[0] == 1 else x.stride(0)
        return x, stride

    def _vec3(self, x, what: str, rows: Optional[int] = None, shape_only: bool = False) -> torch.Tensor:
        if not isinstance(x, torch.Tensor) or x.ndim != 2 or x.shape[1] != 3 or (rows is not None and x.shape[0] != rows) or x.shape[0] < 1:
            raise ValueError(f'ClipMotion: {what} must be a tensor [{rows if rows is not None else "P"},3] with at least one row, '
                             f'got {tuple(getattr(x, "shape", ()))}')
        if shape_only:
            return x
        if not x.is_cuda:
            raise RuntimeError(f'real3dportrait_b200 runs on CUDA tensors only (no CPU fallback); {what} is not a CUDA tensor')
        if x.device != self.basis.device:
            raise ValueError(f'ClipMotion: {what} is on {x.device}, the BFM on {self.basis.device}')
        return capi.f32(x)

    def _vertices(self, id_t, ids, exp_t, exps, euler, trans, B, verts):
        L, p = capi.lib(), capi.ptr
        capi.check(L.r3dp_secc_vertices(p(self.basis), p(self.mean_shape), self.n_kp, self.n_id, self.n_exp,
                                        ctypes.c_void_p(id_t.data_ptr()), ids, ctypes.c_void_p(exp_t.data_ptr()), exps, p(euler), p(trans), B,
                                        CAMERA_DISTANCE, self.tan_half, p(verts), capi.stream()))

    # ---- Face3DHelper.reconstruct_lm2d ---------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def reconstruct_lm2d(self, id_coeff: torch.Tensor, exp_coeff: torch.Tensor, euler: torch.Tensor, trans: torch.Tensor) -> torch.Tensor:
        """Face3DHelper(keypoint_mode='lm68').reconstruct_lm2d: id [T,80], exp [T,64], euler, trans [T,3] (or [B,T,C] each) -> lm2d
        [T,68,2] (or [B,T,68,2]) in image coordinates / 224, y down."""
        bt = id_coeff.shape[:2] if id_coeff.ndim == 3 else None
        if bt is not None:
            id_coeff, exp_coeff, euler, trans = (x.reshape(bt[0] * bt[1], -1) for x in (id_coeff, exp_coeff, euler, trans))
        T = id_coeff.shape[0]
        id_t, ids = self._rows(id_coeff, self.n_id, 'id', T)
        exp_t, exps = self._rows(exp_coeff, self.n_exp, 'exp')
        if exp_t.shape[0] != T:
            raise ValueError(f'ClipMotion: exp has {exp_t.shape[0]} rows, id {T}')
        euler, trans = self._vec3(euler, 'euler', T), self._vec3(trans, 'trans', T)
        verts = torch.empty(T, self.n_kp, 4, device=self.basis.device)
        lm2d = torch.empty(T, self.n_kp, 2, device=self.basis.device)
        with capi.region('motion.lm2d'):
            self._vertices(id_t, ids, exp_t, exps, euler, trans, T, verts)
            capi.check(capi.lib().r3dp_motion_lm2d(capi.ptr(verts), T * self.n_kp, capi.ptr(lm2d), capi.stream()))
        return lm2d if bt is None else lm2d.reshape(bt[0], bt[1], self.n_kp, 2)

    # ---- the clip ------------------------------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def clip(self, id: torch.Tensor, exp: torch.Tensor, src_euler: torch.Tensor, src_trans: torch.Tensor, src_exp: torch.Tensor,
             pose: Optional[Sequence[torch.Tensor]] = None, map_to_init_pose: bool = True,
             out: Optional[Sequence[torch.Tensor]] = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """A clip's motion -> (cameras [T,25], kp_s [1,68,3], kp_d [T,68,3]), fp32 contiguous.

        id [1,80] (the source's, broadcast as src_id.repeat) or [T,80]; exp [T,64], e.g. the column slice rows[:, 80:144] of the engine's
        [id | exp | t | T] rows (fp32 rows with unit column stride are read in place); src_euler, src_trans [1,3] and src_exp [1,64]: the
        source frame's fit (kp_s is taken at id[0], src_exp and the source pose).  pose: None for the 'static' pose (the source pose on
        every frame), else (euler [P,3], trans [P,3]) of the driving sequence, P >= 1, read back and forth with mirror_index.
        map_to_init_pose moves the trajectory so that frame 0 has the source pose (real3d_infer.py's default).  T >= 3: the reference's key-point
        smoothing raises below that.  out=(cameras, kp_s, kp_d): fp32 contiguous CUDA buffers of those shapes, written in place.
        No host sync: the call can be captured in a CUDA graph (with out= given, a replay writes the same buffers)."""
        T = exp.shape[0] if isinstance(exp, torch.Tensor) and exp.ndim == 2 else None
        if T is not None and T < 3:
            raise ValueError(f'ClipMotion.clip: a clip needs at least 3 frames (the 7-frame key-point smoothing mirrors 3 at each end), got {T}')
        if pose is not None and (not isinstance(pose, (tuple, list)) or len(pose) != 2):
            raise ValueError('ClipMotion.clip: pose is None (static) or (euler [P,3], trans [P,3])')
        for shape_only in (True, False):                                               # every shape error before a device error
            exp_t, exps = self._rows(exp, self.n_exp, 'exp', None, shape_only)
            id_t, ids = self._rows(id, self.n_id, 'id', T, shape_only)
            s_exp, _ = self._rows(src_exp, self.n_exp, 'src_exp', 1, shape_only)
            s_e, s_t = self._vec3(src_euler, 'src_euler', 1, shape_only), self._vec3(src_trans, 'src_trans', 1, shape_only)
            if pose is None:
                d_e, d_t = s_e, s_t                                                    # 'static': the source pose, P = 1
            else:
                d_e = self._vec3(pose[0], 'pose euler', None, shape_only)
                d_t = self._vec3(pose[1], 'pose trans', d_e.shape[0], shape_only)
        P = d_e.shape[0]
        dev = self.basis.device
        K = self.n_kp
        if out is None:
            cameras, kp_s, kp_d = torch.empty(T, 25, device=dev), torch.empty(1, K, 3, device=dev), torch.empty(T, K, 3, device=dev)
        else:
            if len(out) != 3:
                raise ValueError('ClipMotion.clip: out = (cameras, kp_s, kp_d)')
            cameras, kp_s, kp_d = out
            for t, shp, what in ((cameras, (T, 25), 'cameras'), (kp_s, (1, K, 3), 'kp_s'), (kp_d, (T, K, 3), 'kp_d')):
                if (not isinstance(t, torch.Tensor) or not t.is_cuda or t.device != dev or t.dtype != torch.float32 or tuple(t.shape) != shp
                        or not t.is_contiguous()):
                    raise ValueError(f'ClipMotion.clip: out {what} must be a contiguous fp32 tensor {list(shp)} on {dev}')
        euler, trans = torch.empty(T, 3, device=dev), torch.empty(T, 3, device=dev)
        verts_s, verts_d = torch.empty(1, K, 4, device=dev), torch.empty(T, K, 4, device=dev)
        L, p, st = capi.lib(), capi.ptr, capi.stream()
        with capi.region('motion.clip'):
            capi.check(L.r3dp_motion_camera(p(s_e), p(s_t), p(d_e), p(d_t), P, T, int(bool(map_to_init_pose)), p(euler), p(trans), p(cameras), st))
            self._vertices(id_t, 0, s_exp, 0, s_e, s_t, 1, verts_s)
            self._vertices(id_t, ids, exp_t, exps, euler, trans, T, verts_d)
            capi.check(L.r3dp_motion_keypoints(p(verts_s), p(verts_d), T, K, p(kp_s), p(kp_d), st))
        return cameras, kp_s, kp_d
