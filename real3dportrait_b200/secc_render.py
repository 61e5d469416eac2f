"""SECC_Renderer (deep_3drecon/secc_renderer.py) on libr3dp_b200: the BFM face mesh of a frame's 3DMM coefficients, rasterised with pytorch3d's
rules and shaded with the per-vertex NCC code, in three launches (r3dp_secc_vertices, r3dp_secc_raster, r3dp_secc_resolve) with no pytorch3d.

The constructor reads the reference's files (BFM_model_front.mat, ncc_code.npy, the two eye face lists) from the same cwd-relative defaults, so
`SECC_Renderer(512)` replaces the reference class where real3d_infer.py builds it.  Only `meanshape`, `idBase`, `exBase` and `tri` are read from
the .mat; converting 01_MorphableModel.mat (the reference's transferBFM09) is not done here."""
from __future__ import annotations

import ctypes
import math
import os
from typing import Optional, Sequence

import numpy as np
import torch
import torch.nn as nn

from . import _capi as capi

FOCAL, CENTER, CAMERA_DISTANCE = 1015.0, 112.0, 10.0        # ParametricFaceModel defaults (bfm.py:29-39)
ZNEAR, ZFAR = 5.0, 15.0                                      # secc_renderer.py:14-15 (no z clipping is applied: pytorch3d's default)


def _need(path: str, what: str) -> str:
    if not os.path.isfile(path):
        raise FileNotFoundError(f'SECC_Renderer: {what} not found at {path!r}')
    return path


def load_bfm(bfm_folder: str, ncc_path: str, eye_faces: Sequence[str]):
    """-> dict of numpy arrays: mean [N,3] float32 recentred (bfm.py:78-81), id_base [3N,n_id], exp_base [3N,n_exp] float32, faces [F,3] int64
    0-based without the eye faces (secc_renderer.py:23-32), ncc [N,3] float32."""
    from scipy.io import loadmat
    mat = loadmat(_need(os.path.join(bfm_folder, 'BFM_model_front.mat'), 'BFM_model_front.mat'))
    missing = [k for k in ('meanshape', 'idBase', 'exBase', 'tri') if k not in mat]
    if missing:
        raise KeyError(f'SECC_Renderer: BFM_model_front.mat lacks {missing}')
    mean = mat['meanshape'].astype(np.float32).reshape(-1, 3)
    mean = mean - np.mean(mean, axis=0, keepdims=True)
    id_base, exp_base = mat['idBase'].astype(np.float32), mat['exBase'].astype(np.float32)
    n = mean.shape[0]
    if id_base.shape[0] != 3 * n or exp_base.shape[0] != 3 * n:
        raise ValueError(f'SECC_Renderer: idBase {id_base.shape} / exBase {exp_base.shape} do not match {n} vertices')
    tri = mat['tri'].astype(np.int64) - 1
    drop = np.zeros(tri.shape[0], dtype=bool)
    for p in eye_faces:
        drop[np.load(_need(p, 'eye face list')).astype(np.int64).reshape(-1) - 1] = True
    faces = tri[~drop]
    ncc = np.load(_need(ncc_path, 'ncc_code.npy'), allow_pickle=True).astype(np.float32)
    if ncc.shape != (3, n):
        raise ValueError(f'SECC_Renderer: ncc_code has shape {ncc.shape}, expected (3, {n})')
    if faces.min() < 0 or faces.max() >= n:
        raise ValueError('SECC_Renderer: tri indexes a vertex outside the mesh')
    return {'mean': mean, 'id_base': id_base, 'exp_base': exp_base, 'faces': faces, 'ncc': ncc.T}


def flatten_btc(*xs):
    """[B,T,C] inputs -> [B*T,C] (secc_renderer.py:42-47); [B,C] inputs pass through."""
    return tuple(x.reshape(x.shape[0] * x.shape[1], -1) if x.ndim == 3 else x for x in xs)


def unflatten_btc(y: torch.Tensor, bt) -> torch.Tensor:
    """[B*T,C,H,W] -> [B,C,T,H,W] (the reference's rearrange '(n t) c h w -> n c t h w') when bt = (B, T); else unchanged."""
    if bt is None:
        return y
    b, t = bt
    return y.reshape(b, t, *y.shape[1:]).permute(0, 2, 1, 3, 4)


class SECC_Renderer(nn.Module):
    """forward(id, exp, euler, trans) -> (face_mask [B,1,S,S], secc [B,3,S,S]) with S = rasterize_size (default 224); [B,T,C] inputs give
    [B,C,T,S,S].  secc is 2 mask sum_i w_i ncc_i - 1 (background -1).  As in the reference, face 0 of the first image of a call counts as
    background (mesh_renderer.py:116 tests pix_to_face > 0 on pytorch3d's packed face index).  CUDA tensors only.

    render(coeff [B, n_id + n_exp], ...) is the same call on one [id | exp] tensor, for FrameEngine(secc_renderer=...).  Calls on one renderer
    are stream-ordered: the kernels share a key buffer per (device, batch, size) that every call leaves empty.  Key buffers live as long as the
    renderer (and whoever holds graph_buffers()); .to() adds buffers for the new device and frees none."""

    def __init__(self, rasterize_size=None, device='cuda', bfm_folder='deep_3drecon/BFM', ncc_path='deep_3drecon/ncc_code.npy',
                 eye_faces=('deep_3drecon/bfm_right_eye_faces.npy', 'deep_3drecon/bfm_left_eye_faces.npy')):
        super().__init__()
        m = load_bfm(bfm_folder, ncc_path, eye_faces)
        self.fov = 2 * np.arctan(CENTER / FOCAL) * 180 / np.pi
        self.tan_half = math.tan(math.radians(self.fov) / 2)
        self.znear, self.zfar = ZNEAR, ZFAR
        self.rasterize_size = int(2 * CENTER if rasterize_size is None else rasterize_size)
        self.n_id, self.n_exp = m['id_base'].shape[1], m['exp_base'].shape[1]
        if (self.n_id + self.n_exp) % 4 or self.n_id + self.n_exp > 256:
            raise NotImplementedError('SECC_Renderer: id + exp coefficients must be a multiple of 4, at most 256')
        self.n_verts, self.n_faces = m['mean'].shape[0], m['faces'].shape[0]
        ncc4 = np.zeros((self.n_verts, 4), dtype=np.float32)
        ncc4[:, :3] = m['ncc']
        # one [3N, n_id + n_exp] basis: each row read once per call (r3dp_secc_vertices)
        c = np.ascontiguousarray                                   # loadmat returns Fortran-ordered arrays
        self.register_buffer('basis', torch.from_numpy(c(np.concatenate([m['id_base'], m['exp_base']], 1))), persistent=False)
        self.register_buffer('mean_shape', torch.from_numpy(c(m['mean'].reshape(-1))), persistent=False)
        self.register_buffer('face_buf', torch.from_numpy(c(m['faces'].astype(np.int32))), persistent=False)
        self.register_buffer('ncc', torch.from_numpy(ncc4), persistent=False)
        self._keys = {}
        self.to(device)

    def key_buffer(self, B: int, S: int) -> torch.Tensor:
        """The [B,S,S] uint64 key buffer (held as int64, all bits set = empty) of this (device, batch, size); filled once, kept empty by every
        call, never dropped: a CUDA graph captured over a call keeps writing to it."""
        key = (self.basis.device, B, S)
        kb = self._keys.get(key)
        if kb is None:
            kb = torch.full((B, S, S), -1, dtype=torch.int64, device=self.basis.device)
            self._keys[key] = kb
        return kb

    def graph_buffers(self, B: int, S: Optional[int] = None):
        """Every buffer of this renderer that a call of batch B at size S (default rasterize_size) reads or writes: a CUDA graph captured over
        such a call holds these, so that a later .to() of the renderer cannot free them under the captured pointers."""
        return (self.basis, self.mean_shape, self.face_buf, self.ncc, self.key_buffer(B, self.rasterize_size if S is None else int(S)))

    def _vec(self, t, B, what, n):
        if t is None:
            return None
        if not t.is_cuda:
            raise RuntimeError('real3dportrait_b200 runs on CUDA tensors only (no CPU fallback); got a CPU tensor')
        t = capi.f32(t)
        if t.shape != (B, n):
            raise ValueError(f'SECC_Renderer: {what} must be [{B},{n}], got {tuple(t.shape)}')
        return t

    def _run(self, id_p, ids, exp_p, exps, B, euler, trans, S, drop_face0, with_mask):
        """id_p / exp_p: device pointers of the [B, >= n_id] / [B, >= n_exp] rows (row strides ids / exps)."""
        L, st, ptr = capi.lib(), capi.stream(), capi.ptr
        dev = self.basis.device
        verts = torch.empty(B, self.n_verts, 4, device=dev)
        secc = torch.empty(B, 3, S, S, device=dev)
        mask = torch.empty(B, 1, S, S, device=dev) if with_mask else None
        keys = self.key_buffer(B, S)
        with capi.region('secc_render'):
            with capi.region('secc_render.vertices'):
                capi.check(L.r3dp_secc_vertices(ptr(self.basis), ptr(self.mean_shape), self.n_verts, self.n_id, self.n_exp, id_p, ids,
                                                exp_p, exps, ptr(euler), ptr(trans), B, CAMERA_DISTANCE, self.tan_half, ptr(verts), st))
            with capi.region('secc_render.raster'):
                capi.check(L.r3dp_secc_raster(ptr(verts), self.n_verts, ptr(self.face_buf, torch.int32), self.n_faces, B, S,
                                              ptr(keys, torch.int64), st))
            with capi.region('secc_render.resolve'):
                capi.check(L.r3dp_secc_resolve(ptr(verts), self.n_verts, ptr(self.face_buf, torch.int32), ptr(self.ncc), B, S, int(drop_face0),
                                               ptr(keys, torch.int64), ptr(secc), ptr(mask), st))
        return mask, secc, verts

    def render(self, coeff: torch.Tensor, euler: Optional[torch.Tensor] = None, trans: Optional[torch.Tensor] = None, size: Optional[int] = None,
               drop_face0: bool = True, with_mask: bool = False):
        """coeff [B, n_id + n_exp] = [id | exp] (CUDA), euler / trans [B,3] or None (zero pose) -> (mask [B,1,S,S] or None, secc [B,3,S,S])."""
        K = self.n_id + self.n_exp
        if coeff.ndim != 2 or coeff.shape[1] != K:
            raise ValueError(f'SECC_Renderer.render: coeff must be [B,{K}] (id | exp), got {tuple(coeff.shape)}')
        B = coeff.shape[0]
        c = self._vec(coeff, B, 'coeff', K)
        S = self.rasterize_size if size is None else int(size)
        exp_p = ctypes.c_void_p(c.data_ptr() + 4 * self.n_id)         # the exp columns of the same rows
        mask, secc, _ = self._run(capi.ptr(c), K, exp_p, K, B, self._vec(euler, B, 'euler', 3), self._vec(trans, B, 'trans', 3), S,
                                  drop_face0, with_mask)
        return mask, secc

    def forward(self, id, exp, euler, trans):
        """id [B,80], exp [B,64], euler, trans [B,3] (or [B,T,C] each) -> (face_mask [B,1,S,S], secc [B,3,S,S]) (or [B,C,T,S,S])."""
        bt = id.shape[:2] if id.ndim == 3 else None
        id, exp, euler, trans = flatten_btc(id, exp, euler, trans)
        B = id.shape[0]
        id_t, exp_t = self._vec(id, B, 'id', self.n_id), self._vec(exp, B, 'exp', self.n_exp)
        mask, secc, _ = self._run(capi.ptr(id_t), self.n_id, capi.ptr(exp_t), self.n_exp, B, self._vec(euler, B, 'euler', 3),
                                  self._vec(trans, B, 'trans', 3), self.rasterize_size, True, True)
        return unflatten_btc(mask, bt), unflatten_btc(secc, bt)
