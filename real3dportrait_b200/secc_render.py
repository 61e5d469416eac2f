"""SECC_Renderer (deep_3drecon/secc_renderer.py) on libr3dp_b200: the BFM face mesh of a frame's 3DMM coefficients, rasterised with pytorch3d's
rules and shaded with the per-vertex NCC code, in three launches (r3dp_secc_vertices, r3dp_secc_raster, r3dp_secc_resolve) with no pytorch3d.

The constructor reads the reference's files (BFM_model_front.mat, ncc_code.npy, the two eye face lists) from the same cwd-relative defaults, so
`SECC_Renderer(512)` replaces the reference class where real3d_infer.py builds it.  Only `meanshape`, `idBase`, `exBase` and `tri` are read from
the .mat; converting 01_MorphableModel.mat (the reference's transferBFM09) is not done here."""
from __future__ import annotations

import ctypes
import math
import os
import random
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

    render(coeff [B, >= n_id + n_exp], ...) is the same call on one [id | exp | ...] tensor, for FrameEngine(secc_renderer=...).  blink(secc,
    ...) closes the eyes of rendered images in place (blink_eye_for_secc, batched).  Calls on one renderer are stream-ordered: the kernels share
    a key buffer and a blink scratch buffer per (device, batch, size).  These buffers live as long as the renderer (and whoever holds
    graph_buffers()); .to() adds buffers for the new device and frees none."""

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
        self._blink = _BlinkBuffers()
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

    def graph_buffers(self, B: int, S: Optional[int] = None, blink: bool = False):
        """Every buffer of this renderer that a call of batch B at size S (default rasterize_size) reads or writes (with blink=True, a blink()
        call's scratch and fault counter too): a CUDA graph captured over such calls holds these, so that a later .to() of the renderer cannot
        free them under the captured pointers."""
        S = self.rasterize_size if S is None else int(S)
        bufs = (self.basis, self.mean_shape, self.face_buf, self.ncc, self.key_buffer(B, S))
        return bufs + (self._blink.scratch(self.basis.device, B, S), self._blink.counter(self.basis.device)) if blink else bufs

    def blink(self, secc: torch.Tensor, p=None, rows: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Close the eyes of secc [B,3,S,S] (fp32 CUDA, contiguous; 64 <= S <= 1024) in place, as blink_eye_for_secc does each image, and
        return it.  Per image, exactly one of:
          p     a float per image (a sequence, or a float64 CUDA tensor [B]): the close-eye fraction; a negative value leaves the image untouched.
          rows  [B, >= 2] fp32 CUDA whose columns 0 and 1 hold (t, T) (a column slice such as coeff[:, 144:] is read in place): p is
                -4/T**2 * t**2 + 4/T * t in double on int(t), int(T).  The image is untouched unless 0 <= t < T <= 4096 and
                int(t) < int(T): T = 0, t >= T, negative, NaN and infinite entries and T > 4096 leave it untouched.
        Untouched images are not written; p = 0 only quantises.  An image on which the reference raises is left as it is and counted
        (blink_faults()).  No host synchronisation (capturable), except to copy a host sequence p."""
        return _blink(self._blink, secc, p, rows)

    def blink_faults(self, reset: bool = True) -> int:
        """Images blink() left unedited because the reference raises on them, since the last reset (one device sync)."""
        return self._blink.faults(self.basis.device, reset)

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
        """coeff [B, n_id + n_exp] = [id | exp] (CUDA; wider rows [id | exp | ...] are read in place), euler / trans [B,3] or None (zero pose) -> (mask [B,1,S,S] or None, secc [B,3,S,S])."""
        K = self.n_id + self.n_exp
        if coeff.ndim != 2 or coeff.shape[1] < K:
            raise ValueError(f'SECC_Renderer.render: coeff must be [B,{K}] (id | exp) or wider, got {tuple(coeff.shape)}')
        B = coeff.shape[0]
        if not coeff.is_cuda:
            raise RuntimeError('real3dportrait_b200 runs on CUDA tensors only (no CPU fallback); got a CPU tensor')
        c = capi.f32(coeff)                                             # wider rows are read in place through their row stride
        S = self.rasterize_size if size is None else int(size)
        W = c.shape[1]
        exp_p = ctypes.c_void_p(c.data_ptr() + 4 * self.n_id)         # the exp columns of the same rows
        mask, secc, _ = self._run(capi.ptr(c), W, exp_p, W, B, self._vec(euler, B, 'euler', 3), self._vec(trans, B, 'trans', 3), S,
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


# ---- blink_eye_for_secc (inference/edit_secc.py) -------------------------------------------------------------------------------------------

class _BlinkBuffers:
    """The blink kernels' scratch per (device, batch, size) and a fault counter per device.  Each call initialises the scratch it reads, so
    a graph needs no memset; buffers are never dropped (a graph captured over a call keeps writing to them)."""

    def __init__(self):
        self._scratch, self._faults = {}, {}

    def scratch(self, device, B: int, S: int) -> torch.Tensor:
        key = (torch.device(device), B, S)
        t = self._scratch.get(key)
        if t is None:
            n = int(capi.lib().r3dp_secc_blink_scratch_bytes(B, S))
            if n == 0:
                raise ValueError(f'blink: SECC images must be square with 64 <= S <= 1024, got S = {S}')
            t = torch.empty(n + 256, dtype=torch.uint8, device=device)       # the kernels want 256-byte alignment
            off = (-t.data_ptr()) % 256
            t = t[off:off + n]
            self._scratch[key] = t
        return t

    def counter(self, device) -> torch.Tensor:
        key = torch.device(device)
        t = self._faults.get(key)
        if t is None:
            t = self._faults[key] = torch.zeros(1, dtype=torch.int32, device=device)
        return t

    def faults(self, device, reset: bool = True) -> int:
        c = self.counter(device)
        n = int(c.item())
        if reset and n:
            c.zero_()
        return n


def _blink(bufs: _BlinkBuffers, secc: torch.Tensor, p, rows):
    if (p is None) == (rows is None):
        raise ValueError('blink: give exactly one of p and rows')
    if not secc.is_cuda:
        raise RuntimeError('real3dportrait_b200 runs on CUDA tensors only (no CPU fallback); got a CPU tensor')
    if secc.dtype != torch.float32 or secc.ndim != 4 or secc.shape[1] != 3 or secc.shape[2] != secc.shape[3] or not secc.is_contiguous():
        raise ValueError(f'blink: secc must be a contiguous fp32 [B,3,S,S], got {secc.dtype} {tuple(secc.shape)}')
    B, S = secc.shape[0], secc.shape[2]
    if not 64 <= S <= 1024:
        raise ValueError(f'blink: 64 <= S <= 1024, got {S}')
    dev = secc.device
    p_t = r_t = None
    stride = 0
    if p is not None:
        if isinstance(p, torch.Tensor):
            p_t = p.to(dev, torch.float64).contiguous()
        else:
            p_t = torch.tensor([float(v) for v in p], dtype=torch.float64).to(dev)
        if p_t.shape != (B,):
            raise ValueError(f'blink: p must hold {B} values, got {tuple(p_t.shape)}')
    else:
        if not rows.is_cuda or rows.dtype != torch.float32 or rows.ndim != 2 or rows.shape[0] != B or rows.shape[1] < 2 or rows.stride(1) != 1:
            raise ValueError(f'blink: rows must be fp32 CUDA [{B}, >= 2] with unit column stride, got {rows.dtype} {tuple(rows.shape)}')
        r_t, stride = rows, rows.stride(0)
        if B > 1 and stride < 2:
            raise ValueError('blink: rows must not overlap')
        stride = max(stride, 2)
    sc, cnt = bufs.scratch(dev, B, S), bufs.counter(dev)
    with capi.region('secc_blink'):
        capi.check(capi.lib().r3dp_secc_blink(capi.ptr(secc), B, S, capi.ptr(p_t, torch.float64),
                                              ctypes.c_void_p(0 if r_t is None else r_t.data_ptr()), stride,
                                              capi.ptr(sc, torch.uint8), capi.ptr(cnt, torch.int32), capi.stream()))
    return secc


_DROPIN = _BlinkBuffers()


def blink_eye_for_secc(img: torch.Tensor, close_eye_percent: float = 0.5) -> torch.Tensor:
    """inference/edit_secc.py's blink_eye_for_secc on the GPU: img [3,S,S] in [-1,1] (CUDA) -> a new [3,S,S] fp32 image on img's device (the
    reference returns a CPU tensor).  Raises ValueError for close_eye_percent outside [0, 1] and wherever the reference raises (then after a
    device sync).  Ties between nearest face pixels go to the lowest row-major index (the reference's k-d tree picks its own)."""
    p = float(close_eye_percent)
    if not 0.0 <= p <= 1.0:
        raise ValueError(f'blink_eye_for_secc: close_eye_percent must lie in [0, 1], got {close_eye_percent}')
    if img.ndim != 3 or img.shape[0] != 3:
        raise ValueError(f'blink_eye_for_secc: img must be [3,S,S], got {tuple(img.shape)}')
    out = capi.f32(img).clone().unsqueeze(0)
    _blink(_DROPIN, out, [p], None)
    if _DROPIN.faults(out.device):
        raise ValueError('blink_eye_for_secc: no eye hole in one of the prior eye regions, or no face pixel left around the eyes '
                         '(the reference raises here too)')
    return out[0]


def period_blink_schedule(num_frames: int, rng=random, fps: int = 25, period: int = 5) -> torch.Tensor:
    """real3d_infer.py's blink_mode='period' windows: int32 [num_frames, 2] of (t, T), T = 0 for frames left untouched.  At every frame i
    with i % (fps * period) == 0 a duration T = rng.randint(8, 12) is drawn, and frames i + t, t < T, get (t, T), stopping at the last frame
    (never blinked).  random.seed(s) before the call reproduces the reference's windows for the same draws."""
    n, every = int(num_frames), int(fps) * int(period)
    if every < 12:
        raise ValueError('period_blink_schedule: fps * period must be at least 12 (windows would overlap)')
    out = torch.zeros(max(n, 0), 2, dtype=torch.int32)
    for i in range(0, n, every):
        T = rng.randint(8, 12)
        for t in range(T):
            if i + t >= n - 1:
                break
            out[i + t, 0], out[i + t, 1] = t, T
    return out
