"""Source images on libr3dp_b200: the torso head's per-clip images from the source image and its segmap, as real3d_infer.py:243-260 builds
them on the host with cv2, scipy and sklearn (DESIGN.md, "Source images"):

  ref_head_img   MediapipeSegmenter._seg_out_img_with_segmap(img, segmap, 'head')   (r3dp_src_compose)
  ref_torso_img  inpaint_torso_job(img, segmap)[0]                                   (r3dp_src_inpaint, r3dp_src_compose)
  bg_img         extract_background([img], [segmap], 'knn')                          (r3dp_src_bg_distance, r3dp_src_bg_fill)

Every output is bit-identical to the reference's ((torch.tensor(u8) - 127.5) / 127.5) of its uint8 image, except that extract_background's
choice among equidistant nearest pixels, which sklearn's k-d tree leaves unspecified, is fixed here: the smallest column, then the smallest
row.  prepare_source's outputs feed FrameEngine: begin_planes(img=ref_head_img, ...) and begin_clip(ref_torso_img, bg_img, segmap, kp_s)."""
from __future__ import annotations

import ctypes
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from . import _capi as capi

MIN_SIZE, MAX_SIZE = 64, 1024
TORSO_ROWS, NECK_ROWS = 9, 53                       # inpaint_torso_job: L = 8 + 1 and 48 + 4 + 1
OUTPUTS = ('ref_head_img', 'ref_torso_img', 'bg_img')
_G_BYTES = 256 << 20                                 # extract_background's per-chunk distance scratch

_tables: Dict[torch.device, Tuple[torch.Tensor, torch.Tensor]] = {}


def darken_table(L: int) -> np.ndarray:
    """inpaint_torso_job's darkening factors, numpy's 0.98 ** np.arange(L) (not bit-identical to Python's 0.98 ** k for every k)."""
    return 0.98 ** np.arange(L)


def _darken_tables(dev: torch.device) -> Tuple[torch.Tensor, torch.Tensor]:
    if dev not in _tables:
        _tables[dev] = tuple(torch.from_numpy(darken_table(L)).to(dev) for L in (TORSO_ROWS, NECK_ROWS))
    return _tables[dev]


def frame_interval(n: int) -> int:
    """extract_background's FRAME_SELECT_INTERVAL for n frames."""
    return 5 if n < 100 else 20 if n < 10000 else n // 500


def selected_frames(n: int) -> range:
    """The frames extract_background reads: [::interval] when n > interval, else frame 0 alone."""
    i = frame_interval(n)
    return range(0, n, i) if n > i else range(0, 1)


# ---- validation ---------------------------------------------------------------------------------------------------------------------------
def _size(H: int, W: int, what: str) -> None:
    if not (MIN_SIZE <= H <= MAX_SIZE and MIN_SIZE <= W <= MAX_SIZE):
        raise ValueError(f'{what}: H and W must lie in [{MIN_SIZE}, {MAX_SIZE}], got {H} x {W}')


def _images(x, what: str, batched: bool) -> torch.Tensor:
    if not isinstance(x, torch.Tensor):
        raise ValueError(f'{what} must be a torch tensor, got {type(x).__name__}')
    nd = 4 if batched else 3
    if x.dtype != torch.uint8 or x.ndim != nd or x.shape[-1] != 3 or (batched and x.shape[0] < 1):
        want = '[N,H,W,3]' if batched else '[H,W,3]'
        raise ValueError(f'{what} must be a uint8 RGB tensor {want}, got {x.dtype} {tuple(x.shape)}')
    _size(x.shape[-3], x.shape[-2], what)
    return x


def _segmaps(x, what: str, lead: Tuple[Tuple[int, ...], ...], H: int, W: int) -> torch.Tensor:
    if not isinstance(x, torch.Tensor):
        raise ValueError(f'{what} must be a torch tensor, got {type(x).__name__}')
    if x.dtype not in (torch.float32, torch.uint8):
        raise ValueError(f'{what} must be float32 or uint8, got {x.dtype}')
    if tuple(x.shape[-3:]) != (6, H, W) or tuple(x.shape[:-3]) not in lead:
        raise ValueError(f'{what} must be {" or ".join(str(list(l) + [6, H, W]) for l in lead)}, got {tuple(x.shape)}')
    return x


def _on_device(xs, whats) -> torch.device:
    """Every shape and dtype error comes first; then CPU tensors (no fallback) and mixed devices."""
    for x, what in zip(xs, whats):
        if not x.is_cuda:
            raise RuntimeError(f'real3dportrait_b200 runs on CUDA tensors only (no CPU fallback); {what} is not a CUDA tensor')
    dev = xs[0].device
    for x, what in zip(xs[1:], whats[1:]):
        if x.device != dev:
            raise ValueError(f'{what} is on {x.device}, {whats[0]} on {dev}')
    return dev


def _out(t, shape, dtype, what: str, device) -> torch.Tensor:
    if (not isinstance(t, torch.Tensor) or not t.is_cuda or t.device != device or t.dtype != dtype or tuple(t.shape) != tuple(shape)
            or not t.is_contiguous()):
        raise ValueError(f'out {what} must be a contiguous {dtype} tensor {list(shape)} on {device}')
    return t


def _seg_u8(seg: torch.Tensor) -> int:
    return int(seg.dtype == torch.uint8)


def _p(t: Optional[torch.Tensor]) -> ctypes.c_void_p:
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


# ---- launches ----------------------------------------------------------------------------------------------------------------------------
def _torso(img: torch.Tensor, seg: torch.Tensor, head_f32=None, torso_f32=None, torso_u8=None) -> None:
    H, W = img.shape[0], img.shape[1]
    tab_t, tab_n = _darken_tables(img.device)
    img2 = torch.empty(H, W, 3, dtype=torch.uint8, device=img.device)
    flags = torch.empty(H, W, dtype=torch.uint8, device=img.device)
    L, st = capi.lib(), capi.stream()
    capi.check(L.r3dp_src_inpaint(_p(img), _p(seg), _seg_u8(seg), H, W, _p(tab_t), _p(tab_n), _p(img2), _p(flags), st))
    capi.check(L.r3dp_src_compose(_p(img), _p(seg), _seg_u8(seg), _p(img2), _p(flags), H, W, _p(head_f32), _p(torso_f32), _p(torso_u8), st))


def _background(frames: torch.Tensor, segs: torch.Tensor, bg_u8=None, bg_f32=None) -> None:
    """frames [N,H,W,3] uint8, segs [N,6,H,W]: the selected frames are read in place (strided by the interval), nothing else is."""
    N, H, W = frames.shape[0], frames.shape[1], frames.shape[2]
    sel = selected_frames(N)
    I, F = sel.step, len(sel)
    dev = frames.device
    chunk = max(1, min(F, _G_BYTES // (2 * H * W)))
    g = torch.empty(chunk, H, W, dtype=torch.int16, device=dev)
    maxd2 = torch.empty(H, W, dtype=torch.int32, device=dev)
    argmax = torch.empty(H, W, dtype=torch.int32, device=dev)
    flags = torch.empty(F + 1, dtype=torch.int32, device=dev)        # has_fg per selected frame, then has_bc
    L, st = capi.lib(), capi.stream()
    capi.check(L.r3dp_src_bg_distance(_p(segs), _seg_u8(segs), I * 6 * H * W, F, H, W, _p(g), chunk, _p(maxd2), _p(argmax), _p(flags), st))
    capi.check(L.r3dp_src_bg_fill(_p(frames), I * H * W * 3, _p(maxd2), _p(argmax), H, W, _p(g), ctypes.c_void_p(flags.data_ptr() + 4 * F),
                                  _p(bg_u8), _p(bg_f32), st))
    if torch.cuda.is_current_stream_capturing():
        return                                      # no sync inside a capture: a replay of a rejected geometry writes zeros where undefined
    f = flags.cpu()                                 # the one host sync: the two geometries where the reference's NearestNeighbors.fit raises
    empty = [sel[i] for i in range(F) if int(f[i]) == 0]
    if empty:
        raise ValueError(f'extract_background: frame(s) {empty} have no foreground pixel (segmap channel 0 is nonzero everywhere)')
    if int(f[F]) == 0:
        raise ValueError('extract_background: no pixel lies farther than 10 from every selected frame\'s foreground, so there is no '
                         'background to extract')


# ---- public interface --------------------------------------------------------------------------------------------------------------------
@torch.no_grad()
def inpaint_torso(img: torch.Tensor, segmap: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """inpaint_torso_job(img, segmap)[0]: img uint8 [H,W,3] RGB, segmap [6,H,W] or [1,6,H,W] float32 / uint8 (CUDA) -> torso_img uint8
    [H,W,3].  out= a contiguous uint8 [H,W,3] buffer on the image's device, written in place."""
    img = _images(img, 'inpaint_torso: img', False)
    H, W = img.shape[0], img.shape[1]
    seg = _segmaps(segmap, 'inpaint_torso: segmap', ((), (1,)), H, W)
    dev = _on_device((img, seg), ('img', 'segmap'))
    img, seg = img.contiguous(), seg.contiguous()
    out = torch.empty(H, W, 3, dtype=torch.uint8, device=dev) if out is None else _out(out, (H, W, 3), torch.uint8, 'torso_img', dev)
    with capi.region('source.torso'):
        _torso(img, seg, torso_u8=out)
    return out


@torch.no_grad()
def extract_background(frames: torch.Tensor, segmaps: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """extract_background(frames, segmaps, 'knn'): frames uint8 [N,H,W,3] RGB, segmaps [N,6,H,W] float32 / uint8 (CUDA) -> the background,
    uint8 [H,W,3].  Only the frames the reference selects are read (interval 5 below 100 frames, 20 below 10 000, else N // 500; [::interval]
    when N exceeds the interval, else frame 0).  Raises ValueError, after one host sync, where the reference's NearestNeighbors.fit raises: a
    selected frame without a foreground (segmap[0] == 0) pixel, or no pixel farther than 10 from every selected frame's foreground.
    out= a contiguous uint8 [H,W,3] buffer, written in place."""
    frames = _images(frames, 'extract_background: frames', True)
    N, H, W = frames.shape[0], frames.shape[1], frames.shape[2]
    segs = _segmaps(segmaps, 'extract_background: segmaps', ((N,),), H, W)
    dev = _on_device((frames, segs), ('frames', 'segmaps'))
    frames, segs = frames.contiguous(), segs.contiguous()
    out = torch.empty(H, W, 3, dtype=torch.uint8, device=dev) if out is None else _out(out, (H, W, 3), torch.uint8, 'bg', dev)
    with capi.region('source.background'):
        _background(frames, segs, bg_u8=out)
    return out


@torch.no_grad()
def prepare_source(img: torch.Tensor, segmap: torch.Tensor, bg_img: Optional[torch.Tensor] = None,
                   out: Optional[Dict[str, torch.Tensor]] = None) -> Dict[str, torch.Tensor]:
    """The torso head's per-clip images from the source image: img uint8 [H,W,3] RGB (load_img_to_512_hwc_array's array), segmap [6,H,W] or
    [1,6,H,W] float32 / uint8 in _cal_seg_map's channel order (0 bg, 1 hair, 2 body skin, 3 face skin, 4 clothes, 5 others), on the GPU ->
    {'ref_head_img', 'ref_torso_img', 'bg_img'}, each float32 [1,3,H,W] in [-1, 1].

    bg_img= a [1,3,H,W] tensor (the caller's --bg_img, already normalised) skips the extraction.  out= a dict of contiguous float32
    [1,3,H,W] buffers with those keys, written in place, so a second clip refills the buffers FrameEngine.begin_clip / begin_planes were fed
    (and a captured graph reads).  The background extraction costs one host sync for its geometry check (skipped inside a CUDA-graph capture)."""
    img = _images(img, 'prepare_source: img', False)
    H, W = img.shape[0], img.shape[1]
    seg = _segmaps(segmap, 'prepare_source: segmap', ((), (1,)), H, W)
    if bg_img is not None and (not isinstance(bg_img, torch.Tensor) or tuple(bg_img.shape) != (1, 3, H, W)):
        raise ValueError(f'prepare_source: bg_img must be a tensor [1,3,{H},{W}], got {tuple(getattr(bg_img, "shape", ()))}')
    dev = _on_device((img, seg) + ((bg_img,) if bg_img is not None else ()), ('img', 'segmap', 'bg_img'))
    img, seg = img.contiguous(), seg.contiguous()
    if out is None:
        res = {k: torch.empty(1, 3, H, W, device=dev) for k in OUTPUTS if k != 'bg_img' or bg_img is None}
    else:
        if not isinstance(out, dict) or set(out) != set(OUTPUTS):
            raise ValueError(f'prepare_source: out must be a dict with the keys {list(OUTPUTS)}')
        res = {k: _out(out[k], (1, 3, H, W), torch.float32, k, dev) for k in OUTPUTS}
    with capi.region('source.prepare'):
        _torso(img, seg, head_f32=res['ref_head_img'], torso_f32=res['ref_torso_img'])
        if bg_img is None:
            _background(img.unsqueeze(0), seg.reshape(1, 6, H, W), bg_f32=res['bg_img'])
        elif out is None:
            res['bg_img'] = bg_img
        elif res['bg_img'].data_ptr() != bg_img.data_ptr():
            res['bg_img'].copy_(bg_img)
    return res
