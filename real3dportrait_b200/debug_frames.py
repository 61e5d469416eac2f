"""The reference's default 'concat_debug' video frames (real3d_infer.py:494-521) on the GPU: every frame is a uint8 RGB strip
[512, 2560, 3] of five panels, source | driving SECC | image_raw (x8 nearest) | depth normalised over the whole clip (x8 nearest, grey) | image,
converted exactly as the reference's float64 torch.cat makes it (DESIGN.md, "Debug video").

`debug_panels` and `depth_panel` are the two entry points FrameEngine(out_mode='concat_debug') calls; `concat_debug_frames` runs both on a
whole clip, for callers that use RenderHead.synthesis directly."""
from __future__ import annotations

from typing import Optional

import torch

from . import _capi as capi

S, RES = 512, 64
FRAME_SHAPE = (S, 5 * S, 3)


def _strip_args(out: torch.Tensor, n: int, what: str):
    """Frame stride and row pitch (bytes) of a uint8 [n,512,2560,3] destination whose pixels are packed within a row."""
    if not out.is_cuda or out.dtype != torch.uint8 or out.ndim != 4 or tuple(out.shape[1:]) != FRAME_SHAPE or out.shape[0] != n:
        raise ValueError(f'{what}: out must be a CUDA uint8 [{n},{S},{5 * S},3] tensor, got {out.dtype} {tuple(out.shape)} on {out.device}')
    if out.stride(3) != 1 or out.stride(2) != 3 or out.stride(1) < 5 * S * 3 or (n > 1 and out.stride(0) < S * out.stride(1)):
        raise ValueError(f'{what}: out must hold each row as 2560 packed RGB pixels and the frames apart, got strides {out.stride()}')
    return out.stride(0), out.stride(1)


def _check(t: torch.Tensor, shape, what: str) -> torch.Tensor:
    if not t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous() or tuple(t.shape) != tuple(shape):
        raise ValueError(f'{what}: expected a contiguous CUDA float32 {list(shape)} tensor, got {t.dtype} {tuple(t.shape)} on {t.device}')
    return t


def debug_panels(ref_gt: torch.Tensor, secc: torch.Tensor, feat: torch.Tensor, image: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """Panels 0, 1, 2 and 4 of B frames into out uint8 [B,512,2560,3] (any frame stride and row pitch); panel 3 is left as it is.
    ref_gt [1,3,512,512], secc [B,3,512,512], feat [B,4096,C] (the render's channels-last features, rgb in channels 0-2), image [B,3,512,512]:
    contiguous CUDA float32.  One launch on the current stream, no sync."""
    B = image.shape[0]
    _check(ref_gt, (1, 3, S, S), 'debug_panels: ref_gt')
    _check(secc, (B, 3, S, S), 'debug_panels: secc')
    _check(image, (B, 3, S, S), 'debug_panels: image')
    if not feat.is_cuda or feat.dtype != torch.float32 or not feat.is_contiguous() or feat.ndim != 3 or tuple(feat.shape[:2]) != (B, RES * RES) \
            or feat.shape[2] < 3:
        raise ValueError(f'debug_panels: feat must be a contiguous CUDA float32 [{B},{RES * RES},C >= 3] tensor, got {feat.dtype} {tuple(feat.shape)}')
    fs, rp = _strip_args(out, B, 'debug_panels')
    capi.check(capi.lib().r3dp_debug_panels(capi.ptr(ref_gt), capi.ptr(secc), capi.ptr(feat), feat.shape[2], capi.ptr(image), B,
                                            capi.C.c_void_p(out.data_ptr()), fs, rp, capi.stream()))
    return out


def depth_panel(depth: torch.Tensor, out: torch.Tensor, scratch: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Panel 3 of F frames into out uint8 [F,512,2560,3]: depth [F,64,64] (or [F,4096], [F,1,64,64]) CUDA float32, normalised by its min
    and max over all F frames.  scratch: 2 int32 on the device (allocated here if None).  Two launches on the current stream, no sync."""
    F = depth.shape[0]
    if not depth.is_cuda or depth.dtype != torch.float32 or not depth.is_contiguous() or depth.numel() != F * RES * RES:
        raise ValueError(f'depth_panel: depth must be a contiguous CUDA float32 [F,64,64] tensor, got {depth.dtype} {tuple(depth.shape)}')
    fs, rp = _strip_args(out, F, 'depth_panel')
    if scratch is None:
        scratch = torch.empty(2, dtype=torch.int32, device=depth.device)
    capi.check(capi.lib().r3dp_debug_depth_panel(capi.ptr(depth), F, capi.ptr(scratch, torch.int32), capi.C.c_void_p(out.data_ptr()), fs, rp,
                                                 capi.stream()))
    return out


@torch.no_grad()
def concat_debug_frames(ref_gt_img: torch.Tensor, drv_secc: torch.Tensor, image_raw: torch.Tensor, image_depth: torch.Tensor,
                        image: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The whole clip's debug frames, as real3d_infer.py:494-521 builds them, in the shapes forward_secc2video holds them:
    ref_gt_img [1,3,512,512], drv_secc [N,3,512,512], image_raw [N,3,64,64], image_depth [N,1,64,64], image [N,3,512,512]
    (RenderHead.synthesis's 'image_raw', 'image_depth' and 'image') -> uint8 [N,512,2560,3] on their device (out=, if given, is filled)."""
    N = image.shape[0]
    dev = image.device
    if tuple(image_raw.shape) != (N, 3, RES, RES) or tuple(image_depth.shape) != (N, 1, RES, RES):
        raise ValueError(f'concat_debug_frames: image_raw must be [{N},3,64,64] and image_depth [{N},1,64,64], '
                         f'got {tuple(image_raw.shape)} and {tuple(image_depth.shape)}')
    if out is None:
        out = torch.empty((N,) + FRAME_SHAPE, dtype=torch.uint8, device=dev)
    feat = image_raw.detach().permute(0, 2, 3, 1).reshape(N, RES * RES, 3).float().contiguous()   # NCHW -> the render's channels-last layout
    debug_panels(capi.f32(ref_gt_img), capi.f32(drv_secc), feat, capi.f32(image), out)
    depth_panel(capi.f32(image_depth), out)
    return out
