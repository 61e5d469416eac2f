"""Host side of r3dp_mf_conv3d (csrc/conv3d_tc.cu), the tensor-core convolution / GEMM shared by the torso motion estimator, the audio2secc
VAE, Img2PlaneModel and SegFormerSECC2PlaneBackbone: its packed weight format (pack_conv3d and the GEMM / 3x3 forms) and its launch.

Format: weights [nph][taps][cop][cin] fp16, the output channels padded with zero filters to a multiple of the kernel's cout tile (cop), the
input channels to the 32-channel K step; with split operands each row is [hi | lo] of w * 2^10, twice as wide.  Bias [cop] fp32."""
from __future__ import annotations

import ctypes
from typing import NamedTuple, Optional, Sequence, Union

import torch

from . import _capi as capi

F16 = torch.float16


def ceil32(n: int) -> int:
    """Channels rounded up to the kernel's 32-channel K step: every cin the kernel reads is a multiple of 32."""
    return (n + 31) // 32 * 32


def cout_pad(cout: int) -> int:
    """cop: cout rounded up to the kernel's cout tile (16, 32, 64 or 128)."""
    tile = 16 if cout <= 16 else 32 if cout <= 32 else 64 if cout <= 64 else 128
    return (cout + tile - 1) // tile * tile


class Packed(NamedTuple):
    w: torch.Tensor                  # fp16 rows of cin ([hi | lo]: 2 * cin) values: [nph, taps, cop, .]; pack_gemm [cop, .], pack_taps [9, cop, .]
    bias: torch.Tensor               # fp32 [cop]
    cout: int
    cop: int


def pack_conv3d(w: torch.Tensor, b: Optional[torch.Tensor], cin: int, split: bool, cin_map=None) -> Packed:
    """Folded float64 weights [nph,O,I,kd,kh,kw] and bias [O] (None: zero) -> Packed, on the weights' device.  cin: the channels the conv
    reads (a multiple of 32); cin_map: the physical input channel of each of the I logical channels."""
    nph, O, I = w.shape[:3]
    taps = w.shape[3] * w.shape[4] * w.shape[5]
    cop = cout_pad(O)
    idx = torch.as_tensor(list(range(I)) if cin_map is None else cin_map, dtype=torch.long, device=w.device)
    wt = torch.zeros(nph, taps, cop, cin, dtype=torch.float64, device=w.device)
    wt[:, :, :O].index_copy_(3, idx, w.permute(0, 3, 4, 5, 1, 2).reshape(nph, taps, O, I))
    if split:
        s = wt * 1024.0
        hi = s.half()
        packed = torch.cat([hi, (s - hi.double()).half()], dim=-1)
    else:
        packed = wt.half()
    bias = torch.zeros(cop, dtype=torch.float32, device=w.device)
    if b is not None:
        bias[:O] = b.float()
    return Packed(packed.contiguous(), bias, O, cop)


def pack_gemm(w: torch.Tensor, b: Optional[torch.Tensor], dev, split: bool = False) -> Packed:
    """GEMM weights [O, K] (float64) -> fp16 [cop, K] ([cop, 2K] = [hi | lo] when split) on dev: pack_conv3d on 1x1x1 taps."""
    pk = pack_conv3d(w.to(dev)[None, :, :, None, None, None], None if b is None else b.to(dev), w.shape[1], split)
    return pk._replace(w=pk.w.view(pk.cop, -1))


def pack_taps(w: torch.Tensor, b: Optional[torch.Tensor], dev, split: bool = False) -> Packed:
    """3x3 conv weights [O, I, 3, 3] (float64) -> fp16 [9, cop, I] ([9, cop, 2I] = [hi | lo] when split) on dev, tap ky*3 + kx: pack_conv3d
    on 1x3x3 taps."""
    pk = pack_conv3d(w.to(dev)[None, :, :, None], None if b is None else b.to(dev), w.shape[1], split)
    return pk._replace(w=pk.w[0])


Operand = Union[torch.Tensor, ctypes.c_void_p, None]


def _f16(t: Operand) -> ctypes.c_void_p:
    return t if isinstance(t, ctypes.c_void_p) else capi.ptr(t, F16)


def launch(pk: Packed, x: Operand, xs: int, xlo: int, cin: int, dims: Sequence[int], taps: Sequence[int], y: torch.Tensor, ys: int,
           yc0: int = 0, ylo: int = 0, relu: int = 0, up: int = 0, res: Operand = None, *, stream: ctypes.c_void_p) -> None:
    """y[..., yc0:yc0 + cout] = act(conv(x) + bias) (+ res) with pk's weights, on `stream` (capi.stream(), looked up once per forward).
    x: fp16 voxels of xs halves (lo half at xlo when split), channels [0, cin) read; a tensor or a pointer (a channel slice of a wider buffer).
    The operands are split when pk's rows hold 2 * cin values ([hi | lo]); they must hold cin or 2 * cin.
    dims (N, D, H, W): the input grid; taps (kd, kh, kw); up: the 4 nearest-up phases of pack_conv3d(compose_nearest_up3d(..)).
    y: a tensor of ys halves per voxel (lo at ylo); fp16, or fp32 for an fp32 store.  relu: 0 none, 1 ReLU, 2 exact GELU.
    res: fp16 in y's layout, added after the activation (a tensor or a pointer)."""
    row = pk.w.shape[-1]
    if row not in (cin, 2 * cin):
        raise ValueError(f'r3dp_mf_conv3d: weights packed for {row} input values per row, the launch reads cin = {cin}')
    out_f32 = y.dtype == torch.float32
    capi.check(capi.lib().r3dp_mf_conv3d(_f16(x), xs, xlo, cin, capi.ptr(pk.w, F16), capi.ptr(pk.bias), _f16(res), *dims, *taps, up, pk.cout,
                                         pk.cop, relu, capi.ptr(y, torch.float32 if out_f32 else F16), ys, yc0, ylo, int(out_f32),
                                         int(row == 2 * cin), stream))
