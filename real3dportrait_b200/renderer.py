"""ImportanceRenderer — host mirror of modules/eg3ds/volumetric_rendering/renderer.py:30-297.

`forward` keeps the reference signature and return tuple; the whole body (box limits, stratified depths, tri-plane
gather, OSG decoder, ray march, importance resampling, merge) is ONE fused CUDA call (r3dp_render_ex).  Jitter uniforms
are drawn here with torch.rand in the reference's order and shapes ([N,M,S,1] then [N*M,S_imp]; renderer.py:226,281), so
`torch.manual_seed` reproduces runs exactly as it does for the reference; tests may instead pass them explicitly through
rendering_options['u_coarse'] / ['u_fine']."""
from __future__ import annotations

import copy
import ctypes as C
from typing import Optional, Union

import torch

from . import _capi as capi
from .decoder import OSGDecoder
from .ray_marcher import MipRayMarcher2


def generate_planes() -> torch.Tensor:
    """The three plane axis frames of the reference (renderer.py:30-47)."""
    return torch.tensor([[[1, 0, 0], [0, 1, 0], [0, 0, 1]],
                         [[1, 0, 0], [0, 0, 1], [0, 1, 0]],
                         [[0, 0, 1], [1, 0, 0], [0, 1, 0]]], dtype=torch.float32)


class PlanesCL:
    """Tri-planes in a channels-last gather layout (one texel's C features = one contiguous 128-byte line).

    layout 'phwc': data [N,3,H,W,C]  (what r3dp_planes_to_channels_last writes)
    layout 'hwpc': data [N,H,W,3,C]  = the plane producer's [N,3*C,H,W] conv output held in torch.channels_last memory
                   (modules/real3d/secc_img2plane.py:73-81 views exactly such a tensor as [B,3,C,H,W]): zero-copy, no repack at all.
    A set with N == 1 may be shared by every frame of a call (frame stride 0): the per-clip canonical planes."""

    def __init__(self, data: torch.Tensor, layout: str = 'phwc'):
        assert layout in ('phwc', 'hwpc', 'pdhwc'), layout
        assert data.is_cuda and data.dtype == torch.float32 and data.is_contiguous()
        assert data.ndim == (6 if layout == 'pdhwc' else 5), (layout, data.shape)
        self.data, self.layout = data, layout

    @property
    def depth(self) -> int:
        """Depth slices per plane: > 1 only for tri-grids ('pdhwc' = [N,3,D,H,W,C], `triplane_feature_type: trigrid | trigrid_v2`)."""
        return self.data.shape[2] if self.layout == 'pdhwc' else 1

    @property
    def dims(self):
        if self.layout == 'phwc':
            N, _, H, W, Cc = self.data.shape
        elif self.layout == 'pdhwc':
            N, _, _, H, W, Cc = self.data.shape
        else:
            N, H, W, _, Cc = self.data.shape
        return N, Cc, H, W

    def c_layout(self, n_frames: int) -> capi.PlaneLayout:
        N, Cc, H, W = self.dims
        if N != n_frames and N != 1:
            raise ValueError(f'plane set holds {N} frames, the call renders {n_frames}')
        D = self.depth
        frame = 0 if (N == 1 and n_frames > 1) else 3 * D * H * W * Cc
        if self.layout == 'phwc':
            return capi.PlaneLayout(frame, H * W * Cc, W * Cc, Cc, 1, 0)
        if self.layout == 'pdhwc':
            return capi.PlaneLayout(frame, D * H * W * Cc, W * Cc, Cc, D, H * W * Cc)
        return capi.PlaneLayout(frame, Cc, W * 3 * Cc, 3 * Cc, 1, 0)


def grids_to_channels_last(grids: torch.Tensor, depth: int) -> PlanesCL:
    """Tri-grids [N,3,C*D,H,W] (channel index c*D + d, as cal_plane leaves them: img2plane_baseline.py:131-136) -> PlanesCL 'pdhwc' [N,3,D,H,W,C]."""
    grids = capi.f32(grids)
    assert grids.ndim == 5 and grids.shape[1] == 3 and grids.shape[2] % depth == 0, (grids.shape, depth)
    N, _, CD, H, W = grids.shape
    Cc = CD // depth
    out = torch.empty(N, 3, depth, H, W, Cc, device=grids.device, dtype=torch.float32)
    with capi.region('repack'):
        capi.check(capi.lib().r3dp_grids_to_channels_last(capi.ptr(grids), N, Cc, depth, H, W, capi.ptr(out), capi.stream()))
    return PlanesCL(out, 'pdhwc')


def planes_to_channels_last(planes: torch.Tensor, out: Optional[torch.Tensor] = None) -> PlanesCL:
    """[N,3,C,H,W] (reference layout, secc_img2plane.py:105-110) -> PlanesCL ('phwc')."""
    planes = capi.f32(planes)
    assert planes.ndim == 5 and planes.shape[1] == 3, planes.shape
    N, _, Cc, H, W = planes.shape
    if out is None:
        out = torch.empty(N, 3, H, W, Cc, device=planes.device, dtype=torch.float32)
    with capi.region('repack'):
        capi.check(capi.lib().r3dp_planes_to_channels_last(capi.ptr(planes), N, Cc, H, W, capi.ptr(out), capi.stream()))
    return PlanesCL(out)


def producer_view(planes: torch.Tensor) -> Optional[PlanesCL]:
    """If `planes` [N,3,C,H,W] (or [N,3*C,H,W]) is a VIEW of a channels_last conv output - memory order [N,H,W,3,C] - wrap it without
    copying; otherwise None.  (`x.to(memory_format=torch.channels_last)` on the producer's last conv makes its output such a tensor.)"""
    t = planes.detach()
    if t.dtype != torch.float32 or not t.is_cuda:
        return None
    if t.ndim == 4 and t.shape[1] % 3 == 0:
        t = t.view(t.shape[0], 3, t.shape[1] // 3, t.shape[2], t.shape[3]) if t.is_contiguous(memory_format=torch.channels_last) else None
        if t is None:
            return None
    if t.ndim != 5 or t.shape[1] != 3:
        return None
    N, _, Cc, H, W = t.shape
    want = (H * W * 3 * Cc, Cc, 1, W * 3 * Cc, 3 * Cc)
    if any(s != w for s, w, n in zip(t.stride(), want, t.shape) if n > 1):      # the stride of a size-1 dim (N == 1 sets) is arbitrary
        return None
    if N == 1:
        t = t.as_strided(t.shape, want)
    return PlanesCL(t.permute(0, 3, 4, 1, 2), 'hwpc')          # [N,H,W,3,C], contiguous by construction


def _as_cl(planes: Union[torch.Tensor, PlanesCL], depth: int = 1) -> PlanesCL:
    if isinstance(planes, PlanesCL):
        return planes
    if depth > 1:
        return grids_to_channels_last(planes, depth)
    pv = producer_view(planes)
    return pv if pv is not None else planes_to_channels_last(planes)


def _plane_sets(planes, depth: int = 1):
    """planes | PlanesCL | (a, b) pair of either -> (first, second-or-None); a pair is sampled set by set and summed in-kernel
    (`cano_planes + secc_planes`, secc_img2plane.py:73-81, without materialising the sum)."""
    if isinstance(planes, (tuple, list)):
        assert len(planes) == 2, 'at most two plane sets'
        a, b = _as_cl(planes[0], depth), _as_cl(planes[1], depth)
        if a.layout != b.layout or a.dims[1:] != b.dims[1:] or a.depth != b.depth:
            raise ValueError('the two plane sets must share layout and shape')
        return a, b
    return _as_cl(planes, depth), None


def _as_phwc(planes) -> PlanesCL:
    """The stand-alone sampler / run_model kernels read the 'phwc' layout only."""
    pcl = _as_cl(planes)
    if pcl.layout != 'phwc':
        pcl = PlanesCL(pcl.data.permute(0, 3, 1, 2, 4).contiguous(), 'phwc')
    return pcl


def sample_from_planes(plane_axes, plane_features, coordinates, mode='bilinear', padding_mode='zeros', box_warp=None):
    """renderer.py:65-75: plane_features [N,3,C,H,W] (or PlanesCL), coordinates [N,P,3] -> [N,3,P,C]."""
    assert padding_mode == 'zeros' and mode == 'bilinear'
    if plane_axes is not None and not torch.equal(plane_axes.detach().cpu().float(), generate_planes()):
        raise NotImplementedError('only the reference plane axes (generate_planes()) are built')
    pcl = _as_phwc(plane_features)
    N, Cc, H, W = pcl.dims
    coords = capi.f32(coordinates)
    P = coords.shape[1]
    out = torch.empty(N, 3, P, Cc, device=coords.device, dtype=torch.float32)
    capi.check(capi.lib().r3dp_triplane_sample(capi.ptr(pcl.data), N, Cc, H, W, capi.ptr(coords), P, C.c_float(float(box_warp)),
                                               capi.ptr(out), capi.stream()))
    return out


def sample_from_trigrids(plane_axes, plane_features, coordinates, mode='bilinear', padding_mode='zeros', box_warp=None, triplane_depth=1):
    """renderer.py:78-89: plane_features [N,3,C*D,H,W] (or PlanesCL 'pdhwc'), coordinates [N,P,3] -> [N,3,P,C] (3-D grid_sample)."""
    assert padding_mode == 'zeros' and mode == 'bilinear'
    if plane_axes is not None and not torch.equal(plane_axes.detach().cpu().float(), generate_planes()):
        raise NotImplementedError('only the reference plane axes (generate_planes()) are built')
    if triplane_depth < 2:
        raise NotImplementedError('tri-grids need triplane_depth >= 2 (Real3D uses 3, egs/os_avatar/img2plane.yaml:66)')
    pcl = _as_cl(plane_features, triplane_depth)
    N, Cc, H, W = pcl.dims
    coords = capi.f32(coordinates)
    P = coords.shape[1]
    out = torch.empty(N, 3, P, Cc, device=coords.device, dtype=torch.float32)
    capi.check(capi.lib().r3dp_trigrid_sample(capi.ptr(pcl.data), N, Cc, pcl.depth, H, W, capi.ptr(coords), P, C.c_float(float(box_warp)),
                                              capi.ptr(out), capi.stream()))
    return out


class ImportanceRenderer(torch.nn.Module):
    def __init__(self, hp=None):
        super().__init__()
        if hp is None:
            hp = {'enable_rescale_plane_regulation': False, 'triplane_feature_type': 'triplane'}
        self.hparams = copy.copy(hp)
        self.ray_marcher = MipRayMarcher2()
        self.plane_axes = generate_planes()
        self.triplane_feature_type = self.hparams.get('triplane_feature_type', 'triplane')
        if self.triplane_feature_type not in ('triplane', 'trigrid', 'trigrid_v2'):
            raise NotImplementedError(f"triplane_feature_type={self.triplane_feature_type!r}: 'triplane', 'trigrid' and 'trigrid_v2' are built ('3dgrid' is not a Real3D config)")
        # tri-grids: depth slices per plane (renderer.py:181); 'triplane' ignores triplane_depth as the reference does
        self.grid_depth = int(self.hparams.get('triplane_depth', 1)) if self.triplane_feature_type != 'triplane' else 1
        if self.triplane_feature_type != 'triplane' and self.grid_depth < 2:
            raise NotImplementedError('tri-grids need triplane_depth >= 2')

    def forward(self, planes, decoder, ray_origins, ray_directions, rendering_options):
        """planes [N,3,C,H,W] | PlanesCL, decoder: OSGDecoder, rays [N,M,3] ->
        (rgb [N,M,C], depth [N,M,1], weights_sum [N,M,1], is_ray_valid [N,M,1] bool)   (renderer.py:118-167)."""
        opt = rendering_options
        if not (opt['ray_start'] == opt['ray_end'] == 'auto'):
            # the reference itself raises NameError on this branch (is_ray_valid undefined, renderer.py:121,167)
            raise NotImplementedError("only ray_start = ray_end = 'auto' is supported (as in every Real3D config)")
        if opt.get('disparity_space_sampling', False):
            raise NotImplementedError('disparity_space_sampling is not used by Real3D-Portrait (img2plane_baseline.py:109)')
        assert opt.get('clamp_mode', 'softplus') == 'softplus', 'MipRayMarcher only supports `clamp_mode`=`softplus`!'
        if opt.get('density_noise', 0) > 0 or (self.hparams.get('enable_rescale_plane_regulation', False) and self.training):
            raise NotImplementedError('training-time density noise / plane rescaling are outside the inference path')
        if not isinstance(decoder, OSGDecoder):
            raise TypeError('the fused renderer needs an OSGDecoder (its four parameter tensors are read by the kernel)')
        pcl, pcl2 = _plane_sets(planes, self.grid_depth)
        if pcl.depth != self.grid_depth:
            raise ValueError(f'planes hold {pcl.depth} depth slices, the renderer is configured for {self.grid_depth}')
        _, Cc, H, W = pcl.dims
        ray_o, ray_d = capi.f32(ray_origins), capi.f32(ray_directions)
        N, M = ray_o.shape[0], ray_o.shape[1]
        S, S_imp = int(opt['depth_resolution']), int(opt.get('depth_resolution_importance', 0) or 0)
        dev = ray_o.device
        u_c = opt.get('u_coarse')
        u_c = torch.rand(N, M, S, 1, device=dev) if u_c is None else capi.f32(u_c)
        u_f = None
        if S_imp > 0:
            u_f = opt.get('u_fine')
            u_f = torch.rand(N * M, S_imp, device=dev) if u_f is None else capi.f32(u_f)
        res = int(round(M ** 0.5))
        res = res if res * res == M else 0
        rgb = torch.empty(N, M, Cc, device=dev)
        depth = torch.empty(N, M, 1, device=dev)
        wsum = torch.empty(N, M, 1, device=dev)
        valid = torch.empty(N, M, 1, device=dev, dtype=torch.bool)
        L = capi.lib()
        ws_bytes = L.r3dp_render_workspace_bytes(N, M)
        ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
        m = decoder.mlp_struct()
        g = capi.RenderArgs()
        g.planes, g.layout = capi.ptr(pcl.data).value, pcl.c_layout(N)
        if pcl2 is not None:
            g.planes2, g.layout2 = capi.ptr(pcl2.data).value, pcl2.c_layout(N)
        g.N, g.C, g.H, g.W, g.M, g.res, g.S, g.S_imp = N, Cc, H, W, M, res, S, S_imp
        g.ray_o, g.ray_d, g.camera = capi.ptr(ray_o).value, capi.ptr(ray_d).value, None
        g.box_warp, g.white_back = float(opt['box_warp']), int(bool(opt.get('white_back', False)))
        g.u_coarse, g.u_fine, g.mlp = capi.ptr(u_c).value, capi.ptr(u_f).value, C.pointer(m)
        g.rgb, g.depth, g.weights_sum = capi.ptr(rgb).value, capi.ptr(depth).value, capi.ptr(wsum).value
        g.is_ray_valid, g.workspace, g.workspace_bytes = capi.ptr(valid, torch.bool).value, capi.ptr(ws, torch.uint8).value, ws_bytes
        with capi.region('render'):
            capi.check(L.r3dp_render_ex(C.byref(g), capi.stream()))
        return rgb, depth, wsum, valid

    def run_model(self, planes, decoder, sample_coordinates, sample_directions, options):
        """renderer.py:169-188: planes, coords [N,P,3] -> {'rgb': [N,P,C], 'sigma': [N,P,1]}."""
        if options.get('density_noise', 0) > 0:
            raise NotImplementedError('density_noise is a training-time option')
        pcl = _as_cl(planes, self.grid_depth) if self.grid_depth > 1 else _as_phwc(planes)
        N, Cc, H, W = pcl.dims
        coords = capi.f32(sample_coordinates)
        P = coords.shape[1]
        if isinstance(decoder, OSGDecoder):
            rgb = torch.empty(N, P, Cc, device=coords.device)
            sigma = torch.empty(N, P, 1, device=coords.device)
            m = decoder.mlp_struct()
            capi.check(capi.lib().r3dp_run_model_grid(capi.ptr(pcl.data), N, Cc, pcl.depth, H, W, capi.ptr(coords), P,
                                                      C.c_float(float(options['box_warp'])), C.byref(m), capi.ptr(rgb), capi.ptr(sigma),
                                                      capi.stream()))
            return {'rgb': rgb, 'sigma': sigma}
        if self.grid_depth > 1:
            return decoder(sample_from_trigrids(None, pcl, coords, box_warp=options['box_warp'], triplane_depth=self.grid_depth), coords)
        feats = sample_from_planes(None, pcl, coords, box_warp=options['box_warp'])
        return decoder(feats, coords)
