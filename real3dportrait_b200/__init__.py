"""real3dportrait_b200 — H100 (sm_90a) implementation of Real3D-Portrait's per-frame volumetric render +
super-resolution hot path behind the reference's own module interfaces.

Host side (this package) mirrors the reference classes; all arithmetic is in libr3dp_b200.so (csrc/, C ABI in
include/r3dp_b200.h).  See DESIGN.md / INTEGRATION.md."""
from .ray_sampler import RaySampler
from .renderer import (ImportanceRenderer, PlanesCL, generate_planes, grids_to_channels_last, planes_to_channels_last, producer_view, sample_from_planes,
                       sample_from_trigrids)
from .ray_marcher import MipRayMarcher2
from .decoder import FullyConnectedLayer, OSGDecoder
from .superresolution import SuperresolutionHybrid8XDC, SynthesisBlock, SynthesisLayer, ToRGBLayer
from .sr_with_ref import SuperresolutionHybrid8XDC_Warp, SynthesisBlockNoUp
from .synthesis import RenderHead
from .secc2plane import SegFormerSECC2PlaneBackbone, canonical_planes_cl

__all__ = ['RaySampler', 'ImportanceRenderer', 'PlanesCL', 'generate_planes', 'planes_to_channels_last',
           'sample_from_planes', 'sample_from_trigrids', 'grids_to_channels_last', 'producer_view', 'MipRayMarcher2', 'FullyConnectedLayer', 'OSGDecoder', 'SuperresolutionHybrid8XDC',
           'SynthesisBlock', 'SynthesisLayer', 'ToRGBLayer', 'SuperresolutionHybrid8XDC_Warp', 'SynthesisBlockNoUp', 'RenderHead',
           'SegFormerSECC2PlaneBackbone', 'canonical_planes_cl']
