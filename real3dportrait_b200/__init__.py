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
from .img2plane import Img2PlaneModel
from .secc_render import SECC_Renderer, blink_eye_for_secc, period_blink_schedule
from .audio2motion import PitchContourVAEModel, VAEModel
from .hubert import HubertModel, get_hubert_from_16k_speech, hubert_frames
from .motion import ClipMotion
from .fit3dmm import Fit3DMM
from .source import extract_background, inpaint_torso, prepare_source
from .debug_frames import concat_debug_frames

__all__ = ['RaySampler', 'ImportanceRenderer', 'PlanesCL', 'generate_planes', 'planes_to_channels_last',
           'sample_from_planes', 'sample_from_trigrids', 'grids_to_channels_last', 'producer_view', 'MipRayMarcher2', 'FullyConnectedLayer', 'OSGDecoder', 'SuperresolutionHybrid8XDC',
           'SynthesisBlock', 'SynthesisLayer', 'ToRGBLayer', 'SuperresolutionHybrid8XDC_Warp', 'SynthesisBlockNoUp', 'RenderHead',
           'SegFormerSECC2PlaneBackbone', 'canonical_planes_cl', 'Img2PlaneModel', 'SECC_Renderer',
           'blink_eye_for_secc', 'period_blink_schedule', 'PitchContourVAEModel', 'VAEModel',
           'HubertModel', 'get_hubert_from_16k_speech', 'hubert_frames', 'ClipMotion', 'Fit3DMM',
           'prepare_source', 'inpaint_torso', 'extract_background', 'concat_debug_frames']
