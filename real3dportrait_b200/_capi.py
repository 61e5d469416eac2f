"""ctypes binding of include/r3dp_b200.h (libr3dp_b200.so).  This is the ONLY compute path of the package: there
is no PyTorch / CPU fallback, and `lib()` raises if the library is missing or the tensor is not on a CUDA device."""
from __future__ import annotations

import ctypes as C
import os
import re
from typing import Optional

import torch

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
#: R3DP_LIB overrides the library file (profiling builds, e.g. lib/libr3dp_b200_dbg.so); it is still this library or nothing
LIB_PATH = os.environ.get('R3DP_LIB') or os.path.join(PKG, 'lib', 'libr3dp_b200.so')
HEADER = os.path.join(ROOT, 'include', 'r3dp_b200.h')

_lib: Optional[C.CDLL] = None


class MlpStruct(C.Structure):
    _fields_ = [('w1', C.c_void_p), ('b1', C.c_void_p), ('w2', C.c_void_p), ('b2', C.c_void_p),
                ('in_features', C.c_int), ('hidden', C.c_int), ('out_dim', C.c_int)]


class PlaneLayout(C.Structure):
    _fields_ = [('frame_stride', C.c_longlong), ('plane_stride', C.c_int), ('row_stride', C.c_int), ('texel_stride', C.c_int),
                ('depth', C.c_int), ('slice_stride', C.c_int)]


class RenderArgs(C.Structure):
    """r3dp_render_args_t (include/r3dp_b200.h)."""
    _fields_ = [('planes', C.c_void_p), ('layout', PlaneLayout), ('planes2', C.c_void_p), ('layout2', PlaneLayout),
                ('N', C.c_int), ('C', C.c_int), ('H', C.c_int), ('W', C.c_int),
                ('ray_o', C.c_void_p), ('ray_d', C.c_void_p), ('camera', C.c_void_p), ('M', C.c_int), ('res', C.c_int),
                ('S', C.c_int), ('S_imp', C.c_int), ('box_warp', C.c_float), ('white_back', C.c_int),
                ('u_coarse', C.c_void_p), ('u_fine', C.c_void_p), ('mlp', C.POINTER(MlpStruct)),
                ('rgb', C.c_void_p), ('depth', C.c_void_p), ('weights_sum', C.c_void_p), ('is_ray_valid', C.c_void_p),
                ('workspace', C.c_void_p), ('workspace_bytes', C.c_size_t)]


_P, _I, _F, _Z = C.c_void_p, C.c_int, C.c_float, C.c_size_t
_M = C.POINTER(MlpStruct)
#: name -> (restype, argtypes): a typed copy of include/r3dp_b200.h so ctypes rejects mis-ordered / mis-typed calls
_SIGNATURES = {
    'r3dp_abi_version': (_I, []),
    'r3dp_last_error': (C.c_char_p, []),
    'r3dp_device_info': (_I, [C.POINTER(_I)] * 3),
    'r3dp_launch_count': (C.c_ulonglong, []),
    'r3dp_peer_copy': (_I, [_P, _I, _P, _I, _Z, _P]),
    'r3dp_gen_rays': (_I, [_P, _P, _I, _I, _P, _P, _P]),
    'r3dp_planes_to_channels_last': (_I, [_P, _I, _I, _I, _I, _P, _P]),
    'r3dp_grids_to_channels_last': (_I, [_P, _I, _I, _I, _I, _I, _P, _P]),
    'r3dp_trigrid_sample': (_I, [_P, _I, _I, _I, _I, _I, _P, _I, _F, _P, _P]),
    'r3dp_run_model_grid': (_I, [_P, _I, _I, _I, _I, _I, _P, _I, _F, _M, _P, _P, _P]),
    'r3dp_triplane_sample': (_I, [_P, _I, _I, _I, _I, _P, _I, _F, _P, _P]),
    'r3dp_run_model': (_I, [_P, _I, _I, _I, _I, _P, _I, _F, _M, _P, _P, _P]),
    'r3dp_decode': (_I, [_P, _I, _I, _I, _I, _M, _P, _P, _P]),
    'r3dp_render_workspace_bytes': (_Z, [_I, _I]),
    'r3dp_render_ex': (_I, [C.POINTER(RenderArgs), _P]),
    'r3dp_render_path': (_I, [C.POINTER(RenderArgs)]),
    'r3dp_ray_march': (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P]),
    'r3dp_sr_styles': (_I, [_P, _P, _P, _I, _I, _I, _F, _P, _P]),
    'r3dp_sr_fold_weights': (_I, [_P, _P, _I, _I, _I, _I, _I, _P, _P]),
    'r3dp_sr_resize_bilinear': (_I, [_P, _I, _I, _I, _I, _I, _P, _P]),
    'r3dp_sr_layer_scratch_bytes': (_Z, [_I, _I, _I, _I]),
    'r3dp_sr_layer_fp32': (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P]),
    'r3dp_sr_torgb_fp32': (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _P]),
    'r3dp_sr_tc_pack_weights': (_I, [_P, _I, _I, _I, _P, _P]),
    'r3dp_sr_tcx_pack_weights': (_I, [_P, _I, _I, _I, _P, _P]),
    'r3dp_sr_tcx_pack_weights_up_composed': (_I, [_P, _I, _I, _I, _P, _P]),
    'r3dp_sr_tcx_input': (_I, [_P, _I, _I, _I, _I, _I, _P, _P]),
    'r3dp_sr_tcx_input_nhwc': (_I, [_P, _I, _I, _I, _I, _I, _P, _P]),
    'r3dp_sr_tcx_scratch_bytes': (_Z, [_I, _I, _I, _I]),
    'r3dp_sr_tcx_layer': (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P]),
    'r3dp_sr_tcx_layer_up_composed': (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P]),
    'r3dp_sr_tcx_layer_torgb': (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P]),
    'r3dp_sr_tcx_last_layer': (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _I, _P]),
    'r3dp_sr_tc_input': (_I, [_P, _I, _I, _I, _I, _I, _P, _P]),
    'r3dp_sr_tc_scratch_bytes': (_Z, [_I, _I, _I, _I]),
    'r3dp_sr_tc_layer': (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P]),
    'r3dp_sr_tc_torgb': (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P]),
    'r3dp_sr_tc_pack_weights_up_composed': (_I, [_P, _I, _I, _I, _P, _P]),
    'r3dp_sr_tc_layer_up_composed': (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P]),
    'r3dp_sr_tc_layer_torgb': (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P]),
    'r3dp_sr_tc_input_nhwc': (_I, [_P, _I, _I, _I, _I, _I, _P, _P]),
    'r3dp_sr_tc_input_nhwc_rgb': (_I, [_P, _I, _I, _I, _I, _I, _P, _P, _I, _P]),
    'r3dp_sr_tc_conv': (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P, _P]),
    'r3dp_sr_tcx_conv': (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P, _P]),
    'r3dp_sr_tcx_conv_res': (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P]),
    'r3dp_sr_tcx_layer_torgb_noup': (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P]),
    'r3dp_sr_tcx_alpha_cat_ex': (_I, [_P, _I, _I, _P, _I, _I, _I, _P, _I, _I, _I, _P, _P]),
    'r3dp_sr_tcx_alpha_mix': (_I, [_P, _I, _P, _I, _P, _I, _I, _I, _I, _P, _P]),
    'r3dp_sr_tcx_torgb_ex': (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P]),
    'r3dp_sr_alpha_mix': (_I, [_P, _I, _P, _I, _P, _I, _I, _I, _I, _P, _P]),
    'r3dp_sr_alpha_gate': (_I, [_P, _I, _I, _P, _I, _I, _I, _P, _P]),
    'r3dp_sr_tc_conv_res': (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P]),
    'r3dp_sr_tc_torgb_ex': (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P]),
    'r3dp_sr_tc_layer_torgb_noup': (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P]),
    'r3dp_sr_alpha_cat': (_I, [_P, _I, _I, _P, _I, _I, _P, _I, _I, _I, _P, _P]),
    'r3dp_sr_alpha_cat_ex': (_I, [_P, _I, _I, _P, _I, _I, _I, _P, _I, _I, _I, _P, _P]),
    'r3dp_sr_cat3': (_I, [_P, _I, _I, _P, _I, _I, _P, _I, _I, _I, _I, _I, _I, _P, _P]),
    'r3dp_sr_tcx_cat3': (_I, [_P, _I, _I, _P, _I, _I, _P, _I, _I, _I, _I, _I, _I, _P, _P]),
    'r3dp_sr_blend': (_I, [_P, _P, _P, _I, _I, _I, _I, _P, _P]),
    'r3dp_sr_person_occlusion': (_I, [_P, _P, _F, _I, _I, _I, _P, _P]),
    'r3dp_sr_resize_aa_down2': (_I, [_P, _I, _I, _I, _I, _P, _P]),
    'r3dp_sr_warp_input': (_I, [_P, _P, _I, _I, _I, _I, _I, _P, _P, _P, _P, _I, _P]),
    'r3dp_sr_tc_prof': (_I, [_I]),
    'r3dp_sr_tc_debug_buffer': (_I, [_P]),
    'r3dp_sr_tc_prof_read': (_I, [C.POINTER(C.c_float), C.POINTER(_I)]),
    'r3dp_sr_tc_last_layer': (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P]),
    'r3dp_sr_tc_last_layer_ex': (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _I, _P]),
    'r3dp_tw_gather3d': (_I, [_P, _I, _P, _I, _I, _I, _I, _I, _P, _I, _P]),
    'r3dp_tw_conv': (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _F, _P, _P, _I, _P]),
    'r3dp_tw_conv_up_nearest': (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _F, _P, _I, _P]),
    'r3dp_tw_affine_relu': (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _P, _P]),
    'r3dp_tw_narrow_conv': (_I, [_P, _I, _I, _I, _P, _I, _I, _P, _I, _I, _P, _P, _I, _I, _I, _I, _I, _I, _I, _P, _P]),
    'r3dp_tw_hid_to_nchw': (_I, [_P, _I, _I, _I, _I, _I, _I, _P, _P]),
    'r3dp_mf_conv3d': (_I, [_P, _I, _I, _I, _P, _P, _P] + [_I] * 11 + [_P] + [_I] * 5 + [_P]),
    'r3dp_mf_input': (_I, [_P, _I, _P, _P] + [_I] * 6 + [_P, _I, _I, _I, _P]),
    'r3dp_mf_pool': (_I, [_P] + [_I] * 7 + [_P, _I, _I, _I, _P]),
    'r3dp_mf_head_input': (_I, [_P, _P, _I, _I, _I, _I, _P, _I, _I, _I, _P]),
    'r3dp_mf_head_bcast': (_I, [_P] + [_I] * 7 + [_P, _I, _I, _I, _I, _P]),
    'r3dp_mf_deform': (_I, [_P, _I, _P, _P] + [_I] * 5 + [_P, _P]),
    'r3dp_mf_occlusion': (_I, [_P] + [_I] * 8 + [_P, _P, _P, _P, _P]),
    'r3dp_sp_prenet': (_I, [_P, _I, _I, _I, _I, _P, _P, _P, _P]),
    'r3dp_sp_embed': (_I, [_P, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P]),
    'r3dp_sp_layernorm': (_I, [_P, _P, _I, _I, _P, _P, _F, _P, _P, _P, _I, _P]),
    'r3dp_sp_patches': (_I, [_P, _I, _I, _I, _I, _I, _I, _I, _P, _P]),
    'r3dp_sp_attention': (_I, [_P, _I, _P, _I, _I, _I, _I, _I, _F, _P, _I, _P]),
    'r3dp_sp_dwconv_gelu': (_I, [_P, _I, _I, _I, _I, _P, _P, _P, _P]),
    'r3dp_sp_head_fuse': (_I, [_P, _I, _P, _I, _P, _I, _P, _I, _I, _P, _P, _P]),
    'r3dp_sp_leaky': (_I, [_P, C.c_longlong, _F, _P]),
    'r3dp_sp_upsample2_flip': (_I, [_P, _I, _I, _I, _I, _P, _P, _P]),
}


def declared_symbols():
    """Names of every function include/r3dp_b200.h declares (used by the symbol-export test)."""
    txt = open(HEADER).read()
    txt = re.sub(r'/\*.*?\*/', '', txt, flags=re.S)
    return sorted(set(re.findall(r'\b(r3dp_[a-z0-9_]+)\s*\(', txt)))


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f'{LIB_PATH} is missing: build it with `python -m real3dportrait_b200.build` '
                '(nvcc, sm_90a).  real3dportrait_b200 has no CPU or PyTorch fallback.')
        L = C.CDLL(LIB_PATH)
        for name, (restype, argtypes) in _SIGNATURES.items():
            fn = getattr(L, name)          # AttributeError here = header and library out of sync
            fn.restype, fn.argtypes = restype, argtypes
        if L.r3dp_abi_version() != 3:
            raise RuntimeError('libr3dp_b200.so ABI version mismatch')
        _lib = L
    return _lib


def check(rc: int) -> None:
    if rc != 0:
        raise RuntimeError('libr3dp_b200: ' + lib().r3dp_last_error().decode())


def stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t: Optional[torch.Tensor], dtype=torch.float32) -> C.c_void_p:
    """Device pointer of a dense CUDA tensor (None -> NULL)."""
    if t is None:
        return C.c_void_p(0)
    if not t.is_cuda:
        raise RuntimeError('real3dportrait_b200 runs on CUDA tensors only (no CPU fallback); got a CPU tensor')
    if t.dtype != dtype:
        raise RuntimeError(f'expected {dtype}, got {t.dtype}')
    if not t.is_contiguous():
        raise RuntimeError('expected a contiguous tensor')
    return C.c_void_p(t.data_ptr())


def f32(t: torch.Tensor) -> torch.Tensor:
    """Borrow as dense fp32 (no copy when already so); detached — this path is inference-only."""
    t = t.detach()
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


def mlp_struct(w1, b1, w2, b2) -> MlpStruct:
    return MlpStruct(ptr(w1).value, ptr(b1).value, ptr(w2).value, ptr(b2).value, w1.shape[1], w1.shape[0], w2.shape[0] - 1)


# ---- optional stage profiler (bench.py): CUDA events on the launching stream around named regions -----------------------
class Profiler:
    def __init__(self):
        self.events = []          # (name, start_event, end_event)

    def totals(self):
        torch.cuda.synchronize()
        out = {}
        for name, a, b in self.events:
            out[name] = out.get(name, 0.0) + a.elapsed_time(b)
        return out


PROF: Optional[Profiler] = None


class region:
    """`with region('sr_conv'):` — no-op unless a Profiler is installed in `_capi.PROF`."""
    __slots__ = ('name', 'a')

    def __init__(self, name):
        self.name = name

    def __enter__(self):
        if PROF is not None:
            self.a = torch.cuda.Event(enable_timing=True)
            self.a.record()
        return self

    def __exit__(self, *exc):
        if PROF is not None:
            b = torch.cuda.Event(enable_timing=True)
            b.record()
            PROF.events.append((self.name, self.a, b))
        return False
