"""Layer-level conformance of the tensor-core SR convolutions (csrc/sr_tc.cu) in both operand modes, through the C entry points:
`tc` (r3dp_sr_tc_*, fp16 operands) and `tcx` (r3dp_sr_tcx_*, split [hi | lo] operands, sr_mode='tc_exact').

* Every conv entry point against a float64 reference built from the operands the kernel reads, with the element-wise bound
  |got - ref| <= alpha |ref| + extra + beta S of tests/sr_conv_reference.py (its docstring derives alpha and extra; beta is measured).
  The case list covers, per entry point and mode: N = 1 and 3, shared and per-sample weights, odd H where the entry point allows it,
  W = 128 / 256 / 384 (384: an odd number of 128-pixel tiles, which turns the phase interleave of multi-phase launches off) and
  O = 128 / 256, plus one launch of more than 2 x 132 units, so that persistent CTAs run units of several images.
  PRODUCTION adds every launch of the benchmarked step at its exact shape (up to 4096 units, about 31 per CTA; W = 512, tiles_x = 4; the
  2048-item FIR pass) and the SECC->plane backbone's to_plane convs (SECC_PRODUCTION), PER_SAMPLE the Nw = N variants of block1's two
  layers; KC32 adds I = 3 / 16 / 32 (the 32-channel K chunks) to every single-phase family and I = 33.  Each launch is compared one image at a time, which bounds the float64 memory.
* test_benchmarked_launches_have_rows records every conv_tc3 call of one eager step of bench.py's engines and fails, naming the launch,
  when one has no row here, or when a PRODUCTION row is not launched.  (The torso warper's r3dp_tw_conv* launches have their own
  recorded-launch test, tests/test_gpu_torso_warper_launches.py.)
* Bit-exact properties: image k of an N = 3 per-sample launch equals the N = 1 launch of image k (and the last image of every N = 4
  launch its N = 1 launch); Nw = 1 equals Nw = N with the weights replicated; a launch repeated gives the same bits; nothing outside the
  logical output is written (canaries, the lo halves and the uint8 frames included) and every fp16 / fp32 element of it is.
* The input and packing kernels: weight packing exactly, the composed up weights against the float64 composition, and every input
  resize against float64 bilinear interpolation and bit for bit against each other."""
import math
import re

import pytest
import torch
import torch.nn.functional as F

from real3dportrait_b200 import _capi as capi
import sr_conv_reference as scr
from launch_harness import Recorder, assert_rows, bits, check_split_layout, given, guarded, guards_intact, split_cat, untouched

pytestmark = pytest.mark.gpu
DEV = 'cuda'
F16 = torch.float16
MODES = ['tc', 'tcx']
RGB_FAMILIES = ('layer_torgb', 'noup', 'last', 'torgb')


def _pad64(c):
    return (c + 63) // 64 * 64


def _store(v, split):
    """fp32 NHWC -> the kernel's activation tensor: fp16, or [hi | lo] with hi = fp16(v), lo = fp16(v - hi)."""
    return split_cat(v) if split else v.half().contiguous()


def _fn(name, split):
    return getattr(capi.lib(), ('r3dp_sr_tcx_' if split else 'r3dp_sr_tc_') + name)


def _pack(wf, split, composed=False):
    Nw, O, I = wf.shape[:3]
    out = torch.empty(Nw, 36 if composed else 9, O, _pad64(I) * (2 if split else 1), device=DEV, dtype=F16)
    capi.check(_fn('pack_weights_up_composed' if composed else 'pack_weights', split)(capi.ptr(wf.contiguous()), Nw, O, I, capi.ptr(out, F16),
                                                                                     capi.stream()))
    return out


# ---- operands, launches, outputs ---------------------------------------------------------------------------------------------------------
def _operands(fam, split, N, Nw, I, O, H, W, seed, skip=False, res=False, **opt):
    """Seeded operands of one launch.  x and the residual are N(0, 1); weights N(0, 1 / fan-in) so that activations stay O(1); the ToRGB
    bias is 1.5 N(0, 1) so that images leave [-1, 1]."""
    g = torch.Generator(device=DEV).manual_seed(seed)

    def rn(*s):
        return torch.randn(*s, generator=g, device=DEV)
    P = dict(fam=fam, split=split, N=N, Nw=Nw, I=I, O=O, H=H, W=W, ksize=3, act=1, clamp=0, u8=False, same_res=0,
             wp=None, bias=None, wrgb=None, brgb=None, img_prev=None, res=None)
    P.update(opt)
    Cp = I if fam == 'torgb' else _pad64(I)                    # torgb_ex reads exactly C channels per half
    xv = torch.zeros(N, H, W, Cp, device=DEV)
    xv[..., :I] = rn(N, H, W, I)
    P['x'] = _store(xv, split)
    if fam != 'torgb':
        Oc = 128 if fam == 'last' else O
        k = P['ksize']
        P['wp'] = _pack(rn(Nw, Oc, I, 3, 3) / math.sqrt(k * k * I), split, composed=fam == 'composed')
        P['bias'] = 0.5 * rn(Oc)
    if fam in RGB_FAMILIES:
        C = {'last': 128, 'torgb': I}.get(fam, O)
        P['wrgb'] = rn(Nw, 3, C) / math.sqrt(C)
        P['brgb'] = 1.5 * rn(3)
    if skip:
        same = fam == 'noup' or (fam == 'torgb' and P['same_res'])
        P['img_prev'] = rn(N, 3, H, W) if same else rn(N, 3, H // 2, W // 2)
    if res:
        P['res'] = _store(rn(N, H, W, O), split)
    return P


def _output_shapes(P):
    N, O, H, W, wide = P['N'], P['O'], P['H'], P['W'], 2 if P['split'] else 1
    fam, shapes = P['fam'], {}
    if fam in ('layer1', 'conv_res', 'layer_torgb', 'noup'):
        shapes['y'] = ((N, H, W, O * wide), F16)
    if fam in ('layer2', 'composed'):
        shapes['y'] = ((N, 2 * H, 2 * W, O * wide), F16)
    if fam == 'last' and P['u8']:
        shapes['u8'] = ((N, H, W, 3), torch.uint8)
    elif fam in RGB_FAMILIES:
        shapes['img'] = ((N, 3, H, W), torch.float32)
    return shapes


def _alloc(P, canary):
    outs, guards = {}, {}
    for name, (shape, dt) in _output_shapes(P).items():
        if not canary:
            outs[name] = torch.empty(shape, device=DEV, dtype=dt)
            continue
        buf, v = guarded(math.prod(shape), dt, device=DEV)
        outs[name], guards[name] = v.view(shape), buf
    return outs, guards


def _launch(P, out):
    L, split, fam = capi.lib(), P['split'], P['fam']
    N, Nw, I, O, H, W = P['N'], P['Nw'], P['I'], P['O'], P['H'], P['W']
    x, wp, bias = capi.ptr(P['x'], F16), capi.ptr(P['wp'], F16), capi.ptr(P['bias'])
    wrgb, brgb, prev = capi.ptr(P['wrgb']), capi.ptr(P['brgb']), capi.ptr(P['img_prev'])
    y, img, st = capi.ptr(out.get('y'), F16), capi.ptr(out.get('img')), capi.stream()
    if fam in ('layer1', 'layer2'):
        up = 1 if fam == 'layer1' else 2
        scratch = torch.empty(_fn('scratch_bytes', split)(N, O, H, W), device=DEV, dtype=torch.uint8) if up == 2 else None
        rc = _fn('layer', split)(x, wp, bias, N, Nw, I, O, H, W, up, y, capi.ptr(scratch, torch.uint8), st)
    elif fam == 'composed':
        rc = _fn('layer_up_composed', split)(x, wp, bias, N, Nw, I, O, H, W, y, st)
    elif fam in ('layer_torgb', 'noup'):
        rc = _fn('layer_torgb' if fam == 'layer_torgb' else 'layer_torgb_noup', split)(x, wp, bias, wrgb, brgb, prev, N, Nw, I, O, H, W, y, img, st)
    elif fam == 'last':
        fn = L.r3dp_sr_tcx_last_layer if split else L.r3dp_sr_tc_last_layer_ex
        rc = fn(x, wp, bias, wrgb, brgb, prev, N, Nw, I, H, W, img, capi.ptr(out.get('u8'), torch.uint8), int(P['clamp']), st)
    elif fam == 'conv_res':
        rc = _fn('conv_res', split)(x, wp, bias, N, Nw, I, O, H, W, P['ksize'], P['act'], capi.ptr(P['res'], F16), y, st)
    else:
        rc = _fn('torgb_ex', split)(x, wrgb, brgb, prev, P['same_res'], N, Nw, I, H, W, img, st)
    capi.check(rc)


def _run(P, canary=False):
    out, guards = _alloc(P, canary)
    _launch(P, out)
    torch.cuda.synchronize()
    for name, buf in guards.items():
        assert guards_intact(buf, out[name].numel()), f'{P["fam"]}: {name} written outside its bounds'
        if buf.dtype != torch.uint8:
            assert not bool(untouched(out[name]).any()), f'{P["fam"]}: elements of {name} left unwritten'
    return out


# ---- float64 reference of one launch -----------------------------------------------------------------------------------------------------
def _reference(P):
    """[(output name, ref, S, alpha, extra)] of one launch (see sr_conv_reference for the bound)."""
    fam, split, N, I = P['fam'], P['split'], P['N'], P['I']
    x = scr.activations(P['x'], I, split)
    a_store, terms = scr.alpha_store(split), []
    if fam == 'torgb':
        a, S = x, x.abs()
    else:
        w = scr.packed_weights(P['wp'], I, split)
        w = scr.per_sample(scr.taps_composed(w) if fam == 'composed' else scr.taps3x3(w), N)
        code, k, extra = P['act'], P['ksize'], scr.FLOOR_F16         # the store's subnormal floor
        gain = scr.act_gain(code)
        if fam == 'layer2':
            grid = scr.conv_transposed(x, w)
            v, s = scr.fir_up(grid), scr.fir_up(scr.conv_transposed(x.abs(), w.abs()))
            extra = extra + gain * (a_store * scr.fir_up(grid.abs()) + 4 * scr.FLOOR_F16)    # the grid is stored (fp16 or split) before the FIR
        elif fam == 'composed':
            v, s = scr.conv_up_composed(x, w), scr.conv_up_composed(x.abs(), w.abs())
        else:
            v, s = scr.conv_same(x, w, k), scr.conv_same(x.abs(), w.abs(), k)
        b = P['bias'].double()
        a = scr.bias_act(v, b, code)
        S = gain * (s + b.abs().view(1, -1, 1, 1))
        ref_y, S_y = a, S
        if P['res'] is not None:
            r = scr.nhwc(P['res'], split)
            ref_y, S_y = a + r, S + r.abs()
            if not split:
                extra = 2 * scr.FLOOR_F16 + scr.ALPHA_F16 * a.abs()  # fp16(fp16(act) + res): the inner rounding
        if fam != 'last':
            terms.append(('y', ref_y, S_y, a_store, extra))
    if fam in RGB_FAMILIES:
        wr, br = scr.per_sample(P['wrgb'].double(), N), P['brgb'].double().view(1, 3, 1, 1)
        img, S_img = scr.torgb(a, wr) + br, scr.torgb(S, wr.abs()) + br.abs()
        if P['img_prev'] is not None:
            ip = P['img_prev'].double()
            if fam == 'noup' or (fam == 'torgb' and P['same_res']):
                img, S_img = img + ip, S_img + ip.abs()
            else:
                img, S_img = img + scr.upsample2x(ip), S_img + scr.upsample2x(ip.abs())
        extra = None
        if P['clamp'] or P['u8']:                                   # clamp is 1-Lipschitz: the bound of the unclamped value holds
            extra, img = scr.ALPHA_F32 * img.abs(), img.clamp(-1, 1)
        terms.append(('img', img, S_img, 0.0 if extra is not None else scr.ALPHA_F32, extra))
    return terms


def _got(P, out, name):
    return scr.nhwc(out['y'], P['split']) if name == 'y' else out[name].double()


# fam, N, Nw, I, O, H, W, options.  Each row runs in both modes.
CASES = [
    ('layer1', 1, 1, 64, 128, 7, 384, {}),
    ('layer1', 3, 3, 96, 256, 96, 256, {}),                        # 288 units; I = 96 pads to 128
    ('layer1', 3, 1, 256, 128, 6, 128, {}),
    ('layer2', 1, 1, 32, 128, 7, 384, {}),                         # 3 x blocks: no phase interleave
    ('layer2', 2, 2, 96, 256, 33, 256, {}),                        # 272 units
    ('layer2', 3, 3, 256, 128, 4, 128, {}),
    ('layer2', 3, 1, 32, 256, 5, 256, {}),
    ('composed', 1, 1, 32, 256, 7, 384, {}),
    ('composed', 2, 2, 64, 128, 33, 256, {}),                      # 272 units; I = 64 = COMPOSE_MAX_CIN
    ('composed', 3, 1, 64, 256, 4, 128, {}),
    ('layer_torgb', 3, 3, 128, 256, 96, 256, {'skip': True}),      # 288 units, per-sample wrgb, ToRGB over two cout blocks
    ('layer_torgb', 1, 1, 64, 128, 6, 384, {'skip': True}),
    ('layer_torgb', 3, 1, 256, 128, 4, 128, {'skip': True}),       # shared wrgb
    ('last', 3, 3, 128, 128, 96, 256, {'skip': True}),             # 288 units, fp32 image
    ('last', 1, 1, 256, 128, 6, 384, {'clamp': 1}),                # clamped, no skip image
    ('last', 3, 1, 64, 128, 4, 128, {'u8': True, 'skip': True}),   # uint8 frames
    ('last', 1, 1, 128, 128, 2, 128, {'u8': True}),
    ('conv_res', 1, 1, 64, 128, 7, 128, {'act': 0}),
    ('conv_res', 3, 3, 128, 256, 96, 256, {'act': 1, 'res': True}),        # 288 units
    ('conv_res', 3, 1, 96, 128, 5, 384, {'ksize': 1, 'act': 2, 'res': True}),
    ('conv_res', 1, 1, 256, 256, 5, 128, {'act': 3, 'res': True}),
    ('conv_res', 2, 1, 768, 128, 3, 256, {'ksize': 1, 'act': 2}),          # the weight_fuse=False fuse conv: 12 chunks (36 split) in one tile
    ('conv_res', 3, 3, 64, 256, 7, 256, {'ksize': 1, 'act': 3}),
    ('noup', 1, 1, 64, 128, 7, 384, {'skip': True}),
    ('noup', 3, 3, 128, 256, 96, 256, {'skip': True}),             # 288 units
    ('noup', 3, 1, 96, 128, 5, 128, {}),                           # no skip image
    ('torgb', 3, 3, 256, 0, 8, 256, {'skip': True}),
    ('torgb', 1, 1, 128, 0, 6, 384, {'skip': True, 'same_res': 1}),
    ('torgb', 3, 1, 96, 0, 4, 128, {'same_res': 1}),
]
#: every conv_tc3 launch of the benchmarked step (bench.py at batch 4, static styles: one shared weight set), at its exact shape and options;
#: test_benchmarked_launches_have_rows keeps this list equal to what the step launches
PRODUCTION = [
    # SR, FrameEngine in 'tc' and 'tc_exact', and the torso head's block0 / block1
    ('composed', 4, 1, 32, 256, 128, 128, {}),                     # block0.conv0: 1024 units
    ('layer_torgb', 4, 1, 256, 256, 256, 256, {'skip': True}),     # block0.conv1 + torgb
    ('layer2', 4, 1, 256, 128, 256, 256, {}),                      # block1.conv0: transposed conv, 2048 FIR work items, 513-row edge column
    ('last', 4, 1, 128, 128, 512, 512, {'skip': True, 'clamp': 1}),   # block1.conv1 + torgb: tiles_x = 4, 4096 units (the engine's clamped frames)
    ('last', 4, 1, 128, 128, 512, 512, {'skip': True}),            # the same, unclamped (RenderHead.synthesis of the torso head)
    # torso head, fuse mode v2, per step at 256^2
    ('conv_res', 4, 1, 64, 256, 256, 256, {'ksize': 1, 'act': 0}),        # torso_encoder
    ('conv_res', 4, 1, 512, 256, 256, 256, {'act': 2}),                    # fuse_head_torso_convs[0]
    ('conv_res', 4, 1, 256, 256, 256, 256, {'act': 0}),                    # fuse_head_torso_convs[2], fuse_fg_bg_convs[4], bg_encoder[4]
    ('layer1', 4, 1, 256, 256, 256, 256, {}),                              # head_torso_block.conv0
    ('noup', 4, 1, 256, 256, 256, 256, {'skip': True}),                    # head_torso_block.conv1 + torgb
    ('conv_res', 4, 1, 512, 128, 256, 256, {'ksize': 1, 'act': 2}),        # fuse_fg_bg_convs[0] (64 couts padded to 128)
    ('conv_res', 4, 1, 128, 256, 256, 256, {'act': 2}),                    # fuse_fg_bg_convs[2], bg_encoder[2]
    ('conv_res', 4, 1, 64, 128, 256, 256, {'act': 2}),                     # bg_encoder[0] (uncached step)
    # torso head, per clip (begin_clip): bg_encoder on the reference background
    ('conv_res', 1, 1, 64, 128, 256, 256, {'act': 2}),
    ('conv_res', 1, 1, 128, 256, 256, 256, {'act': 2}),
    ('conv_res', 1, 1, 256, 256, 256, 256, {'act': 0}),
]
#: to_plane_cnn.0/2/4 of the SECC->plane backbone (3x3, 256 -> 256, nn.LeakyReLU(0.01)) at 512^2, forward at B = 4 and 1; the backbone does
#: not run in the benchmarked step, so test_backbone_launches_have_rows (tests/test_gpu_secc2plane_launches.py) keeps these launched
SECC_PRODUCTION = [
    ('conv_res', 4, 1, 256, 256, 128, 128, {'act': 2}),
    ('conv_res', 1, 1, 256, 256, 128, 128, {'act': 2}),
]
PRODUCTION += SECC_PRODUCTION
#: Img2PlaneModel's r3dp_sr_tc_conv launches at 512^2, forward at B = 4 and 1: LowResolutionViT's conv_after_upsample1 / 2 (ReLU, act 3)
#: and TriplanePredictorViT's second_conv, second_conv_after_cat and third_conv_after_cat (LeakyReLU(0.01), act 2); not in the benchmarked
#: step, so test_launches_have_rows (tests/test_gpu_img2plane_launches.py) keeps these launched
IMG2PLANE_PRODUCTION = [(fam, B, 1, I, O, h, h, opt) for B in (4, 1) for fam, I, O, h, opt in (
    ('conv_res', 256, 128, 128, {'act': 3}), ('conv_res', 128, 128, 256, {'act': 3}), ('conv_res', 256, 128, 256, {'act': 2}),
    ('conv_res', 128, 128, 256, {'act': 2}))]
PRODUCTION += IMG2PLANE_PRODUCTION
#: block1's two layers with per-sample weights: weight-tap addressing per image at tiles_x = 4 and in the 2048-item FIR pass
PER_SAMPLE = [
    ('layer2', 4, 4, 256, 128, 256, 256, {}),
    ('last', 4, 4, 128, 128, 512, 512, {'skip': True, 'clamp': 1}),
]
#: I <= 32 runs the 32-channel K chunks (a 16-slot weight-tap ring, 64-byte swizzle) on every single-phase family; I = 33 is the smallest
#: launch on 64-channel chunks with padding
KC32 = [
    ('layer1', 3, 3, 3, 128, 6, 128, {}),
    ('layer1', 1, 1, 16, 256, 7, 384, {}),
    ('layer1', 2, 1, 32, 256, 96, 256, {}),                        # 384 units
    ('conv_res', 3, 3, 32, 128, 5, 256, {'res': True}),
    ('conv_res', 1, 1, 3, 256, 7, 128, {'act': 3, 'res': True}),
    ('conv_res', 2, 1, 16, 128, 6, 384, {'ksize': 1, 'act': 2}),
    ('conv_res', 3, 3, 32, 256, 4, 128, {'ksize': 1, 'act': 0, 'res': True}),
    ('layer_torgb', 3, 3, 32, 256, 8, 256, {'skip': True}),
    ('layer_torgb', 1, 1, 3, 128, 6, 128, {'skip': True}),
    ('layer_torgb', 2, 1, 16, 128, 4, 384, {}),
    ('noup', 3, 1, 16, 256, 6, 256, {'skip': True}),
    ('noup', 1, 1, 32, 128, 7, 384, {}),
    ('noup', 2, 2, 3, 128, 5, 128, {'skip': True}),
    ('last', 3, 3, 32, 128, 8, 256, {'skip': True}),
    ('last', 1, 1, 16, 128, 6, 128, {'clamp': 1}),
    ('last', 3, 1, 3, 128, 4, 128, {'u8': True, 'skip': True}),
    ('last', 1, 1, 32, 128, 2, 384, {'u8': True}),
    ('layer1', 2, 2, 33, 128, 7, 256, {}),                         # 64-channel chunks, 31 of them padding
]
CASES += PRODUCTION + PER_SAMPLE + KC32


def _case_id(c):
    fam, N, Nw, I, O, H, W, opt = c
    return f'{fam}-N{N}w{Nw}-I{I}-O{O}-{H}x{W}' + ''.join(f'-{k}{int(v)}' for k, v in sorted(opt.items()))


def _check_images(P, out, mode, tag):
    """The bound on every output of a launch, one image at a time: the float64 reference of a whole N = 4 launch at 512^2 would take over
    10 GB at once."""
    for k in range(P['N']):
        one = {name: t[k:k + 1] for name, t in out.items()}
        for name, ref, S, alpha, extra in _reference(_slice(P, k)):
            scr.check_bound(_got(P, one, name), ref, S, alpha, scr.BETA[mode], extra, f'{tag} image {k} {name}')


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('case', CASES, ids=[_case_id(c) for c in CASES])
def test_conv_vs_float64(case, mode):
    fam, N, Nw, I, O, H, W, opt = case
    split = mode == 'tcx'
    P = _operands(fam, split, N, Nw, I, O, H, W, seed=1000 + CASES.index(case), **opt)
    tag = f'{mode} {_case_id(case)}'
    if P['u8']:
        P_f32 = dict(P, u8=False, clamp=1)                            # the same launch with a clamped fp32 image
        out = _run(P_f32)
        _check_images(P_f32, out, mode, tag)
        u8 = _run(P, canary=True)['u8']
        assert torch.equal(u8, scr.to_uint8(out['img'])), f'{tag}: uint8 frames differ from the conversion of the fp32 image'
        return
    out = _run(P, canary=True)
    _check_images(P, out, mode, tag)
    if split and 'y' in out:
        check_split_layout(out['y'])
    if case in PRODUCTION or case in PER_SAMPLE:                      # the last image is computed by the CTAs' last units
        k = N - 1
        _assert_same_bits(_run(_slice(P, k)), {name: t[k:k + 1] for name, t in out.items()}, f'{tag}: image {k} vs its N=1 launch')


# ---- bit-exact properties ----------------------------------------------------------------------------------------------------------------
#: per entry point: N = 3 per-sample launches of more than 132 units where the entry point is a persistent conv
BITS = {
    'layer1': (96, 256, 96, 256, {}),                               # I, O, H, W, options
    'layer2': (96, 128, 33, 256, {}),
    'composed': (32, 256, 33, 256, {}),
    'layer_torgb': (64, 256, 96, 256, {'skip': True}),
    'last': (128, 128, 96, 256, {'skip': True}),
    'conv_res': (64, 128, 96, 256, {'act': 2, 'res': True}),
    'noup': (64, 256, 96, 256, {'skip': True}),
    'torgb': (128, 0, 8, 256, {'skip': True}),
    'last-kc32': (32, 128, 96, 256, {'skip': True}),                # the 32-channel K chunks: 288 units, fp32 image and uint8 frames
}


def _slice(P, k):
    Q = dict(P, N=1, Nw=1)
    for key in ('x', 'img_prev', 'res'):
        if P[key] is not None:
            Q[key] = P[key][k:k + 1]
    for key in ('wp', 'wrgb'):
        if P[key] is not None:
            Q[key] = P[key][k:k + 1] if P['Nw'] > 1 else P[key]
    return Q


def _weights_of_set0(P, replicate):
    Q = dict(P, Nw=P['N'] if replicate else 1)
    for key in ('wp', 'wrgb'):
        if P[key] is not None:
            Q[key] = P[key][:1].expand(P['N'], *P[key].shape[1:]).contiguous() if replicate else P[key][:1]
    return Q


def _assert_same_bits(a, b, what):
    for name in a:
        assert torch.equal(bits(a[name]), bits(b[name])), f'{what}: {name} differs'


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('key', list(BITS))
def test_conv_bits_slicing_shared_determinism_canaries(key, mode):
    I, O, H, W, opt = BITS[key]
    split, fam = mode == 'tcx', key.split('-')[0]
    P = _operands(fam, split, 3, 3, I, O, H, W, seed=2000 + list(BITS).index(key), **opt)
    full = _run(P, canary=True)
    _assert_same_bits(full, _run(P, canary=True), f'{fam} {mode}: repeated launch')
    for k in range(3):
        one = _run(_slice(P, k))
        _assert_same_bits(one, {n: t[k:k + 1] for n, t in full.items()}, f'{fam} {mode}: image {k} of the N=3 launch vs its N=1 launch')
    _assert_same_bits(_run(_weights_of_set0(P, False), canary=True), _run(_weights_of_set0(P, True)), f'{fam} {mode}: Nw=1 vs replicated weights')
    if fam == 'last':
        Q = dict(P, u8=True)
        _assert_same_bits(_run(Q, canary=True), _run(Q, canary=True), f'{fam} {mode}: repeated uint8 launch')
    if split and 'y' in full:
        check_split_layout(full['y'])


# ---- the launches of the benchmarked step ------------------------------------------------------------------------------------------------
#: the C entry points that launch conv_tc3
CONV_ENTRY = re.compile(r'r3dp_sr_tcx?_(layer|layer_up_composed|layer_torgb|layer_torgb_noup|conv|conv_res|last_layer|last_layer_ex)$')


def _row_of_call(name, a):
    """The CASES row of one recorded launch."""
    op, opt = name.split('_', 3)[3], {}
    if op in ('layer', 'layer_up_composed'):
        fam = 'composed' if op == 'layer_up_composed' else ('layer1' if a[9] == 1 else 'layer2')
        N, Nw, I, O, H, W = a[3:9]
    elif op in ('layer_torgb', 'layer_torgb_noup'):
        fam = 'layer_torgb' if op == 'layer_torgb' else 'noup'
        N, Nw, I, O, H, W = a[6:12]
        opt['skip'] = given(a[5])
    elif op in ('conv', 'conv_res'):
        fam = 'conv_res'
        N, Nw, I, O, H, W, opt['ksize'], opt['act'] = a[3:11]
        opt['res'] = op == 'conv_res' and given(a[11])
    else:                                                             # last_layer(_ex): 128 couts, the image only
        fam, O = 'last', 128
        N, Nw, I, H, W = a[6:11]
        opt['skip'] = given(a[5])
        if op == 'last_layer_ex' or name.startswith('r3dp_sr_tcx_'):
            opt['u8'], opt['clamp'] = given(a[12]), a[13]
    return fam, N, Nw, I, O, H, W, {k: v for k, v in opt.items() if v != DEFAULT_OPT[k]}


#: the options of a CASES row that _operands() defaults
DEFAULT_OPT = {'ksize': 3, 'act': 1, 'skip': False, 'res': False, 'clamp': 0, 'u8': False, 'same_res': 0}


def row_signature(row):
    """What decides a launch: the row with every option at its default made explicit (a uint8 launch clamps)."""
    fam, N, Nw, I, O, H, W, opt = row
    o = dict(DEFAULT_OPT, **opt)
    return (fam, N, Nw, I, O, H, W, o['ksize'], o['act'], bool(o['skip']), bool(o['res']), int(bool(o['clamp'] or o['u8'])), bool(o['u8']),
            o['same_res'])


def test_benchmarked_launches_have_rows():
    """Every conv_tc3 launch of the benchmarked step has a float64 row of the same shape and options: bench.py's FrameEngine(batch=4) in 'tc'
    and in 'tc_exact', and its configs[4], the torso head (stub warper, fuse mode v2) through RenderHead.synthesis without the clip's
    constants and through the engine after begin_clip().  One eager step of each, recorded at the C entry points."""
    from real3dportrait_b200 import engine, synthetic as syn
    B = 4
    planes, cams = syn.make_planes(B, seed=80).to(DEV), syn.make_cameras(B, seed=81).to(DEV)
    u_c, u_f = (u.to(DEV) for u in syn.make_jitter(B, 64 * 64, 48, 48, seed=82))
    mlp = syn.make_decoder_params(seed=4)
    with Recorder(capi.lib(), CONV_ENTRY.match) as rec:
        for mode in ('tc', 'tc_exact'):
            eng = engine.FrameEngine(batch=B, sr_mode=mode, use_graph=False, hp={'num_samples_fine': 0})
            eng.load_params(mlp, syn.make_sr_params(seed=5))
            eng.step(planes, cams, u_c)
        eng = engine.FrameEngine(batch=B, sr_mode='tc', use_graph=False, hp=dict(syn.WARP_HPARAMS, num_samples_fine=48),
                                 torso_model=syn.StubTorsoModel())
        eng.load_params(mlp, syn.make_sr_warp_params(seed=6))
        inp = {k: v.to(DEV) for k, v in syn.make_warp_inputs(1, seed=7).items()}
        kp_d = (torch.rand(B, 68, 3, generator=torch.Generator().manual_seed(9)) * 2 - 1).to(DEV)
        cond = {'ref_torso_img': inp['ref_torso_rgb'].expand(B, -1, -1, -1).contiguous(),
                'bg_img': inp['ref_bg_rgb'].expand(B, -1, -1, -1).contiguous(), 'segmap': inp['segmap'].expand(B, -1, -1, -1).contiguous(),
                'kp_s': inp['kp_s'].expand(B, -1, -1).contiguous(), 'kp_d': kp_d}
        eng.head.synthesis(planes, cams, cond=cond, u_coarse=u_c, u_fine=u_f)
        eng.begin_clip(inp['ref_torso_rgb'], inp['ref_bg_rgb'], inp['segmap'], inp['kp_s'])
        eng.step(planes, cams, u_c, u_f, kp_d=kp_d)
        torch.cuda.synchronize()
    have = {row_signature(row) for row in CASES}
    launches = {}
    for name, args in rec.calls:
        row = _row_of_call(name, args)
        launches.setdefault(row_signature(row), (name, row))
    assert {row[0] for _, row in launches.values()} >= {'composed', 'layer_torgb', 'layer2', 'last', 'conv_res', 'layer1', 'noup'}
    missing = [f'{name}: {row} (in CASES)' for key, (name, row) in launches.items() if key not in have]
    stale = [f'PRODUCTION {row}' for row in PRODUCTION if row not in SECC_PRODUCTION and row not in IMG2PLANE_PRODUCTION
             and row_signature(row) not in launches]
    assert_rows(missing, stale, 'the benchmarked step')


# ---- packing kernels ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('I', [32, 96, 256, 768])
def test_pack_weights_exact(I, mode):
    """[Nw,O,I,3,3] fp32 -> [Nw,9,O,Ip]: fp16(w), or [hi | lo] with hi = fp16(1024 w), lo = fp16(1024 w - hi) (torch fp32); padding exactly 0."""
    split, Nw, O, Ip = mode == 'tcx', 2, 128, _pad64(I)
    wf = torch.randn(Nw, O, I, 3, 3, generator=torch.Generator(device=DEV).manual_seed(3000 + I), device=DEV)
    wp = _pack(wf, split)
    torch.cuda.synchronize()
    t = wf.reshape(Nw, O, I, 9).permute(0, 3, 1, 2)                 # [Nw,9,O,I]
    halves = [t.half()] if not split else [(1024 * t).half()]
    if split:
        halves.append((1024 * t - halves[0].float()).half())
    for h, want in enumerate(halves):
        got = wp[..., h * Ip:(h + 1) * Ip]
        assert torch.equal(bits(got[..., :I].contiguous()), bits(want.contiguous())), (mode, I, h)
        assert bool((bits(got[..., I:]) == 0).all()), (mode, I, h)


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('I', [32, 64])
def test_pack_weights_up_composed_vs_float64(I, mode):
    """Composed up weights against the float64 composition.  The kernel sums at most 4 products g_u g_v w (exact: g_u g_v = k / 16) with fp32
    fmas, <= 4 roundings of partial sums bounded by S = compose(|w|): 2^-22 S; asserted 2^-21 S plus the rounding of the store and its
    subnormal floor (2^-25, or 2^-35 for split weights stored x 2^10)."""
    split, Nw, O, Ip = mode == 'tcx', 2, 128, _pad64(I)
    wf = torch.randn(Nw, O, I, 3, 3, generator=torch.Generator(device=DEV).manual_seed(3100 + I), device=DEV)
    wpc = _pack(wf, split, composed=True)
    torch.cuda.synchronize()
    layout = lambda G: G.permute(0, 3, 4, 5, 1, 2).reshape(Nw, 36, O, I)      # [Nw,O,I,4,3,3] -> the packed [Nw,36,O,I]  # noqa: E731
    ref, S = layout(scr.compose_up_weights(wf.double())), layout(scr.compose_up_weights(wf.double().abs()))
    floor = scr.FLOOR_F16 / (scr.SPLIT_WEIGHT_SCALE if split else 1.0)
    scr.check_bound(scr.packed_weights(wpc, I, split), ref, S, scr.alpha_store(split), 2.0 ** -21, floor, tag=f'{mode} composed weights I={I}')
    for h in range(2 if split else 1):
        assert bool((bits(wpc[..., h * Ip + I:(h + 1) * Ip]) == 0).all())


# ---- input resizes -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('src', [64, 37, 128])
def test_input_resizes_vs_float64_and_each_other(src):
    """r3dp_sr_resize_bilinear, tc/tcx_input (NCHW source), tc/tcx_input_nhwc and input_nhwc_rgb (split 0/1) at src -> 128.
    fp32 result vs float64 F.interpolate(bilinear, align_corners=False): the source coordinates are exact for these sizes, the mix is 3
    roundings of partial sums bounded by S = interp(|x|): asserted 2^-21 S.  They share one helper, so every fp16 output is fp16 (or the
    split pair) of the fp32 resize bit for bit, rgb_out is its channels 0..2 bit for bit, and the padding channels are zero."""
    L, N, C, size = capi.lib(), 2, 40, 128
    Cp = _pad64(C)
    x = torch.randn(N, C, src, src, generator=torch.Generator(device=DEV).manual_seed(4000 + src), device=DEV)
    x_nhwc = x.permute(0, 2, 3, 1).contiguous()
    ref = F.interpolate(x.double(), size=(size, size), mode='bilinear', align_corners=False)
    S = F.interpolate(x.double().abs(), size=(size, size), mode='bilinear', align_corners=False)
    y32 = torch.empty(N, C, size, size, device=DEV)
    capi.check(L.r3dp_sr_resize_bilinear(capi.ptr(x), N, C, src, src, size, capi.ptr(y32), capi.stream()))
    outs = {}
    for split in (False, True):
        wide = 2 if split else 1
        for name in ('input', 'input_nhwc', 'input_nhwc_rgb'):
            y = torch.empty(N, size, size, Cp * wide, device=DEV, dtype=F16)
            if name == 'input':
                capi.check(_fn('input', split)(capi.ptr(x), N, C, src, src, size, capi.ptr(y, F16), capi.stream()))
            elif name == 'input_nhwc':
                capi.check(_fn('input_nhwc', split)(capi.ptr(x_nhwc), N, C, src, src, size, capi.ptr(y, F16), capi.stream()))
            else:
                rgb = torch.empty(N, 3, size, size, device=DEV)
                capi.check(L.r3dp_sr_tc_input_nhwc_rgb(capi.ptr(x_nhwc), N, C, src, src, size, capi.ptr(y, F16), capi.ptr(rgb), int(split), capi.stream()))
                outs[('rgb', split)] = rgb
            outs[(name, split)] = y
    torch.cuda.synchronize()
    scr.check_bound(y32, ref, S, 0.0, 2.0 ** -21, tag=f'resize_bilinear {src}->{size}')
    v = y32.permute(0, 2, 3, 1)
    hi = v.half()
    lo = (v - hi.float()).half()
    for (name, split), y in outs.items():
        if name == 'rgb':
            assert torch.equal(bits(y), bits(y32[:, :3].contiguous())), (name, split)
            continue
        halves = (hi, lo) if split else (hi,)
        for h, want in enumerate(halves):
            got = y[..., h * Cp:(h + 1) * Cp]
            assert torch.equal(bits(got[..., :C].contiguous()), bits(want.contiguous())), (name, split, h)
            assert bool((bits(got[..., C:]) == 0).all()), (name, split, h)
        scr.check_bound(scr.nhwc(y, split)[:, :C], ref, S, scr.alpha_store(split), 2.0 ** -21, scr.FLOOR_F16,
                        tag=f'{name} split={int(split)} {src}->{size}')
