"""Conformance of the torso head's fusion, gating and resampling kernels (csrc/sr_tc.cu) through their C entry points, in both operand
modes where both exist: `tc` (fp16 operands) and `tcx` (split [hi | lo] operands, sr_mode='tc_exact').

* Each entry point against the float64 reference of tests/torso_fusion_reference.py with its derived bound, at the production shape
  (N = 1 and 3, 256 x 256, C = 256), at small ragged shapes whose last block of 256 threads is partial and at odd H and W.  Operands are
  channel slices of wider tensors (pixel stride > wide * C, the lo half at half the stride), the last operand is one frame shared by an
  N = 3 batch, alpha takes the values 0 and 1 exactly, logits saturate the sigmoid (+-20, +-88, +-65504) under caps above and below it,
  head alphas sit at fp32(thr) and one ulp either side, and torso + head leaves [0, 1].
* Every output lies inside a NaN canary: nothing outside it is written, every element of it is, and the operands are left untouched
  (their padding channels included).
* Bit-exact properties: frame k of an N = 3 launch equals the N = 1 launch of frame k, and a repeated launch gives the same bits.
* The v3 head-mask chain (sr_with_ref.py:129-143): the head's split-operand alpha predictor, the gate, the quantile threshold and the
  person mask, against a float64 head_torso_alpha_predictor on the same weights."""
import math

import pytest
import torch
import torch.nn.functional as F

import real3dportrait_b200 as r3
import sr_conv_reference as scr
import torso_fusion_reference as tfr
from real3dportrait_b200 import _capi as capi, sr_tc, synthetic as syn
from launch_harness import bits, check_split_layout, guarded, guards_intact, untouched

pytestmark = pytest.mark.gpu
DEV = 'cuda'
F16 = torch.float16
MODES = ['tc', 'tcx']


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _pad64(c):
    return (c + 63) // 64 * 64


# ---- canaries ------------------------------------------------------------------------------------------------------------------------------
def _run(launch, shapes, inputs=(), canary=True):
    """Allocate the outputs named in shapes {name: (shape, dtype)} (inside sentinel-filled guards when canary), launch(out), and check that
    nothing outside an output is written, every element of one is, and no input tensor changed."""
    outs, guards = {}, {}
    for name, (shape, dt) in shapes.items():
        if not canary:
            outs[name] = torch.empty(shape, device=DEV, dtype=dt)
            continue
        buf, v = guarded(math.prod(shape), dt, device=DEV)
        outs[name], guards[name] = v.view(shape), buf
    before = [t.clone() for t in inputs]
    launch(outs)
    torch.cuda.synchronize()
    for name, buf in guards.items():
        assert guards_intact(buf, outs[name].numel()), f'{name} written outside its bounds'
        assert not bool(untouched(outs[name]).any()), f'elements of {name} left unwritten'
    for t, t0 in zip(inputs, before):
        assert torch.equal(bits(t), bits(t0)), 'an operand was written'
    return outs


# ---- operands ------------------------------------------------------------------------------------------------------------------------------
def _operand(N, H, W, C, split, stride, seed, scale=1.0):
    """A channel slice of a wider NHWC fp16 tensor [N,H,W,stride]: channels 0..C-1 hold fp16(v) (the hi halves), and when split the lo halves
    sit at stride / 2.  Every other channel holds large junk, so a read at a wrong offset shows.  Returns (buffer, float64 value read)."""
    g = _gen(seed)
    buf = (1000 * torch.randn(N, H, W, stride, generator=g, device=DEV)).half()
    v = scale * torch.randn(N, H, W, C, generator=g, device=DEV)
    hi = v.half()
    buf[..., :C] = hi
    val = hi.double()
    if split:
        lo = (v - hi.float()).half()
        buf[..., stride // 2:stride // 2 + C] = lo
        val = val + lo.double()
    return buf, val


def _alpha(N, H, W, seed, shape=None):
    """Seeded alpha in [0, 1] with exact 0 and 1 at the first pixels."""
    a = torch.rand(N, H, W, generator=_gen(seed), device=DEV)
    flat = a.view(-1)
    flat[:2] = torch.tensor([0.0, 1.0], device=DEV)
    flat[-1] = 1.0
    return a.view(shape) if shape else a


def _stride(C, split, extra):
    """Pixel stride of an operand: wide * C plus `extra` channels per half (lo at half the stride)."""
    return (2 if split else 1) * (C + extra)


# ---- entry points: make(mode, case, seed) -> P, run(P, canary) -> outputs, check(P, outputs) -> worst ratio; P['frame_keys'] are per frame --
def _frame(P, k):
    Q = dict(P, N=1)
    for key in P['frame_keys']:
        Q[key] = P[key][k:k + 1]
    return Q


def _make_alpha_cat(mode, case, seed):
    N, H, W, Ca, Cb, extra, shared = case
    split = mode == 'tcx'
    xa, va = _operand(N, H, W, Ca, split, _stride(Ca, split, extra), seed)
    xb, vb = _operand(1 if shared else N, H, W, Cb, split, _stride(Cb, split, 2 * extra), seed + 1)
    return dict(entry='alpha_cat', mode=mode, N=N, H=H, W=W, Ca=Ca, Cb=Cb, shared=shared, xa=xa, va=va, xb=xb, vb=vb, al=_alpha(N, H, W, seed + 2),
                frame_keys=['xa', 'va', 'al'] + ([] if shared else ['xb', 'vb']))


def _launch_alpha_cat(P, out, fn=None):
    L = capi.lib()
    fn = fn or (L.r3dp_sr_tcx_alpha_cat_ex if P['mode'] == 'tcx' else L.r3dp_sr_alpha_cat_ex)
    capi.check(fn(capi.ptr(P['xa'], F16), P['Ca'], P['xa'].shape[-1], capi.ptr(P['xb'], F16), P['Cb'], P['xb'].shape[-1],
                  int(P['shared'] and P['N'] > 1), capi.ptr(P['al']), P['N'], P['H'], P['W'], capi.ptr(out['y'], F16), capi.stream()))


def _run_alpha_cat(P, canary=True):
    wide = 2 if P['mode'] == 'tcx' else 1
    return _run(lambda o: _launch_alpha_cat(P, o), {'y': ((P['N'], P['H'], P['W'], wide * (P['Ca'] + P['Cb'])), F16)}, (P['xa'], P['xb'], P['al']), canary)


def _check_alpha_cat(P, out):
    split, tag = P['mode'] == 'tcx', f"alpha_cat {P['mode']}"
    ref = tfr.alpha_cat(P['va'], P['vb'], P['al'])
    got = tfr.join(out['y']) if split else out['y']
    r = scr.check_bound(got, ref, ref.abs(), tfr.ALPHA_CAT[P['mode']], 0.0, tfr.FLOOR_F16, tag)
    if split:
        check_split_layout(out['y'])
        return r
    a = P['al'][..., None]                                                   # the torch fp32 restatement: (x.float() * m).half(), bit for bit
    want = torch.cat([(P['va'].float() * a).half(), (P['vb'].float().expand(P['N'], -1, -1, -1) * (1 - a)).half()], dim=-1)
    assert torch.equal(bits(out['y']), bits(want)), f'{tag}: differs from (x.float() * m).half()'
    if not P['shared']:                                                      # r3dp_sr_alpha_cat = alpha_cat_ex without a shared operand
        o2 = _run(lambda o: capi.check(capi.lib().r3dp_sr_alpha_cat(
            capi.ptr(P['xa'], F16), P['Ca'], P['xa'].shape[-1], capi.ptr(P['xb'], F16), P['Cb'], P['xb'].shape[-1], capi.ptr(P['al']), P['N'], P['H'],
            P['W'], capi.ptr(o['y'], F16), capi.stream())), {'y': (tuple(out['y'].shape), F16)})
        assert torch.equal(bits(o2['y']), bits(out['y'])), f'{tag}: r3dp_sr_alpha_cat differs from r3dp_sr_alpha_cat_ex'
    return r


def _make_cat3(mode, case, seed):
    N, H, W, Ca, Cb, extra, shared = case
    split = mode == 'tcx'
    Cc = Ca + Cb                                                             # three different widths
    xa, _ = _operand(N, H, W, Ca, split, _stride(Ca, split, extra), seed)
    xb, _ = _operand(N, H, W, Cb, split, _stride(Cb, split, 2 * extra), seed + 1)
    xc, _ = _operand(1 if shared else N, H, W, Cc, split, _stride(Cc, split, extra), seed + 2)
    return dict(entry='cat3', mode=mode, N=N, H=H, W=W, Ca=Ca, Cb=Cb, Cc=Cc, shared=shared, xa=xa, xb=xb, xc=xc,
                frame_keys=['xa', 'xb'] + ([] if shared else ['xc']))


def _run_cat3(P, canary=True):
    L, wide = capi.lib(), 2 if P['mode'] == 'tcx' else 1
    fn = L.r3dp_sr_tcx_cat3 if P['mode'] == 'tcx' else L.r3dp_sr_cat3

    def launch(o):
        capi.check(fn(capi.ptr(P['xa'], F16), P['Ca'], P['xa'].shape[-1], capi.ptr(P['xb'], F16), P['Cb'], P['xb'].shape[-1], capi.ptr(P['xc'], F16),
                      P['Cc'], P['xc'].shape[-1], int(P['shared'] and P['N'] > 1), P['N'], P['H'], P['W'], capi.ptr(o['y'], F16), capi.stream()))
    return _run(launch, {'y': ((P['N'], P['H'], P['W'], wide * (P['Ca'] + P['Cb'] + P['Cc'])), F16)}, (P['xa'], P['xb'], P['xc']), canary)


def _check_cat3(P, out):
    """A copy: each half of the output is the concatenation of the operands' halves, bit for bit."""
    halves = 2 if P['mode'] == 'tcx' else 1
    for h in range(halves):
        parts = [P[k][..., h * P[k].shape[-1] // 2:][..., :P['C' + k[1]]] if halves == 2 else P[k][..., :P['C' + k[1]]] for k in ('xa', 'xb', 'xc')]
        want = tfr.cat3(*parts)
        Ct = want.shape[-1]
        assert torch.equal(bits(out['y'][..., h * Ct:(h + 1) * Ct]), bits(want.contiguous())), f"cat3 {P['mode']}: half {h} differs from torch.cat"
    return 0.0


def _make_alpha_mix(mode, case, seed):
    N, H, W, C, _, extra, _ = case
    split = mode == 'tcx'
    xa, va = _operand(N, H, W, C, split, _stride(C, split, extra), seed)
    xb, vb = _operand(N, H, W, C, split, _stride(C, split, 2 * extra), seed + 1)
    return dict(entry='alpha_mix', mode=mode, N=N, H=H, W=W, C=C, xa=xa, va=va, xb=xb, vb=vb, al=_alpha(N, H, W, seed + 2),
                frame_keys=['xa', 'va', 'xb', 'vb', 'al'])


def _run_alpha_mix(P, canary=True):
    L, wide = capi.lib(), 2 if P['mode'] == 'tcx' else 1
    fn = L.r3dp_sr_tcx_alpha_mix if P['mode'] == 'tcx' else L.r3dp_sr_alpha_mix

    def launch(o):
        capi.check(fn(capi.ptr(P['xa'], F16), P['xa'].shape[-1], capi.ptr(P['xb'], F16), P['xb'].shape[-1], capi.ptr(P['al']), P['C'], P['N'], P['H'],
                      P['W'], capi.ptr(o['y'], F16), capi.stream()))
    return _run(launch, {'y': ((P['N'], P['H'], P['W'], wide * P['C']), F16)}, (P['xa'], P['xb'], P['al']), canary)


def _check_alpha_mix(P, out):
    split = P['mode'] == 'tcx'
    ref, S = tfr.alpha_mix(P['va'], P['vb'], P['al'])
    r = scr.check_bound(tfr.join(out['y']) if split else out['y'], ref, S, tfr.ALPHA_MIX[P['mode']], tfr.BETA_MIX[P['mode']], tfr.FLOOR_F16,
                        f"alpha_mix {P['mode']}")
    if split:
        check_split_layout(out['y'])
    return r


GATE_EDGES = (20.0, -20.0, 88.0, -88.0, 65504.0, -65504.0, 0.0)


def _make_alpha_gate(mode, case, seed):
    """mode 'tc': lo_off = 0 (the logit is channel 0); 'tcx': the logit is hi + lo, lo at lo_off = stride / 2 (the split conv output)."""
    N, H, W, _, _, extra, _ = case
    split = mode == 'tcx'
    stride = 2 * (8 + extra)
    buf, v = _operand(N, H, W, 1, split, stride, seed, scale=4.0)
    lo_off = stride // 2 if split else 0
    flat, vf = buf.view(-1, stride), v.view(-1)
    n_e = min(len(GATE_EDGES), flat.shape[0])
    e = torch.tensor(GATE_EDGES[:n_e], device=DEV)
    flat[:n_e, 0] = e.half()
    if split:
        flat[:n_e, lo_off] = 0
    vf[:n_e] = e.double()
    cap = torch.rand(N, 1, H, W, generator=_gen(seed + 1), device=DEV)
    cap.view(-1)[::2] = 1.0                                                  # caps above (1) and below the sigmoid
    return dict(entry='alpha_gate', mode=mode, N=N, H=H, W=W, buf=buf, v=v, lo_off=lo_off, cap=cap, frame_keys=['buf', 'v', 'cap'])


def _run_alpha_gate(P, canary=True):
    def launch(o):
        capi.check(capi.lib().r3dp_sr_alpha_gate(capi.ptr(P['buf'], F16), P['buf'].shape[-1], P['lo_off'], capi.ptr(P['cap']), P['N'], P['H'], P['W'],
                                                 capi.ptr(o['a']), capi.stream()))
    return _run(launch, {'a': ((P['N'], 1, P['H'], P['W']), torch.float32)}, (P['buf'], P['cap']), canary)


def _check_alpha_gate(P, out):
    ref, S, extra = tfr.alpha_gate(P['v'].permute(0, 3, 1, 2), P['cap'], P['lo_off'] > 0)
    return scr.check_bound(out['a'], ref, S, 0.0, tfr.BETA_GATE, extra, f"alpha_gate lo_off={P['lo_off']}")


def _make_person(mode, case, seed):
    """mode selects the threshold: 'tc' 0.9 (fp32(0.9) < 0.9), 'tcx' 0.3 (fp32(0.3) > 0.3).  The first pixels hold fp32(thr) and one ulp
    either side, and 0 and 1; torso occlusion in [-0.5, 1.5], so that torso + head leaves [0, 1] on both sides."""
    N, H, W = case[:3]
    thr = 0.9 if mode == 'tc' else 0.3
    t = torch.tensor(thr, dtype=torch.float32, device=DEV)
    al = _alpha(N, H, W, seed, (N, 1, H, W))
    edges = torch.stack([torch.nextafter(t, torch.zeros_like(t)), t, torch.nextafter(t, torch.ones_like(t)), torch.zeros_like(t), torch.ones_like(t)])
    al.view(-1)[:min(5, al.numel())] = edges[:min(5, al.numel())]
    torso = 2 * torch.rand(N, 1, H, W, generator=_gen(seed + 1), device=DEV) - 0.5
    return dict(entry='person', mode=mode, N=N, H=H, W=W, thr=thr, al=al, torso=torso, frame_keys=['al', 'torso'])


def _run_person(P, canary=True):
    def launch(o):
        capi.check(capi.lib().r3dp_sr_person_occlusion(capi.ptr(P['al']), capi.ptr(P['torso']), P['thr'], P['N'], P['H'], P['W'], capi.ptr(o['p']),
                                                       capi.stream()))
    return _run(launch, {'p': ((P['N'], 1, P['H'], P['W']), torch.float32)}, (P['al'], P['torso']), canary)


def _check_person(P, out):
    want = tfr.person_occlusion_f32(P['al'], P['torso'], P['thr'])
    assert torch.equal(bits(out['p']), bits(want)), f"person_occlusion thr={P['thr']}: differs from the torch fp32 restatement"
    return 0.0


def _make_blend(mode, case, seed):
    N, H, W, C = case[:4]
    C = 3 if C >= 256 else C
    g = _gen(seed)
    return dict(entry='blend', mode=mode, N=N, H=H, W=W, C=C, a=torch.randn(N, C, H, W, generator=g, device=DEV),
                b=torch.randn(N, C, H, W, generator=g, device=DEV), al=_alpha(N, H, W, seed + 1, (N, 1, H, W)), frame_keys=['a', 'b', 'al'])


def _run_blend(P, canary=True):
    def launch(o):
        capi.check(capi.lib().r3dp_sr_blend(capi.ptr(P['a']), capi.ptr(P['b']), capi.ptr(P['al']), P['N'], P['C'], P['H'], P['W'], capi.ptr(o['y']),
                                            capi.stream()))
    return _run(launch, {'y': ((P['N'], P['C'], P['H'], P['W']), torch.float32)}, (P['a'], P['b'], P['al']), canary)


def _check_blend(P, out):
    ref, S = tfr.blend(P['a'], P['b'], P['al'])
    return scr.check_bound(out['y'], ref, S, 0.0, tfr.BETA_BLEND, tag='blend')


def _make_aa_down2(mode, case, seed):
    """Output h x w = H x W of the case (512 -> 256 at the production shape)."""
    N, H, W = case[:3]
    C = 3 if case[3] >= 256 else case[3]
    x = torch.rand(N, C, 2 * H, 2 * W, generator=_gen(seed), device=DEV) * 2 - 0.5
    return dict(entry='aa_down2', mode=mode, N=N, H=H, W=W, C=C, x=x, frame_keys=['x'])


def _run_aa_down2(P, canary=True):
    def launch(o):
        capi.check(capi.lib().r3dp_sr_resize_aa_down2(capi.ptr(P['x']), P['N'], P['C'], P['H'], P['W'], capi.ptr(o['y']), capi.stream()))
    return _run(launch, {'y': ((P['N'], P['C'], P['H'], P['W']), torch.float32)}, (P['x'],), canary)


def _check_aa_down2(P, out):
    x = P['x'].double()
    return scr.check_bound(out['y'], tfr.aa_down2(x), tfr.aa_down2(x.abs()), 0.0, tfr.BETA_AA, tag=f"aa_down2 {P['H']}x{P['W']}")


def _make_warp_input(mode, case, seed):
    """The renderer's channels-last features [N,h,w,C] and weights [N,h*w,1] -> x0 at size, rgb0, rgb_256, w_256.  Sizes are powers of two
    (exact source coordinates, torso_fusion_reference).  The production case is the renderer's 128^2 at size 128; the others have
    h, w < size, so that w_256's own source coordinates matter."""
    N, H, W = case[:3]
    h, w, size, C = {256: (128, 128, 128, 32), 7: (3, 4, 4, 8), 5: (37, 45, 64, 8)}[H]
    g = _gen(seed)
    return dict(entry='warp_input', mode=mode, N=N, h=h, w=w, size=size, C=C, x=torch.randn(N, h, w, C, generator=g, device=DEV),
                ws=torch.rand(N, h * w, 1, generator=g, device=DEV), frame_keys=['x', 'ws'])


def _run_warp_input(P, canary=True):
    N, size, wide = P['N'], P['size'], 2 if P['mode'] == 'tcx' else 1

    def launch(o):
        capi.check(capi.lib().r3dp_sr_warp_input(capi.ptr(P['x']), capi.ptr(P['ws']), N, P['C'], P['h'], P['w'], size, capi.ptr(o['x0'], F16),
                                                 capi.ptr(o['rgb0']), capi.ptr(o['rgb_256']), capi.ptr(o['w_256']), int(wide == 2), capi.stream()))
    shapes = {'x0': ((N, size, size, _pad64(P['C']) * wide), F16), 'rgb0': ((N, 3, size, size), torch.float32),
              'rgb_256': ((N, 3, 256, 256), torch.float32), 'w_256': ((N, 1, 256, 256), torch.float32)}
    return _run(launch, shapes, (P['x'], P['ws']), canary)


def _check_warp_input(P, out):
    split, C, Cp = P['mode'] == 'tcx', P['C'], _pad64(P['C'])
    refs = tfr.warp_input(P['x'], P['ws'], P['h'], P['w'], P['size'])
    beta = {'rgb0': tfr.BETA_BILINEAR, 'rgb_256': tfr.BETA_BILINEAR_TWICE, 'w_256': tfr.BETA_BILINEAR}
    r = max(scr.check_bound(out[k], *refs[k], 0.0, beta[k], tag=f"warp_input {P['mode']} {k}") for k in beta)
    x0 = out['x0']
    r = max(r, scr.check_bound(scr.nhwc(x0, split)[:, :C], *refs['x0'], tfr.alpha_store(split), tfr.BETA_BILINEAR_STORE, tfr.FLOOR_F16,
                               f"warp_input {P['mode']} x0"))
    v = out['rgb0'].permute(0, 2, 3, 1)                                     # x0's channels 0..2 are the store of rgb0, bit for bit
    hi = v.half()
    halves = (hi, (v - hi.float()).half()) if split else (hi,)
    for h, want in enumerate(halves):
        got = x0[..., h * Cp:(h + 1) * Cp]
        assert torch.equal(bits(got[..., :3].contiguous()), bits(want.contiguous())), f'warp_input: x0 half {h} is not the store of rgb0'
        assert bool((bits(got[..., C:]) == 0).all()), f'warp_input: x0 padding channels of half {h} are not zero'
    return r


ENTRIES = {
    'alpha_cat': (_make_alpha_cat, _run_alpha_cat, _check_alpha_cat),
    'cat3': (_make_cat3, _run_cat3, _check_cat3),
    'alpha_mix': (_make_alpha_mix, _run_alpha_mix, _check_alpha_mix),
    'alpha_gate': (_make_alpha_gate, _run_alpha_gate, _check_alpha_gate),
    'person': (_make_person, _run_person, _check_person),
    'blend': (_make_blend, _run_blend, _check_blend),
    'aa_down2': (_make_aa_down2, _run_aa_down2, _check_aa_down2),
    'warp_input': (_make_warp_input, _run_warp_input, _check_warp_input),
}
#: (N, H, W, Ca, Cb, extra channels per half of the operand stride, shared last operand).  'tc' / 'tcx' select the operand mode of the
#: entry points that have both; alpha_gate uses them for lo_off = 0 / > 0, person_occlusion for its two thresholds, blend and aa_down2
#: (fp32 only) run the same case twice with the same bits.
CASES = [
    (1, 256, 256, 256, 256, 0, False),          # production
    (3, 256, 256, 256, 256, 0, True),           # production, one shared frame (the per-clip background features)
    (3, 7, 9, 24, 40, 8, True),                 # ragged: the last block is partial, strides wider than the operands
    (2, 5, 7, 64, 16, 16, False),               # odd H and W
]


def _case_id(c):
    N, H, W, Ca, Cb, extra, shared = c
    return f'N{N}-{H}x{W}-C{Ca}+{Cb}-pad{extra}' + ('-shared' if shared else '')


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('case', CASES, ids=[_case_id(c) for c in CASES])
@pytest.mark.parametrize('entry', list(ENTRIES))
def test_fusion_vs_float64(entry, case, mode):
    make, run, check = ENTRIES[entry]
    P = make(mode, case, seed=100 * list(ENTRIES).index(entry) + CASES.index(case))
    check(P, run(P))


@pytest.mark.parametrize('hw', [(1, 1), (1, 6), (5, 1), (2, 3)])
def test_aa_down2_edge_shapes(hw):
    """Output sides of 1 and 2 (every tap of the filter at a border), where torch's antialiased resize cannot be the reference."""
    P = _make_aa_down2('tc', (3, *hw, 4), seed=6000 + hw[0] * 10 + hw[1])
    _check_aa_down2(P, _run_aa_down2(P))


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('entry', list(ENTRIES))
def test_fusion_bits_per_frame_and_repeat(entry, mode):
    """Frame k of an N = 3 launch = the N = 1 launch of frame k (a shared operand stays shared), and a repeated launch gives the same bits."""
    make, run, _ = ENTRIES[entry]
    P = make(mode, CASES[2], seed=5000 + list(ENTRIES).index(entry))
    full = run(P)
    again = run(P)
    for name in full:
        assert torch.equal(bits(full[name]), bits(again[name])), f'{entry} {mode}: repeated launch differs in {name}'
    for k in range(P['N']):
        one = run(_frame(P, k), canary=False)
        for name in full:
            assert torch.equal(bits(one[name]), bits(full[name][k:k + 1])), f'{entry} {mode}: frame {k} of the N=3 launch differs in {name}'


# ---- the v3 head-mask chain ------------------------------------------------------------------------------------------------------------------
def _chain_bound(x, layers, w_scale=2.0 ** -22, w_floor=2.0 ** -35):
    """Float64 forward of the alpha predictor's convs and an element-wise bound E on the kernel chain's error at every layer.  Layer l:
    E_l = conv(E_{l-1}, |W|) (Lipschitz propagation; LeakyReLU is 1-Lipschitz) + alpha_split |y_l| + FLOOR + beta_tcx S_l (the layer's own
    bound, sr_conv_reference) + the split weights' rounding, 2^-22 S_l + 2^-35 conv(|x|, 1), with S_l = conv(|x| + E, |W|) + |b|.
    The input is the split store of the fp32 inp7: E_0 = 2^-22 |x| + FLOOR."""
    E = scr.ALPHA_SPLIT * x.abs() + scr.FLOOR_F16
    for w, b, act in layers:
        ones = torch.ones_like(w)
        y = F.conv2d(x, w, b, padding=1)
        S = F.conv2d(x.abs() + E, w.abs(), b.abs(), padding=1)
        E = (F.conv2d(E, w.abs(), padding=1) + scr.ALPHA_SPLIT * y.abs() + scr.FLOOR_F16 + (scr.BETA['tcx'] + w_scale) * S
             + w_floor * F.conv2d(x.abs() + E, ones, padding=1))
        x = F.leaky_relu(y, 0.01) if act else y
    return x, E


@pytest.mark.parametrize('N', [1, 3])
def test_v3_mask_chain_vs_float64(N):
    """sr_with_ref.py:129-143 at 256^2: inp7 -> the split convs ap0 / ap2 / ap4 -> r3dp_sr_alpha_gate -> the 5 % quantile threshold ->
    r3dp_sr_person_occlusion, against the float64 head_torso_alpha_predictor on the module's weights.  The capped alpha must hold the
    chain's bound; the person masks may then differ only where the float64 alpha lies within that bound plus |thr_gpu - thr_ref| of
    the float64 threshold."""
    m = r3.SuperresolutionHybrid8XDC_Warp(channels=32, img_resolution=512, sr_num_fp16_res=0, sr_antialias=True, sr_mode='tc',
                                          hp=dict(syn.WARP_HPARAMS, htbsr_head_weight_fuse_mode='v3'), torso_model=syn.StubTorsoModel())
    m.load_state_dict(syn.make_sr_warp_params(seed=6, fuse_mode='v3'), strict=True)
    m = m.to(DEV).eval()
    g = _gen(7000 + N)
    rgb_h = 0.8 * torch.randn(N, 3, 256, 256, generator=g, device=DEV)
    weights_256 = torch.rand(N, 1, 256, 256, generator=g, device=DEV)
    rgb_torso = 0.8 * torch.randn(N, 3, 256, 256, generator=g, device=DEV)
    torso_occ = 1.4 * torch.rand(N, 1, 256, 256, generator=g, device=DEV) - 0.2
    thr0 = float(m.hparams['htbsr_head_threshold'])
    ap = m.head_torso_alpha_predictor
    with torch.no_grad():
        inp7 = torch.cat([rgb_h.clamp(-1, 1) / 2 + 0.5, weights_256, rgb_torso.clamp(-1, 1) / 2 + 0.5], dim=1)
        # the synthetic predictor keeps every alpha below the 0.9 threshold: shift its last bias (before the weights are packed) so that the
        # median logit sits at logit(0.93) and the head mask straddles the threshold
        logit0, _ = _chain_bound(inp7.double(), [(ap[i].weight.double(), ap[i].bias.double(), i < 4) for i in (0, 2, 4)])
        ap[4].bias += math.log(0.93 / 0.07) - float(logit0.median())
        plain = m._plain()
        t = sr_tc.to_nhwc_f16(inp7, 256, split=True)
        t = m._conv(m._conv(m._conv(t, plain['ap0'], 2, split=True), plain['ap2'], 2, split=True), plain['ap4'], 0, split=True)
        alpha = _run(lambda o: capi.check(capi.lib().r3dp_sr_alpha_gate(capi.ptr(t, F16), t.shape[-1], t.shape[-1] // 2, capi.ptr(weights_256), N, 256,
                                                                          256, capi.ptr(o['a']), capi.stream())),
                     {'a': ((N, 1, 256, 256), torch.float32)})['a']
        sel = alpha[alpha > 0.05]
        thr_gpu = max(float(sel.quantile(0.05)), thr0) if sel.numel() else thr0
        person = _run(lambda o: capi.check(capi.lib().r3dp_sr_person_occlusion(capi.ptr(alpha), capi.ptr(torso_occ), thr_gpu, N, 256, 256,
                                                                                capi.ptr(o['p']), capi.stream())),
                      {'p': ((N, 1, 256, 256), torch.float32)})['p']
        layers = [(ap[i].weight.double(), ap[i].bias.double(), i < 4) for i in (0, 2, 4)]
        logit, E = _chain_bound(inp7.double(), layers)
    s = torch.sigmoid(logit)
    cap = weights_256.double()
    alpha_ref = torch.minimum(s, cap)
    # the logit moves by at most E (sigmoid' = s (1 - s), which changes by at most a factor exp(E) over that step), then the gate's own bound
    # on the computed logit hi + lo (torso_fusion_reference)
    _, _, extra_gate = tfr.alpha_gate(logit, cap, True)
    bound = (s * (1 - s) * E + tfr.BETA_GATE * s) * E.exp() + extra_gate
    r = scr.check_bound(alpha, alpha_ref, bound, 0.0, 1.0, tag=f'v3 capped alpha N={N} (S = the derived bound, so the ratio is error / bound)')
    sel = alpha_ref[alpha_ref > 0.05]
    thr_ref = max(float(sel.quantile(0.05)), thr0) if sel.numel() else thr0
    band = (alpha_ref - thr_ref).abs() <= bound + abs(thr_gpu - thr_ref)
    person_ref = tfr.person_occlusion(alpha_ref, torso_occ, thr_ref)
    # outside the band both sides take the same branch: the masks differ by the alpha error and the rounding of torso + head (u of <= 2.5)
    d = (person.double() - person_ref).abs()
    outside = ~band
    allowed = bound + 2.5 * tfr.U
    bad = outside & ~(d <= allowed)
    forced_gpu, forced_ref = int((alpha > thr_gpu).sum()), int((alpha_ref > thr_ref).sum())
    print(f'v3 chain N={N}: worst error / bound {r:.3e}, max logit bound {float(E.max()):.3e}, thr gpu {thr_gpu!r} ref {thr_ref!r}, '
          f'{int(band.sum())} of {band.numel()} pixels in the disagreement band, forced to 1: gpu {forced_gpu} ref {forced_ref}, '
          f'masks differ (beyond the alpha bound) at {int((d > allowed).sum())} pixels')
    assert not bool(bad.any()), f'v3 chain: {int(bad.sum())} person-mask pixels differ outside the band'
    assert forced_ref > 0 and forced_ref < alpha.numel(), 'the head mask no longer straddles the threshold'
