"""The bars of tests/torso_fusion_reference.py have teeth (no GPU needed): a float32 restatement of each kernel of csrc/sr_tc.cu passes
its bar, and a restatement with one plausible bug (a mutant) fails it.  Also: the antialiased 1/2 filter matrix is torch's, and the torso
head refuses sr_antialias=False, whose down-sampling it does not build."""
import pytest
import torch
import torch.nn.functional as F

import real3dportrait_b200 as r3
import sr_conv_reference as scr
import torso_fusion_reference as tfr
from real3dportrait_b200 import synthetic as syn


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _split(v):
    hi = v.half()
    return hi, (v - hi.float()).half()


def _fma(a, b, c):
    """fp32 fmaf through float64: the product of two fp32 values is exact in float64, one rounding to fp32 remains (up to a double
    rounding far inside the bars)."""
    return (a.double() * b.double() + c.double()).float()


def _fails(fn):
    with pytest.raises(AssertionError):
        fn()


# ---- alpha_cat / cat3 ------------------------------------------------------------------------------------------------------------------
def _cat_operands(N=3, H=4, W=5, Ca=16, Cb=24, shared=True, seed=1):
    g = _g(seed)
    xa = torch.randn(N, H, W, Ca, generator=g)
    xb = torch.randn(1 if shared else N, H, W, Cb, generator=g)
    al = torch.rand(N, H, W, generator=g)
    al[0, 0, :2] = torch.tensor([0.0, 1.0])
    return xa, xb, al


def _alpha_cat_tc(xa16, xb16, al, shared_index=True):
    """r3dp_sr_alpha_cat_ex: fp16(x * m) in fp32.  shared_index=False: the shared operand read at the pixel index of the whole batch
    (frames 1.. read whatever follows frame 0: here, other data)."""
    N = xa16.shape[0]
    xb = xb16.float().expand(N, -1, -1, -1).clone()
    if not shared_index:
        xb[1:] = torch.randn(xb[1:].shape, generator=_g(99)).half().float()
    a = al[..., None]
    return torch.cat([(xa16.float() * a).half(), (xb * (1 - a)).half()], dim=-1)


def test_alpha_cat_tc_bar_and_mutant():
    xa, xb, al = _cat_operands()
    xa16, xb16 = xa.half(), xb.half()
    ref = tfr.alpha_cat(xa16, xb16, al)
    got = _alpha_cat_tc(xa16, xb16, al)
    scr.check_bound(got, ref, ref.abs(), tfr.ALPHA_CAT['tc'], 0.0, tfr.FLOOR_F16, 'alpha_cat tc sim')
    _fails(lambda: scr.check_bound(_alpha_cat_tc(xa16, xb16, al, shared_index=False), ref, ref.abs(), tfr.ALPHA_CAT['tc'], 0.0, tfr.FLOOR_F16))


def _alpha_cat_tcx(xa, xb, al, lo_zero=False):
    """r3dp_sr_tcx_alpha_cat_ex: (hi + lo) * m in fp32, then the [hi | lo] split of the (Ca + Cb)-channel result."""
    N = xa[0].shape[0]
    a = al[..., None]
    va = (xa[0].float() + xa[1].float()) * a
    vb = (xb[0].float() + xb[1].float()).expand(N, -1, -1, -1) * (1 - a)
    v = torch.cat([va, vb], dim=-1)
    hi, lo = _split(v)
    return torch.cat([hi, torch.zeros_like(lo) if lo_zero else lo], dim=-1)


def test_alpha_cat_tcx_bar_and_mutant():
    xa, xb, al = _cat_operands(seed=2)
    sa, sb = _split(xa), _split(xb)
    ref = tfr.alpha_cat(sa[0].double() + sa[1].double(), sb[0].double() + sb[1].double(), al)
    got = tfr.join(_alpha_cat_tcx(sa, sb, al))
    scr.check_bound(got, ref, ref.abs(), tfr.ALPHA_CAT['tcx'], 0.0, tfr.FLOOR_F16, 'alpha_cat tcx sim')
    _fails(lambda: scr.check_bound(tfr.join(_alpha_cat_tcx(sa, sb, al, lo_zero=True)), ref, ref.abs(), tfr.ALPHA_CAT['tcx'], 0.0, tfr.FLOOR_F16))


# ---- alpha_mix / blend -------------------------------------------------------------------------------------------------------------------
def _mix_f32(a, b, al, fused):
    """a * al + b * (1 - al) in fp32, with the first product contracted into an fma or not."""
    m = 1 - al
    if fused:
        return _fma(a, al, b * m)
    return a * al + b * m


@pytest.mark.parametrize('fused', [False, True])
def test_alpha_mix_tc_bar_either_contraction(fused):
    g = _g(3)
    xa, xb = torch.randn(2, 3, 5, 16, generator=g).half(), torch.randn(2, 3, 5, 16, generator=g).half()
    al = torch.rand(2, 3, 5, generator=g)
    ref, S = tfr.alpha_mix(xa, xb, al)
    got = _mix_f32(xa.float(), xb.float(), al[..., None], fused).half()
    scr.check_bound(got, ref, S, tfr.ALPHA_MIX['tc'], tfr.BETA_MIX['tc'], tfr.FLOOR_F16, f'alpha_mix tc sim fused={fused}')


def test_alpha_mix_tcx_bar_and_mutant():
    """Mutant: the lo half read at the full pixel stride instead of half of it (with stride 2C: the next pixel's hi half)."""
    g = _g(4)
    N, H, W, C = 2, 3, 5, 16
    a, b = _split(torch.randn(N, H, W, C, generator=g)), _split(torch.randn(N, H, W, C, generator=g))
    al = torch.rand(N, H, W, generator=g)
    ref, S = tfr.alpha_mix(a[0].double() + a[1].double(), b[0].double() + b[1].double(), al)

    def run(lo_of):
        v = _mix_f32(a[0].float() + lo_of(a).float(), b[0].float() + lo_of(b).float(), al[..., None], False)
        return tfr.join(torch.cat(_split(v), dim=-1))

    def next_hi(t):
        flat = t[0].reshape(-1, C)
        return torch.cat([flat[1:], torch.zeros(1, C, dtype=flat.dtype)]).reshape(t[0].shape)
    scr.check_bound(run(lambda t: t[1]), ref, S, tfr.ALPHA_MIX['tcx'], tfr.BETA_MIX['tcx'], tfr.FLOOR_F16, 'alpha_mix tcx sim')
    _fails(lambda: scr.check_bound(run(next_hi), ref, S, tfr.ALPHA_MIX['tcx'], tfr.BETA_MIX['tcx'], tfr.FLOOR_F16))


def test_blend_bar_and_mutant():
    """Mutant: alpha of frame 0 used for every frame."""
    g = _g(5)
    a, b = torch.randn(3, 3, 4, 6, generator=g), torch.randn(3, 3, 4, 6, generator=g)
    al = torch.rand(3, 1, 4, 6, generator=g)
    ref, S = tfr.blend(a, b, al)
    for fused in (False, True):
        scr.check_bound(_mix_f32(a, b, al, fused), ref, S, 0.0, tfr.BETA_BLEND, tag=f'blend sim fused={fused}')
    _fails(lambda: scr.check_bound(_mix_f32(a, b, al[:1].expand_as(al), False), ref, S, 0.0, tfr.BETA_BLEND))


# ---- alpha_gate / person_occlusion -------------------------------------------------------------------------------------------------------
def gate_logits(n, seed):
    """n logits as (hi, lo) fp16 pairs: random fp32 values plus the saturation edges +-20, +-88, +-65504 (lo = 0 there)."""
    v = 4 * torch.randn(n, generator=_g(seed))
    edges = torch.tensor([20.0, -20.0, 88.0, -88.0, 65504.0, -65504.0, 0.0])
    v[:edges.numel()] = edges
    return _split(v)


def test_alpha_gate_bar_and_mutant():
    """Mutant: lo_off ignored (the logit is the hi half alone)."""
    hi, lo = gate_logits(4096, 6)
    cap = torch.rand(4096, generator=_g(7))
    cap[::2] = 1.0                                                            # caps above and below the sigmoid
    for summed in (False, True):
        v32 = hi.float() + lo.float() if summed else hi.float()
        ref, S, extra = tfr.alpha_gate(hi.double() + (lo.double() if summed else 0), cap, summed)
        got = torch.minimum(1.0 / (1.0 + torch.exp(-v32)), cap)
        scr.check_bound(got, ref, S, 0.0, tfr.BETA_GATE, extra, f'alpha_gate sim summed={summed}')
    ref, S, extra = tfr.alpha_gate(hi.double() + lo.double(), cap, True)
    _fails(lambda: scr.check_bound(torch.minimum(1.0 / (1.0 + torch.exp(-hi.float())), cap), ref, S, 0.0, tfr.BETA_GATE, extra))


def test_person_occlusion_threshold_is_fp32_and_strict():
    """torch compares an fp32 tensor with a Python float in fp32 (as the kernel does with the float it is passed): at thr = 0.3, whose
    fp32 value lies above 0.3, alpha = fp32(0.3) is not above the threshold.  Mutant: >= instead of >."""
    thr = 0.3
    t32 = torch.tensor(thr, dtype=torch.float32)
    assert float(t32) > thr
    alpha = torch.stack([torch.nextafter(t32, torch.tensor(0.0)), t32, torch.nextafter(t32, torch.tensor(1.0))]).view(1, 1, 1, 3)
    torso = torch.tensor([0.5, 0.2, -0.4]).view(1, 1, 1, 3)
    got = tfr.person_occlusion_f32(alpha, torso, thr)
    assert torch.equal(got[..., :2], torso[..., :2] + alpha[..., :2])       # at fp32(thr) not forced to 1: compared in fp32
    assert float(got[..., 2]) == 0.6000000238418579                          # fp32(-0.4) + 1
    mutant = (torso + torch.where(alpha >= t32, torch.ones_like(alpha), alpha)).clamp(0, 1)
    assert not torch.equal(mutant, got)


# ---- resize_aa_down2 -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('hw', [(256, 256), (3, 5), (7, 2), (2, 9), (1, 1)])
def test_aa_down2_matrix_is_torch_antialias(hw):
    """The filter matrices against F.interpolate(antialias=True) in float64.  Not at shapes with exactly one output side of 1: torch 2.11
    returns wrong values there ([1,1,4,2] -> (2,1) gives one value for both rows), so those are covered by the matrix alone (below)."""
    h, w = hw
    x = torch.randn(2, 3, 2 * h, 2 * w, generator=_g(8), dtype=torch.float64)
    ref = F.interpolate(x, size=(h, w), mode='bilinear', align_corners=False, antialias=True)
    assert torch.allclose(tfr.aa_down2(x), ref, rtol=1e-13, atol=1e-13)


def test_aa_down2_matrix_rows():
    assert torch.equal(tfr.aa_down2_matrix(1), torch.tensor([[0.5, 0.5]], dtype=torch.float64))
    M = tfr.aa_down2_matrix(4)
    assert torch.allclose(M[0, :3], torch.tensor([3.0, 3.0, 1.0], dtype=torch.float64) / 7)
    assert torch.allclose(M[-1, -3:], torch.tensor([1.0, 3.0, 3.0], dtype=torch.float64) / 7)
    assert torch.allclose(M[1, 1:5], torch.tensor([1.0, 3.0, 3.0, 1.0], dtype=torch.float64) / 8)


def aa_down2_f32(x, renormalise=True):
    """aa_down2_kernel in fp32: weights k / sum of the taps inside (k / 2 when not renormalised), two fma chains."""
    h, w = x.shape[-2] // 2, x.shape[-1] // 2
    k4 = torch.tensor([0.25, 0.75, 0.75, 0.25])

    def weights(n):
        idx = 2 * torch.arange(n)[:, None] - 1 + torch.arange(4)[None]
        inside = (idx >= 0) & (idx < 2 * n)
        wt = torch.where(inside, k4, torch.zeros(()))
        s = wt.sum(1, keepdim=True) if renormalise else torch.full((n, 1), 2.0)
        return wt / s, idx.clamp(0, 2 * n - 1)
    wy, iy = weights(h)
    wx, ix = weights(w)
    acc = torch.zeros(*x.shape[:-2], h, w)
    for u in range(4):
        rows = x[..., iy[:, u], :]                                            # [..., h, 2w]
        row = torch.zeros(*x.shape[:-2], h, w)
        for v in range(4):
            row = _fma(wx[:, v], rows[..., ix[:, v]], row)
        acc = _fma(wy[:, u, None], row, acc)
    return acc


@pytest.mark.parametrize('hw', [(16, 16), (3, 5), (1, 4), (1, 1)])
def test_aa_down2_bar_and_mutant(hw):
    """Mutant: the taps divided by 2 instead of their sum (no border renormalisation)."""
    h, w = hw
    x = torch.rand(2, 3, 2 * h, 2 * w, generator=_g(9)) + 0.5
    ref, S = tfr.aa_down2(x.double()), tfr.aa_down2(x.double().abs())
    scr.check_bound(aa_down2_f32(x), ref, S, 0.0, tfr.BETA_AA, tag=f'aa_down2 sim {hw}')
    _fails(lambda: scr.check_bound(aa_down2_f32(x, renormalise=False), ref, S, 0.0, tfr.BETA_AA))


# ---- warp_input ----------------------------------------------------------------------------------------------------------------------------
def _coord(o, n, size):
    s = torch.clamp_min(_fma(o.float() + 0.5, torch.tensor(n / size, dtype=torch.float32), torch.tensor(-0.5)), 0.0)
    i0 = torch.clamp_max(s.long(), n - 1)
    return i0, torch.clamp_max(i0 + 1, n - 1), s - i0.float()


def bilinear_f32(x, h, w, size, coord_hw=None):
    """bilinear_coord + bilinear_mix on fp32 [N,C,h,w] -> [N,C,size,size].  coord_hw: the source extent the coordinates are computed
    for (a mutant passes the wrong one; the flat frame is then read past its end, here zeros)."""
    ch, cw = coord_hw or (h, w)
    o = torch.arange(size)
    y0, y1, ty = _coord(o, ch, size)
    x0, x1, tx = _coord(o, cw, size)
    flat = torch.cat([x.reshape(*x.shape[:2], h * w), torch.zeros(*x.shape[:2], ch * cw)], -1)

    def at(yy, xx):
        return flat[..., (yy[:, None] * w + xx[None, :]).reshape(-1)].reshape(*x.shape[:2], size, size)
    ty, tx = ty[:, None], tx[None, :]
    r0 = _fma(at(y0, x0), 1 - ty, at(y1, x0) * ty)
    r1 = _fma(at(y0, x1), 1 - ty, at(y1, x1) * ty)
    return _fma(r0, 1 - tx, r1 * tx)


def test_warp_input_bar_and_mutant():
    """All four outputs of warp_input_kernel restated in fp32 against the float64 references.  Mutant: w_256 resized with the
    coordinates of a size x size source instead of h x w."""
    N, C, h, w, size = 2, 8, 37, 45, 64
    g = _g(10)
    x = torch.randn(N, h, w, C, generator=g)
    wsum = torch.rand(N, h * w, 1, generator=g)
    refs = tfr.warp_input(x, wsum, h, w, size)
    rgb0 = bilinear_f32(x.permute(0, 3, 1, 2)[:, :3], h, w, size)
    ws = wsum.view(N, 1, h, w)
    got = {'rgb0': rgb0, 'rgb_256': bilinear_f32(rgb0, size, size, 256), 'w_256': bilinear_f32(ws, h, w, 256)}
    beta = {'rgb0': tfr.BETA_BILINEAR, 'rgb_256': tfr.BETA_BILINEAR_TWICE, 'w_256': tfr.BETA_BILINEAR}
    for k, v in got.items():
        scr.check_bound(v, *refs[k], 0.0, beta[k], tag=f'warp_input sim {k}')
    x0 = bilinear_f32(x.permute(0, 3, 1, 2), h, w, size).half()
    scr.check_bound(x0, *refs['x0'], tfr.ALPHA_F16, tfr.BETA_BILINEAR_STORE, tfr.FLOOR_F16, 'warp_input sim x0')
    _fails(lambda: scr.check_bound(bilinear_f32(ws, h, w, 256, coord_hw=(size, size)), *refs['w_256'], 0.0, tfr.BETA_BILINEAR))


# ---- the torso head's options --------------------------------------------------------------------------------------------------------
def test_torso_head_rejects_sr_antialias_false():
    """The head down-samples its 512^2 reference images with the antialiased filter only; sr_antialias=False would need plain bilinear
    down-sampling there, which is not built."""
    kw = dict(channels=32, img_resolution=512, sr_num_fp16_res=0, hp=syn.WARP_HPARAMS)
    with pytest.raises(NotImplementedError, match='sr_antialias'):
        r3.SuperresolutionHybrid8XDC_Warp(sr_antialias=False, **kw)
    assert r3.SuperresolutionHybrid8XDC_Warp(sr_antialias=True, **kw).sr_antialias
