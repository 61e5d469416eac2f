"""SegFormerSECC2PlaneBackbone on the H100: the whole backbone against the reference's fixture (128^2) and against the float64
restatement computed on the device (512^2, B = 1 and 4), batch independence, forward == begin_clip + planes_cl, and the render of the
(canonical, secc) pair against the render of the materialised sum.

Bars are relative to the output range R = max |ref|: the backbone runs ~40 fp16-operand GEMMs/convs in sequence (the `tc` contract), so
its error is a few fp16 ulps of R, not fp32-grade.  The measured ratios are printed (pytest -s) and recorded in DESIGN.md."""
import pytest
import torch

import secc2plane_reference as ref
from conftest import load_golden
import real3dportrait_b200 as r3
from real3dportrait_b200 import _capi as capi
from real3dportrait_b200 import synthetic as syn

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
BAR = 3e-3          # |got - ref| <= BAR * max|ref|; measured <= 9.0e-4 on an H100 (DESIGN.md)


def module(mode='cano_src_tgt', seed=7):
    m = r3.SegFormerSECC2PlaneBackbone(pncc_cond_mode=mode)
    m.load_state_dict(ref.make_params({k: v.shape for k, v in m.state_dict().items()}, seed), strict=True)
    return m.to(DEV).eval()


def rel(got, want):
    return float((got.double() - want.double()).abs().max()) / float(want.double().abs().max())


@torch.no_grad()
def test_backbone_matches_reference_fixture():
    g = load_golden('secc2plane_small')
    m = module(seed=int(g['param_seed']))
    cano, src, tgt = ref.make_inputs(1, int(g['size']), int(g['input_seed']))
    out = m(torch.cat([cano, src, tgt], 1).to(DEV))
    assert out.shape == (1, 3, 32, 64, 64)
    r = rel(out[..., ::2, ::2].cpu(), g['planes_s2'])
    print(f'secc2plane 128^2 vs reference fixture: max err / range = {r:.2e}')
    assert r < BAR, r


@torch.no_grad()
@pytest.mark.parametrize('mode', ['cano_src_tgt', 'cano_tgt'])
def test_backbone_matches_float64_at_512(mode):
    m = module(mode)
    sd = ref.to64(m.state_dict(), DEV)
    cano, src, tgt = ref.make_inputs(4, 512, 3)
    parts = [cano, src] if mode == 'cano_src_tgt' else [cano]
    x = torch.cat([p.expand(4, -1, -1, -1) for p in parts] + [tgt], 1).to(DEV)
    out = m(x)
    want = ref.forward(sd, x.double())
    r = rel(out, want)
    print(f'secc2plane 512^2 B=4 ({mode}) vs float64: max err / range = {r:.2e}')
    assert r < BAR, r
    # image k of the batch is bit-identical to that frame alone
    for k in range(4):
        assert torch.equal(m(x[k:k + 1].contiguous()), out[k:k + 1]), k


@torch.no_grad()
def test_planes_cl_equals_forward():
    m = module()
    cano, src, tgt = (t.to(DEV) for t in ref.make_inputs(2, 512, 5))
    full = m(torch.cat([cano.expand(2, -1, -1, -1), src.expand(2, -1, -1, -1), tgt], 1))
    m.begin_clip(cano, src)
    pcl = m.planes_cl(tgt)
    assert pcl.layout == 'hwpc' and tuple(pcl.data.shape) == (2, 256, 256, 3, 32)
    got = pcl.data.permute(0, 3, 4, 1, 2)
    assert torch.equal(got, full)       # the prenet's fmas run in the same order on both paths: bias, cano/src taps, tgt taps
    # a second clip refills the cached image
    m.begin_clip(-cano, src)
    full2 = m(torch.cat([-cano.expand(2, -1, -1, -1), src.expand(2, -1, -1, -1), tgt], 1))
    assert torch.equal(m.planes_cl(tgt).data.permute(0, 3, 4, 1, 2), full2)


@torch.no_grad()
def test_render_of_pair_equals_render_of_sum():
    m = module()
    cano_in, src, tgt = (t.to(DEV) for t in ref.make_inputs(2, 512, 9))
    m.begin_clip(cano_in, src)
    secc_cl = m.planes_cl(tgt)
    cano = syn.make_planes(1, seed=0).to(DEV)
    cano_cl = r3.canonical_planes_cl(cano)
    cam = syn.make_cameras(2, seed=1).to(DEV)
    u_c, _ = syn.make_jitter(2, 4096, 48, 0, seed=2)
    head = r3.RenderHead(hp={'num_samples_fine': 0})
    sd = {'decoder.' + k: v for k, v in syn.make_decoder_params(seed=4).items()}
    sd.update({'superresolution.' + k: v for k, v in syn.make_sr_params(seed=5).items()})
    head.load_state_dict(sd, strict=True)
    head = head.to(DEV).eval()
    summed = (cano + secc_cl.data.permute(0, 3, 4, 1, 2)).contiguous()      # [2,3,32,256,256], materialised
    capi.PROF = capi.Profiler()
    try:
        pair = head.synthesis((cano_cl, secc_cl), cam, u_coarse=u_c.to(DEV))
        names = {n for n, _, _ in capi.PROF.events}
    finally:
        capi.PROF = None
    assert 'repack' not in names, names
    full = head.synthesis(summed, cam, u_coarse=u_c.to(DEV))
    d_raw = float((pair['image_raw'] - full['image_raw']).abs().max())
    d_img = float((pair['image'] - full['image']).abs().max())
    print(f'pair vs materialised sum: image_raw {d_raw:.2e}, image {d_img:.2e}')
    assert d_raw < 1e-4 and d_img < 1e-3, (d_raw, d_img)
