"""SegFormerSECC2PlaneBackbone at the input sizes below 512^2, B = 3, against the float64 restatement computed on the device.

forward accepts any H = W that is a multiple of 32 in [32, 512].  32^2 runs stage 4 on one token (Tk = 1) and fuses a 1 x 1 head level;
96^2 gives partial 128-query tiles (576 queries), Tk = 9 and 3 x 3 tokens in stage 4; 480^2 runs to_plane_cnn on r3dp_mf_conv3d +
r3dp_sp_leaky (its 120^2 rows are not whole 128-pixel tiles) near the production size, with Tk = 225 and 14400 queries.  The bar is the
whole-backbone one of test_gpu_secc2plane.py (max |err| <= 3e-3 max |ref|); every frame must equal the same frame run alone bit for bit,
and at 96^2 planes_cl must equal forward."""
import pytest
import torch

import secc2plane_reference as ref
from test_gpu_secc2plane import BAR, DEV, module, rel

pytestmark = pytest.mark.gpu


def _input(mode, B, H, seed):
    cano, src, tgt = ref.make_inputs(B, H, seed)
    parts = [cano, src] if mode == 'cano_src_tgt' else [cano]
    return torch.cat([p.expand(B, -1, -1, -1) for p in parts] + [tgt], 1).to(DEV), (cano, src, tgt)


@torch.no_grad()
@pytest.mark.parametrize('H,mode', [(32, 'cano_src_tgt'), (96, 'cano_src_tgt'), (96, 'cano_tgt'), (480, 'cano_src_tgt')])
def test_backbone_sizes_vs_float64(H, mode):
    m = module(mode)
    B = 3
    x, _ = _input(mode, B, H, 20 + H)
    out = m(x)
    assert out.shape == (B, 3, 32, H // 2, H // 2)
    want = ref.forward(ref.to64(m.state_dict(), DEV), x.double())
    r = rel(out, want)
    print(f'secc2plane {H}^2 B={B} ({mode}) vs float64: max err / range = {r:.2e}')
    assert r < BAR, r
    for k in range(B):
        assert torch.equal(m(x[k:k + 1].contiguous()), out[k:k + 1]), k


@torch.no_grad()
def test_planes_cl_equals_forward_at_96():
    m = module()
    x, (cano, src, tgt) = _input('cano_src_tgt', 3, 96, 31)
    full = m(x)
    m.begin_clip(cano.to(DEV), src.to(DEV))
    pcl = m.planes_cl(tgt.to(DEV))
    assert pcl.layout == 'hwpc' and tuple(pcl.data.shape) == (3, 48, 48, 3, 32)
    assert torch.equal(pcl.data.permute(0, 3, 4, 1, 2), full)
