"""Img2PlaneModel on the device against the float64 restatement (tests/img2plane_reference.py) at 512^2 (B = 4, 1), 144^2 and 32^2 (B = 3)
and 16^2 (B = 1), and against the reference's own fixture at 128^2.  Bar: max |err| <= 3e-3 max |ref| (secc2plane's).  Also: planes_cl
equals forward bit for bit and writes into a caller's buffer; one 512^2 B = 1 forward allocates under 512 MB above its inputs and weights."""
import pytest
import torch

import img2plane_reference as ref
from conftest import load_golden
from real3dportrait_b200.img2plane import Img2PlaneModel

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
#: stays at 3e-3: fp16 operand rounding alone moves the planes by ~1.25e-3 max|ref|, and accumulating the same rounded operands in fp32
#: instead of float64 moves them ~1e-3 again (tests/test_cpu_img2plane_launches.py), so no emulation tightens it; faults below it are
#: the per-launch tests' (tests/test_gpu_img2plane_launches.py)
BAR = 3e-3


def _model(seed=5, scale='standard'):
    m = Img2PlaneModel(hp={'img2plane_backbone_scale': scale})
    sd = ref.make_params({k: v.shape for k, v in m.state_dict().items()}, seed)
    m.load_state_dict(sd, strict=True)
    return m.to(DEV).eval(), {k: (v.to(DEV, torch.float64) if v.is_floating_point() else v.to(DEV)) for k, v in sd.items()}


@pytest.mark.parametrize('B,H,scale', [(4, 512, 'standard'), (1, 512, 'standard'), (3, 144, 'standard'), (3, 32, 'standard'),
                                       (1, 16, 'standard'), (1, 64, 'small'), (1, 64, 'large')], ids=lambda v: str(v))
@torch.no_grad()
def test_forward_matches_float64_restatement(B, H, scale):
    m, sd = _model(scale=scale)
    x = ref.make_inputs(B, H, 11).to(DEV)
    got = m(x)
    want = ref.forward(sd, x.double(), scale)
    assert got.shape == want.shape == (B, 3, 32, H // 2, H // 2)
    err = float((got.double() - want).abs().max()) / float(want.abs().max())
    print(f'img2plane B{B} {H}^2 {scale}: max|err| / max|ref| = {err:.2e}')
    assert err <= BAR, err


@torch.no_grad()
def test_forward_matches_reference_fixture():
    g = load_golden('img2plane_small')
    m, _ = _model(int(g['param_seed']))
    x = ref.make_inputs(1, int(g['size']), int(g['input_seed'])).to(DEV)
    got = m(x)[..., ::2, ::2].double().cpu()
    want = g['planes_s2'].double()
    err = float((got - want).abs().max()) / float(want.abs().max())
    print(f'img2plane vs the reference fixture (128^2): {err:.2e}')
    assert err <= BAR, err


@torch.no_grad()
def test_planes_cl_equals_forward_and_fills_out():
    m, _ = _model()
    x = ref.make_inputs(2, 144, 3).to(DEV)
    f = m(x)
    cl = m.planes_cl(x)
    assert cl.layout == 'hwpc' and tuple(cl.data.shape) == (2, 72, 72, 3, 32)
    assert torch.equal(cl.data.permute(0, 3, 4, 1, 2), f)
    out = torch.full((2, 72, 72, 3, 32), float('nan'), device=DEV)
    cl2 = m.planes_cl(x, out=out)
    assert cl2.data.data_ptr() == out.data_ptr() and torch.equal(out, cl.data)
    with pytest.raises(ValueError):
        m.planes_cl(x, out=torch.empty(1, 72, 72, 3, 32, device=DEV))


@torch.no_grad()
def test_peak_memory_512():
    m, _ = _model()
    x = ref.make_inputs(1, 512, 2).to(DEV)
    m(x)                                                              # weights packed
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = m(x)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print(f'img2plane 512^2 B = 1: peak allocation {peak / 2**20:.1f} MB above inputs and weights')
    assert peak < 512 * 2**20
    del out


def test_gpu_rejects_bad_inputs():
    m, _ = _model()
    with pytest.raises(ValueError):
        m(torch.zeros(1, 3, 64, 80, device=DEV))
    with pytest.raises(ValueError):
        m(torch.zeros(1, 3, 72, 72, device=DEV))
