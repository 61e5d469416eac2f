"""Host side of torso_stage2='cuda' without a GPU: the weight folding against torch's own eval-mode spectral norm and BatchNorm, the nearest-up
phase composition in float64, the float64 restatement of stage 2 against the reference Generator, and the option's validation."""
import pytest
import torch
import torch.nn.functional as F

import real3dportrait_b200 as r3
from real3dportrait_b200 import synthetic as syn, torso_warp as tw
import torso_warper_ref as twr


class _Block(torch.nn.Module):
    """A ConvBlock2D 'CNA' shape (layers = conv, BN, act) built from torch's own spectral_norm and BatchNorm2d."""

    def __init__(self, i, o):
        super().__init__()
        self.layers = torch.nn.Sequential(torch.nn.utils.spectral_norm(torch.nn.Conv2d(i, o, 3, 1, 1)), torch.nn.BatchNorm2d(o), torch.nn.ReLU())


def test_folded_weights_equal_torch_eval():
    """sn_weight equals the `weight` torch's spectral-norm hook computes in eval mode; fold_cna equals conv -> BN (eval) in float64."""
    b = twr.randomize(_Block(24, 16), seed=3).double()
    x = torch.randn(2, 24, 9, 11, dtype=torch.float64)
    conv = b.layers[0]
    b.layers(x)                                                           # eval forward: the hook sets conv.weight without a power iteration
    assert torch.allclose(tw.sn_weight(conv), conv.weight.detach(), rtol=0, atol=1e-14)
    w, bias = tw.fold_cna(b)
    ref = b.layers[1](b.layers[0](x))
    assert float((F.conv2d(x, w, bias, padding=1) - ref).abs().max()) < 1e-12


@pytest.mark.parametrize('H,W', [(5, 7), (8, 8)])
def test_nearest_up_composition_float64(H, W):
    """The four parity phases of 2x2 composed taps reproduce upsample(x2, nearest) -> conv3x3 to 1e-12 in float64, borders included."""
    g = torch.Generator().manual_seed(H * W)
    x = torch.randn(2, 6, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(5, 6, 3, 3, generator=g, dtype=torch.float64)
    b = torch.randn(5, generator=g, dtype=torch.float64)
    ref = F.conv2d(F.interpolate(x, scale_factor=2, mode='nearest'), w, b, padding=1)
    got = twr.conv_up_nearest_phases(x, tw.compose_nearest_up(w), b)
    assert float((got - ref).abs().max()) < 1e-12


def test_folded_stage2_matches_reference_generator():
    """The float64 restatement of stage 2 (what the kernels compute) against the reference's network2.Generator + predictor in float64."""
    cls = twr.ref_classes()
    if cls is None:
        pytest.skip('the reference warper modules are not staged under oracle/_ref (oracle/make_ref.py)')
    gen = twr.randomize(cls[0](), seed=21).double()
    pred = twr.randomize(twr.make_predictor(), seed=22).double()
    fs, deformation, occ = twr.make_stage2_inputs(2, 16, seed=23)
    with torch.no_grad():
        ref = twr.reference_stage2(gen, pred, fs.double(), deformation.double(), occ.double())
        got = twr.folded_stage2_f64(gen, pred, fs, deformation, occ)
    for r, o in zip(ref, got):
        assert float((r - o).abs().max()) < 1e-9 * max(1.0, float(r.abs().max()))


def test_torso_stage2_option_validation():
    kw = dict(channels=32, img_resolution=512, sr_num_fp16_res=0, sr_antialias=True, torso_model=syn.StubTorsoModel())
    m = r3.SuperresolutionHybrid8XDC_Warp(hp=syn.WARP_HPARAMS, **kw)
    assert m.torso_stage2 == 'torch'
    with pytest.raises(ValueError):
        r3.SuperresolutionHybrid8XDC_Warp(hp=syn.WARP_HPARAMS, torso_stage2='eager', **kw)
    with pytest.raises(NotImplementedError):
        r3.SuperresolutionHybrid8XDC_Warp(hp=dict(syn.WARP_HPARAMS, torso_model_version='v1'), torso_stage2='cuda', **kw)
    with pytest.raises(NotImplementedError):
        r3.SuperresolutionHybrid8XDC_Warp(hp=syn.WARP_HPARAMS, torso_stage2='cuda', sr_mode='fp32', **kw)
    # the option adds no state_dict key
    assert set(r3.SuperresolutionHybrid8XDC_Warp(hp=syn.WARP_HPARAMS, torso_stage2='cuda', **kw).state_dict()) == set(m.state_dict())
