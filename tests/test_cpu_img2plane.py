"""Img2PlaneModel on the host: the float64 restatement against the reference's own fixture, state_dict compatibility with the reference
class, the float64 BatchNorm fold, the block counts of each backbone scale and the rejected configurations."""
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import img2plane_reference as ref
from conftest import load_golden
from real3dportrait_b200 import img2plane as ip
from real3dportrait_b200.img2plane import Img2PlaneModel

HERE = os.path.dirname(os.path.abspath(__file__))
REF_ROOT = ref.reference_checkout()


def _params(m, seed):
    return ref.make_params({k: v.shape for k, v in m.state_dict().items()}, seed)


def _to64(sd):
    return {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}


def test_restatement_matches_reference_fixture():
    g = load_golden('img2plane_small')
    m = Img2PlaneModel()
    sd = _to64(_params(m, int(g['param_seed'])))
    x = ref.make_inputs(1, int(g['size']), int(g['input_seed']))
    with torch.no_grad():
        out = ref.forward(sd, x.double())
    want = g['planes_s2'].double()
    got = out[..., ::2, ::2]
    assert got.shape == want.shape
    err = float((got - want).abs().max())
    assert err <= 1e-6 * float(want.abs().max()), err              # float32 storage of a float64 run


def test_fixture_activations_are_order_one():
    """No stage of the seeded network dominates: every stage's output stays within a factor of 20 of unit RMS."""
    m = Img2PlaneModel()
    sd = _to64(_params(m, 5))
    x = ref.with_coords(ref.make_inputs(1, 64, 9).double())
    with torch.no_grad():
        e = ref.encoder(sd, x)
        dec = ref.decoder(sd, e)
        low = ref.low_vit(sd, dec, 5)
        high = ref.high_res(sd, x)
        planes = ref.tri_vit(sd, low, high, 1)
    for name, t in (('encoder', e), ('decoder', dec), ('low', low), ('high', high), ('planes', planes)):
        rms = float(t.pow(2).mean().sqrt())
        assert 0.05 < rms < 20, (name, rms)


_KEYS_SCRIPT = r'''
import json, sys
sys.path.insert(0, sys.argv[2])
import img2plane_reference as ref
hp = json.loads(sys.argv[3])
Ref = ref.reference_class(sys.argv[1], hp)
m = Ref(out_channels=96, hp=hp)
print(json.dumps({k: list(v.shape) for k, v in m.state_dict().items()}))
'''


@pytest.mark.skipif(REF_ROOT is None, reason='needs a reference checkout (R3DP_REFERENCE)')
@pytest.mark.parametrize('scale', ['small', 'standard', 'large'])
def test_state_dict_matches_reference_class(scale):
    """Keys and shapes equal the reference class's, built in a child process behind the shims and the network guard."""
    hp = {'img2plane_input_mode': 'rgb', 'img2plane_backbone_scale': scale, 'triplane_feature_type': 'triplane', 'triplane_depth': 1}
    r = subprocess.run([sys.executable, '-c', _KEYS_SCRIPT, REF_ROOT, HERE, json.dumps(hp)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    theirs = json.loads(r.stdout.strip().splitlines()[-1])
    ours = {k: list(v.shape) for k, v in Img2PlaneModel(hp=hp).state_dict().items()}
    assert list(theirs) == list(ours)
    assert theirs == ours


def test_state_dict_round_trip():
    m = Img2PlaneModel()
    sd = _params(m, 3)
    m.load_state_dict(sd, strict=True)
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), k


@pytest.mark.parametrize('scale,counts', [('small', (2, 1)), ('standard', (5, 1)), ('large', (10, 3))])
def test_block_counts_follow_hp(scale, counts):
    m = Img2PlaneModel(hp={'img2plane_backbone_scale': scale})
    assert (m.low_reso_vit.num_blocks, m.triplane_predictor_vit.num_blocks) == counts
    keys = m.state_dict().keys()
    assert f'low_reso_vit.block{counts[0]}.attn.q.weight' in keys and f'low_reso_vit.block{counts[0] + 1}.attn.q.weight' not in keys
    assert f'triplane_predictor_vit.block{counts[1]}.attn.sr.weight' in keys


def test_bn_fold_equals_conv_then_bn():
    m = Img2PlaneModel()
    m.load_state_dict(_params(m, 4))
    blk = m.low_reso_encoder.encoder.layer3[0]
    x = torch.randn(2, 128, 9, 9, dtype=torch.float64)
    bn = blk.bn1
    want = F.batch_norm(F.conv2d(x, blk.conv1.weight.detach().double(), None, 1, 2, 2), bn.running_mean.double(), bn.running_var.double(),
                        bn.weight.double(), bn.bias.double(), False, 0.0, bn.eps)
    w, b = ip.fold_conv_bn(blk.conv1.weight, bn)
    got = F.conv2d(x, w, b, 1, 2, 2)
    assert float((got - want).detach().abs().max()) <= 1e-12 * float(want.abs().max())


@pytest.mark.parametrize('hp', [{'img2plane_input_mode': 'rgb_alpha'}, {'img2plane_input_mode': 'rgb_camera'},
                                {'img2plane_input_mode': 'rgb_alpha_camera'}, {'triplane_feature_type': 'trigrid'},
                                {'triplane_feature_type': 'trigrid_v2'}, {'triplane_depth': 2}, {'img2plane_backbone_scale': 'huge'}])
def test_unsupported_configurations_raise(hp):
    with pytest.raises(NotImplementedError):
        Img2PlaneModel(hp=hp)


def test_other_out_channels_raise():
    with pytest.raises(NotImplementedError):
        Img2PlaneModel(out_channels=64)


@pytest.mark.parametrize('shape', [(1, 3, 64, 96), (1, 3, 72, 72), (1, 3, 8, 8), (1, 4, 64, 64), (3, 64, 64)])
def test_bad_inputs_raise(shape):
    with pytest.raises(ValueError):
        Img2PlaneModel._check_image(torch.zeros(shape), 'forward')


def test_cpu_tensors_raise():
    with pytest.raises(RuntimeError, match='CUDA'):
        Img2PlaneModel()(torch.zeros(1, 3, 64, 64))
