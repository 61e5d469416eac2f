"""PitchContourVAEModel / VAEModel on the host: the float64 restatement against the reference's own fixture, state_dict compatibility
(keys and shapes of both classes at A = 1024 and 13, strict loading), the host folds (weight norm, BatchNorm, Flips, cond_proj's blink /
amplitude columns, the gate pairing, g_pre_net over groups of four, the transposed conv) against the unfolded restatement, the seeded
prior draw, f0_to_coarse, and every rejected configuration and input that needs no device."""
import os

import numpy as np
import pytest
import torch

import audio2motion_reference as ref
from real3dportrait_b200 import PitchContourVAEModel, VAEModel
from real3dportrait_b200 import audio2motion as a2m

CASES = [('pitch', 1024), ('vae', 1024), ('vae', 13)]
REF_ROOT = ref.reference_checkout()
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'audio2motion_small.npz')


def _golden():
    """The fixture: numeric arrays as tensors, the state_dict key / shape lists as numpy string arrays."""
    z = np.load(GOLDEN)
    return {k: (z[k].item() if z[k].ndim == 0 else z[k] if z[k].dtype.kind == 'U' else torch.from_numpy(z[k])) for k in z.files}


def _model(kind, A, hp=ref.HP_PITCH):
    return PitchContourVAEModel(hp, audio_in_dim=A) if kind == 'pitch' else VAEModel(audio_in_dim=A)


def _seeded(m, seed):
    sd = ref.make_params({k: v.shape for k, v in m.state_dict().items()}, seed)
    m.load_state_dict(sd, strict=True)
    return sd


def _runs(g):
    for kind, A in CASES:
        for Tx in (64, 400):
            for B in (1, 2):
                for ti, temp in enumerate((1.0, 0.2)):
                    yield kind, A, Tx, B, temp, f'{kind}{A}_{Tx}_{B}_{ti}'


@pytest.mark.parametrize('kind,A', CASES)
def test_restatement_matches_reference_fixture(kind, A):
    g = _golden()
    sd = _seeded(_model(kind, A), int(g['param_seed']))
    n = 0
    for k2, A2, Tx, B, temp, key in _runs(g):
        if (k2, A2) != (kind, A):
            continue
        batch = ref.make_batch(B, Tx, A, int(g['input_seed']) + Tx + B, pitch=kind == 'pitch')
        out = ref.forward(sd, batch, g['z_' + key], temp, pitch=kind == 'pitch')
        want = g['out_' + key].double()
        err = float((out[:, ::4] - want).abs().max())
        assert err <= 1e-6 * float(want.abs().max()), (key, err)           # float32 storage of a float64 run
        n += 1
    assert n == 8


@pytest.mark.parametrize('kind,A', CASES)
def test_state_dict_keys_and_shapes_match_reference(kind, A):
    g = _golden()
    m = _model(kind, A)
    sd = m.state_dict()
    assert list(sd.keys()) == list(g[f'keys_{kind}{A}'])
    assert [','.join(map(str, v.shape)) for v in sd.values()] == list(g[f'shapes_{kind}{A}'])
    m2 = _model(kind, A)
    m2.load_state_dict(ref.make_params({k: v.shape for k, v in sd.items()}, 3), strict=True)


def test_pitch_model_at_mfcc_width_and_eye_amp():
    m = PitchContourVAEModel({'use_mouth_amp_embed': True, 'use_eye_amp_embed': True}, audio_in_dim=13)
    sd = m.state_dict()
    assert sd['mel_encoder.0.weight'].shape == (128, 13, 3) and sd['cond_proj.weight'].shape == (128, 640)
    assert 'eye_amp_embed' in sd and 'vae.encoder.wn.in_layers.7.weight_v' in sd and 'vae.prior_flow.flows.6.post.weight' in sd
    assert 'vae.prior_flow.flows.1.pre.weight' not in sd                      # the Flips hold no parameters
    assert 'vae.prior_flow' not in {k.rsplit('.', 5)[0] for k in VAEModel(use_prior_flow=False).state_dict()}


@pytest.mark.parametrize('kind,A,hp', [('pitch', 1024, ref.HP_PITCH), ('pitch', 13, {'use_mouth_amp_embed': True, 'use_eye_amp_embed': True}),
                                       ('pitch', 1024, {}), ('vae', 1024, None), ('vae', 13, None)])
def test_folds_match_unfolded_restatement(kind, A, hp):
    """fold_weights (what the kernels run) against the network as the reference writes it, both in float64."""
    m = _model(kind, A, hp)
    sd = _seeded(m, 4)
    P = a2m.fold_weights(m)
    for B, Tx in ((1, 64), (2, 96)):
        batch = ref.make_batch(B, Tx, A, seed=Tx, pitch=kind == 'pitch')
        if kind == 'pitch':
            batch['eye_amp'] = torch.full((B, 1), 0.3)
        z = torch.randn(B, 16, Tx // 8, generator=torch.Generator().manual_seed(B))
        for temp in (0.0, 0.7):
            want = ref.forward(sd, batch, z, temp, pitch=kind == 'pitch', hp=hp or {})
            got = ref.forward_folded(P, batch, z, temp, pitch=kind == 'pitch', hp=hp or {})
            assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max())


def test_weight_norm_and_bn_folds():
    m = VAEModel()
    _seeded(m, 2)
    conv = m.vae.decoder.wn.in_layers[1]
    want = torch._weight_norm(conv.weight_v.double(), conv.weight_g.double(), 0)
    assert torch.allclose(a2m.wn_weight(conv), want, rtol=1e-14, atol=0)
    w, b = a2m.fold_conv_bn(m.mel_encoder[0].weight, m.mel_encoder[1])
    x = torch.randn(2, 1024, 9, dtype=torch.float64)
    bn = m.mel_encoder[1].double().eval()
    ref_y = bn(torch.nn.functional.conv1d(x, m.mel_encoder[0].weight.double(), padding=1))
    assert torch.allclose(torch.nn.functional.conv1d(x, w, b, padding=1), ref_y, rtol=1e-12, atol=1e-12)


def test_gate_pairing_and_wn_pack():
    H, k = 64, 3
    w_in = torch.randn(2 * H, H, k, dtype=torch.float64)
    w_rs = torch.randn(2 * H, H, dtype=torch.float64)
    steps = a2m.pack_wn_layer(w_in, w_rs)
    NC = H // 32
    assert steps.shape == (NC * k * NC + (2 * H // 64) * NC, 2, 64, 32) and steps.dtype == torch.float16
    val = (steps[:, 0].double() + steps[:, 1].double()) / 1024
    # step (j, tap, c), row 2m = tanh row 32 j + m, row 2m + 1 = sigmoid row H + 32 j + m
    j, tap, c, m = 1, 2, 1, 5
    s = (j * k + tap) * NC + c
    assert torch.allclose(val[s, 2 * m], w_in[32 * j + m, 32 * c:32 * c + 32, tap], rtol=2 ** -20)
    assert torch.allclose(val[s, 2 * m + 1], w_in[H + 32 * j + m, 32 * c:32 * c + 32, tap], rtol=2 ** -20)
    n = 1
    assert torch.allclose(val[NC * k * NC + n * NC + c], w_rs[64 * n:64 * n + 64, 32 * c:32 * c + 32], rtol=2 ** -20)


def test_noise_draw_matches_reference_draw():
    g = _golden()
    m = _model('pitch', 1024)
    for ti in (0, 1):
        for Tx, B in ((64, 1), (400, 2)):
            torch.manual_seed(int(g['noise_seed']) + ti)
            z = m.vae.prior_dist.sample([B, 16, Tx // 8])
            assert torch.equal(z, g[f'z_pitch1024_{Tx}_{B}_{ti}'])


def test_f0_to_coarse_restated():
    f0 = torch.cat([torch.linspace(-700.0, 2000.0, 50001), torch.tensor([0.0, 50.0, 1100.0, 1e6])])
    got = a2m.f0_to_coarse(f0.clone())
    assert torch.equal(got, ref.f0_to_coarse_ref(f0.clone()))
    assert int(got.min()) == 1 and int(got.max()) == 255
    if REF_ROOT:
        ref.reference_classes(REF_ROOT)
        from utils.commons.pitch_utils import f0_to_coarse
        assert torch.equal(got, f0_to_coarse(f0.clone()))


def test_rejected_configurations():
    with pytest.raises(NotImplementedError, match='sqz_prior'):
        VAEModel(sqz_prior=True)
    with pytest.raises(NotImplementedError, match='in_out_dim'):
        PitchContourVAEModel({}, in_out_dim=71)
    with pytest.raises(NotImplementedError, match='audio_in_dim'):
        VAEModel(audio_in_dim=80)
    m = _model('pitch', 1024)
    batch = ref.make_batch(1, 64, 1024, seed=1)
    with pytest.raises(NotImplementedError, match='train'):
        m(batch, {}, train=True)
    with pytest.raises(RuntimeError, match='CUDA'):                            # CPU inputs
        m(batch, {})
    b = ref.make_batch(1, 60, 1024, seed=1)
    with pytest.raises(ValueError, match='multiple of 8'):
        m(b, {})
    b = dict(batch)
    b['f0'] = batch['f0'][:, :32]
    with pytest.raises(ValueError, match='f0'):
        m(b, {})
    b = dict(batch)
    b['audio'] = torch.zeros(1, 64, 13)
    with pytest.raises(ValueError, match='audio'):
        m(b, {})
    b = dict(batch)
    b['y_mask'] = torch.ones(1, 64)
    with pytest.raises(ValueError, match='y_mask'):
        m(b, {})
    with pytest.raises(ValueError, match='z'):
        m(batch, {}, z=torch.zeros(1, 16, 9))
