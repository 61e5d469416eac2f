"""HuBERT host side: the float64 restatement against the reference's extract_hubert (fixture), the folds, the frame / segment rule,
state_dict parity, loading, and every rejected configuration and input.  No GPU needed."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import hubert_reference as hr  # noqa: E402
from real3dportrait_b200 import hubert as hb  # noqa: E402
from real3dportrait_b200 import HubertModel, get_hubert_from_16k_speech, hubert_frames  # noqa: E402


def small_cfg(g):
    return {k[7:]: (tuple(v.tolist()) if v.ndim else v.item()) for k, v in g.items() if k.startswith('config.')}


def load_fixture():
    z = np.load(os.path.join(ROOT, 'tests', 'golden', 'hubert_small.npz'))
    return {k: (torch.from_numpy(z[k]) if z[k].dtype.kind in 'fiub' and z[k].ndim else z[k]) for k in z.files}


@pytest.fixture(scope='module')
def fx():
    return load_fixture()


@pytest.fixture(scope='module')
def small(fx):
    cfg = small_cfg(fx)
    m = HubertModel(cfg)
    sd = hr.formula_params({k: tuple(v.shape) for k, v in m.state_dict().items()})
    m.load_state_dict({k: v.float() for k, v in sd.items()}, strict=True)
    return cfg, m, sd


@pytest.mark.parametrize('L', [400, 4000, 330000])
def test_restatement_matches_reference(fx, small, L):
    cfg, _, sd = small
    ref = fx[f'hubert_{L}'].double()
    got = hr.get_hubert(sd, cfg, hr.wave(L))
    assert got.shape == ref.shape
    assert float((got - ref).abs().max()) <= 1e-5 * float(ref.abs().max())


@pytest.mark.parametrize('L', [4000, 330000])
def test_folded_matches_unfolded(small, L):
    cfg, m, sd = small
    m64 = HubertModel(cfg).double()
    m64.load_state_dict(sd, strict=True)
    x = hr.normalise(hr.wave(L))
    T = hubert_frames(L)
    segs = hb._segments(T)
    ref = torch.cat([hr.forward_unfolded(sd, cfg, x[320000 * i:320000 * i + 320 * (n - 1) + 400]) for i, n in enumerate(segs)])
    got = hr.forward_folded(hb.fold_weights(m64), cfg, x[:320 * (T - 1) + 400], segs)
    assert float((got - ref).abs().max()) <= 1e-12 * float(ref.abs().max())


def test_frame_and_segment_rule(fx):
    for L, T in zip(fx['T_lens'].tolist(), fx['T_ref'].tolist()):
        assert hubert_frames(L) == T == hr.frames(L)
        segs = hb._segments(T)
        assert sum(segs) == T and all(s == 1000 for s in segs[:-1]) and 1 <= segs[-1] <= 1000
    assert hubert_frames(400) == 1 and hubert_frames(719) == 1 and hubert_frames(720) == 2
    with pytest.raises(ValueError):
        hubert_frames(399)


def test_large_key_parity(fx):
    cfg = dict(hr_large_cfg())
    sd = HubertModel(cfg).state_dict()
    keys = [str(k) for k in fx['large_keys'].tolist()]
    shapes = [str(s) for s in fx['large_shapes'].tolist()]
    assert list(sd.keys()) == keys
    assert [','.join(map(str, v.shape)) for v in sd.values()] == shapes


def hr_large_cfg():
    return dict(conv_dim=(512,) * 7, hidden_size=1024, num_attention_heads=16, intermediate_size=4096, num_hidden_layers=24,
                num_conv_pos_embeddings=128, num_conv_pos_embedding_groups=16, feat_extract_norm='layer', do_stable_layer_norm=True,
                conv_bias=True)


def test_both_weight_norm_forms(small):
    cfg, m, sd = small
    old = dict(sd)
    p = 'encoder.pos_conv_embed.conv.'
    old[p + 'weight_g'] = old.pop(p + 'parametrizations.weight.original0')
    old[p + 'weight_v'] = old.pop(p + 'parametrizations.weight.original1')
    m2 = HubertModel(cfg)
    m2.load_state_dict(old, strict=True)
    w1, w2 = hb.pos_conv_weight(m.encoder.pos_conv_embed), hb.pos_conv_weight(m2.encoder.pos_conv_embed)
    assert torch.equal(w1, w2)


def test_pos_conv_weight_norm_matches_torch(small):
    _, m, _ = small
    # parametrizations.weight_norm(dim=2) recomputes the weight itself: the fold must agree with it
    w_torch = m.encoder.pos_conv_embed.conv.weight.double()
    assert float((hb.pos_conv_weight(m.encoder.pos_conv_embed) - w_torch).abs().max()) < 1e-6


def test_from_pretrained_transformers_snapshot(tmp_path, small):
    transformers = pytest.importorskip('transformers')
    cfg, _, sd = small
    ref = transformers.HubertModel(transformers.HubertConfig(**cfg))
    ref.load_state_dict({k: v.float() for k, v in sd.items()}, strict=True)
    ref.save_pretrained(str(tmp_path / 'plain'))
    ctc = transformers.HubertForCTC(transformers.HubertConfig(**cfg, vocab_size=32))
    ctc.hubert.load_state_dict({k: v.float() for k, v in sd.items()}, strict=True)
    ctc.save_pretrained(str(tmp_path / 'ctc'))
    for d in ('plain', 'ctc'):
        m = HubertModel.from_pretrained(str(tmp_path / d))
        got = m.state_dict()
        for k, v in ref.state_dict().items():
            assert torch.equal(got[k], v), (d, k)


@pytest.mark.parametrize('change', [
    dict(feat_extract_norm='group'), dict(do_stable_layer_norm=False), dict(hidden_act='relu'), dict(feat_extract_activation='relu'),
    dict(conv_pos_batch_norm=True), dict(conv_kernel=(10, 3, 3, 3, 3, 3, 2)), dict(conv_stride=(5, 2, 2, 2, 2, 2, 1)),
    dict(conv_dim=(32,) * 6 + (64,)), dict(conv_dim=(48,) * 7), dict(conv_dim=(1024,) * 7), dict(num_attention_heads=4),
    dict(num_conv_pos_embedding_groups=4), dict(num_conv_pos_embeddings=64), dict(intermediate_size=200)])
def test_rejected_configs(fx, change):
    with pytest.raises(NotImplementedError):
        HubertModel(dict(small_cfg(fx), **change))


def test_rejected_inputs(small):
    cfg, m, _ = small
    with pytest.raises(NotImplementedError):
        m.train()
    with pytest.raises(RuntimeError):
        m(torch.zeros(1, 4000))
    with pytest.raises(NotImplementedError):
        m(torch.zeros(1, 4000), attention_mask=torch.ones(1, 4000))
    with pytest.raises(NotImplementedError):
        m(torch.zeros(1, 4000), output_hidden_states=True)
    with pytest.raises(NotImplementedError):
        m(torch.zeros(1, 4000), output_attentions=True)
    with pytest.raises(RuntimeError):
        get_hubert_from_16k_speech(np.zeros(4000, np.float32), m)
    with pytest.raises(ValueError):
        get_hubert_from_16k_speech(np.zeros(399, np.float32), m)
    with pytest.raises(ValueError):
        get_hubert_from_16k_speech(np.zeros((4000, 2, 2), np.float32), m)


def test_fp16_range_checks(small):
    cfg, m, sd = small
    P = hb.fold_weights(m)
    bound = hb.check_pos_conv_range(P, True)
    # the bound holds for standardised rows at their extreme (one-hot-like rows reach |z|_2 = sqrt(C) in one direction)
    z = torch.randn(4096, P['proj'][0].shape[1], dtype=torch.float64)
    z = (z - z.mean(1, keepdim=True)) / z.std(1, unbiased=False, keepdim=True)
    assert float((z @ P['proj'][0].t() + P['proj'][1]).abs().max()) <= bound
    big = {'proj': (P['proj'][0] * 1e5, P['proj'][1]), 'conv': P['conv']}
    with pytest.raises(ValueError):
        hb.check_pos_conv_range(big, True)
    with pytest.raises(ValueError):
        hb.pack_split(torch.full((2, 64), 64.0, dtype=torch.float64))
    hb.pack_split(torch.full((2, 64), 63.9, dtype=torch.float64))
