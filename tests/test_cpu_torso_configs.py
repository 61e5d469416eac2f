"""CPU checks of the torso head's other reference configurations: weight_fuse=False (cat[x, x_torso, x_bg] -> fuse_fg_bg_convs(768 -> 64) -> block1
without a skip image, sr_with_ref.py:57-58,158-161) and torso_model_version 'v1' (the warper takes no head weights image, sr_with_ref.py:84-85).
The oracle against the reference class's fixture, the state_dict layout, the warper's argument list and the new C entry points."""
import os

import pytest
import torch

import real3dportrait_b200 as r3
import torso_config_oracle as tco
from oracle import real3d_oracle as orc
from real3dportrait_b200 import _capi, engine, synthetic as syn

CPU = torch.device('cpu')
NOFUSE = dict(syn.WARP_HPARAMS, weight_fuse=False)


def _maxdiff(a, b):
    return float((a.float() - b.float()).abs().max())


def _head(hp, torso_model=None):
    return r3.SuperresolutionHybrid8XDC_Warp(channels=32, img_resolution=512, sr_num_fp16_res=0, sr_antialias=True, hp=hp, torso_model=torso_model)


def test_oracle_weight_fuse_false_vs_reference(golden):
    """The oracle's weight_fuse=False branch against the reference class run with the stub torso model (fixture sr_warp_nofuse)."""
    g = golden('render_full48')
    fimg, wimg = orc.feature_image(g['rgb'], 64), orc.feature_image(g['wsum'], 64)
    inp = syn.make_warp_inputs(1, seed=7)
    img, _ = tco.superres_warp(fimg[:, :3], fimg, torch.ones(1, 14, 512), inp['ref_torso_rgb'], inp['ref_bg_rgb'], wimg, inp['segmap'],
                               inp['kp_s'], inp['kp_d'], syn.make_sr_warp_params(seed=6, weight_fuse=False), syn.StubTorsoModel(), weight_fuse=False)
    img, ref = img[..., ::2, ::2], golden('sr_warp_nofuse')['image_s2']
    assert _maxdiff(img, ref) < 2e-5, _maxdiff(img, ref)                       # fp32 re-association noise between two CPU implementations


def test_weight_fuse_false_state_dict_layout():
    """The reference class accepted make_sr_warp_params(weight_fuse=False) with strict=True (tests/golden/make_golden_torso_configs.py): no head_torso_* children and a
    768-input fuse_fg_bg_convs.0, whatever the fuse mode.  Every other key keeps its weight_fuse=True value."""
    want = syn.make_sr_warp_params(weight_fuse=False)
    assert want['fuse_fg_bg_convs.0.weight'].shape == (64, 768, 1, 1) and not any(k.startswith('head_torso') for k in want)
    base = syn.make_sr_warp_params()
    assert all(torch.equal(v, base[k]) for k, v in want.items() if not k.startswith('fuse_fg_bg_convs.0.'))
    for mode in ('v1', 'v2', 'v3', 'v4'):                                       # the reference ignores the fuse mode without weight_fuse
        m = _head(dict(NOFUSE, htbsr_head_weight_fuse_mode=mode))
        sd = m.state_dict()
        assert set(sd) == set(want), set(sd) ^ set(want)
        assert all(sd[k].shape == v.shape for k, v in want.items())
        m.load_state_dict(want, strict=True)
        assert m.fuse_mode is None and not hasattr(m, 'fuse_head_torso_convs')
    with pytest.raises(NotImplementedError):                                    # an unknown fuse mode still raises when it is used
        _head(dict(syn.WARP_HPARAMS, htbsr_head_weight_fuse_mode='v4'))
    with pytest.raises(NotImplementedError):
        _head(dict(syn.WARP_HPARAMS, torso_model_version='v3'))


def test_torso_v1_state_dict_and_warper_argument_list():
    """torso_model_version 'v1' changes only the warper call: the same children, and run_torso() passes model.py's argument list."""
    for wf in (True, False):
        m = _head(dict(syn.WARP_HPARAMS, torso_model_version='v1', weight_fuse=wf), torso_model=syn.StubTorsoModelV1())
        m.load_state_dict(syn.make_sr_warp_params(weight_fuse=wf), strict=True)
    inp = syn.make_warp_inputs(1, seed=7)
    t256, rgb256, w256 = orc.aa_down2(inp['ref_torso_rgb']), torch.rand(1, 3, 256, 256), torch.rand(1, 1, 256, 256)
    st = {'torso_args': (t256, inp['segmap'], inp['kp_s'], inp['kp_d'], rgb256, w256), 'target_torso_mask': None}
    stub = syn.StubTorsoModelV1()
    rgb_torso, ret = _head(dict(syn.WARP_HPARAMS, torso_model_version='v1'), torso_model=stub).run_torso(st)
    assert stub.calls == 1 and rgb_torso.shape == (1, 3, 256, 256) and ret['deformed_torso_hid'].shape == (1, 64, 256, 256)
    with pytest.raises(TypeError):                                              # a v1 warper cannot take the v2 argument list, nor the reverse
        _head(syn.WARP_HPARAMS, torso_model=syn.StubTorsoModelV1()).run_torso(st)
    with pytest.raises(TypeError):
        _head(dict(syn.WARP_HPARAMS, torso_model_version='v1'), torso_model=syn.StubTorsoModel()).run_torso(st)


def test_oracle_torso_v1_calls_the_v1_warper():
    """The oracle's torso_version='v1' passes model.py's argument list; with a v2 warper that returns the same outputs the image is the same.
    Covered for weight_fuse=False and for the released fuse mode v2."""
    g = torch.Generator().manual_seed(3)
    fimg, wimg = torch.rand(1, 32, 32, 32, generator=g) * 2 - 1, torch.rand(1, 1, 32, 32, generator=g)
    inp = syn.make_warp_inputs(1, seed=7)
    for wf in (False, True):
        p = syn.make_sr_warp_params(seed=6, weight_fuse=wf)
        v1 = syn.StubTorsoModelV1()
        as_v2 = lambda t, s, ks, kd, h, w, **kw: v1(t, s, ks, kd, h, **kw)      # noqa: E731
        args = (fimg[:, :3], fimg, torch.ones(1, 14, 512), inp['ref_torso_rgb'], inp['ref_bg_rgb'], wimg, inp['segmap'], inp['kp_s'], inp['kp_d'], p)
        a, _ = tco.superres_warp(*args, v1, weight_fuse=wf, torso_version='v1')
        b, _ = tco.superres_warp(*args, as_v2, weight_fuse=wf)
        assert v1.calls == 2 and torch.equal(a, b)


def test_engine_constructs_both_configurations():
    for hp in (NOFUSE, dict(NOFUSE, htbsr_head_weight_fuse_mode='v3'), dict(syn.WARP_HPARAMS, torso_model_version='v1')):
        warper = syn.StubTorsoModelV1() if hp['torso_model_version'] == 'v1' else syn.StubTorsoModel()
        eng = engine.FrameEngine(batch=2, device=CPU, hp=dict(hp, num_samples_fine=48), torso_model=warper, out_uint8=True)
        assert eng.torso and eng.eager_reason is None                          # weight_fuse=False ignores fuse mode v3: its steps are captured


def test_cat3_entry_points_are_declared_typed_and_exported():
    for name in ('r3dp_sr_cat3', 'r3dp_sr_tcx_cat3'):
        assert name in _capi.declared_symbols()
        restype, argtypes = _capi._SIGNATURES[name]
        assert restype is _capi._I and len(argtypes) == 15
        if os.path.exists(_capi.LIB_PATH):                                      # built library (python -m real3dportrait_b200.build)
            assert hasattr(_capi.lib(), name)
