"""CPU checks of sr_mode='tc_exact' in the torso head and in large_sr: which modes construct, how RenderHead maps sr_mode to the torso head,
and that the split entry points are declared in the header and typed in _capi."""
import pytest

import real3dportrait_b200 as r3
from real3dportrait_b200 import _capi, synthetic as syn

SPLIT_TORSO_SYMBOLS = ('r3dp_sr_tcx_conv_res', 'r3dp_sr_tcx_layer_torgb_noup', 'r3dp_sr_tcx_alpha_cat_ex', 'r3dp_sr_tcx_alpha_mix',
                       'r3dp_sr_tcx_torgb_ex')
SR_KW = dict(channels=32, img_resolution=512, sr_num_fp16_res=0, sr_antialias=True)


@pytest.mark.parametrize('fuse', ['v1', 'v2', 'v3'])
def test_torso_head_constructs_in_tc_exact_and_rejects_fp32(fuse):
    hp = dict(syn.WARP_HPARAMS, htbsr_head_weight_fuse_mode=fuse)
    m = r3.SuperresolutionHybrid8XDC_Warp(hp=hp, sr_mode='tc_exact', **SR_KW)
    assert m.sr_mode == 'tc_exact' and m._split
    assert set(m.state_dict().keys()) == set(syn.make_sr_warp_params(fuse_mode=fuse))
    with pytest.raises(NotImplementedError):
        r3.SuperresolutionHybrid8XDC_Warp(hp=hp, sr_mode='fp32', **SR_KW)


def test_large_sr_constructs_in_tc_exact_and_rejects_fp32():
    sr = r3.SuperresolutionHybrid8XDC(large_sr=True, sr_mode='tc_exact', resblocks_in_large_sr=2, **SR_KW)
    assert sr.sr_mode == 'tc_exact'
    sr.load_state_dict(syn.make_sr_large_params(seed=8, n_res=2), strict=True)
    with pytest.raises(NotImplementedError):
        r3.SuperresolutionHybrid8XDC(large_sr=True, sr_mode='fp32', resblocks_in_large_sr=2, **SR_KW)


@pytest.mark.parametrize('sr_mode,torso_mode', [('tc_exact', 'tc_exact'), ('tc', 'tc'), ('fp32', 'tc'), (None, 'tc')])
def test_render_head_maps_sr_mode_to_the_torso_head(sr_mode, torso_mode):
    kw = {} if sr_mode is None else {'sr_mode': sr_mode}
    head = r3.RenderHead(hp=syn.WARP_HPARAMS, torso_model=syn.StubTorsoModel(), **kw)
    assert isinstance(head.superresolution, r3.SuperresolutionHybrid8XDC_Warp)
    assert head.superresolution.sr_mode == torso_mode


def test_split_torso_entry_points_are_declared_and_typed():
    declared = set(_capi.declared_symbols())
    for name in SPLIT_TORSO_SYMBOLS:
        assert name in declared and name in _capi._SIGNATURES, name
        twin = name.replace('r3dp_sr_tcx_', 'r3dp_sr_tc_')
        if twin not in _capi._SIGNATURES:                                          # r3dp_sr_alpha_cat_ex, r3dp_sr_alpha_mix
            twin = name.replace('r3dp_sr_tcx_', 'r3dp_sr_')
        assert _capi._SIGNATURES[name] == _capi._SIGNATURES[twin], (name, twin)      # same arguments as the fp16 twin
