"""CPU checks of the torso head in FrameEngine: the one-launch input entry point is declared, typed and exported; the engine validates
uint8 frames against the head's effective sr_mode and rejects steps without clip constants and kp_d on a plain engine."""
import os

import pytest
import torch

from real3dportrait_b200 import _capi, engine, synthetic as syn

CPU = torch.device('cpu')


def test_warp_input_entry_point_is_declared_typed_and_exported():
    assert 'r3dp_sr_warp_input' in _capi.declared_symbols()
    restype, argtypes = _capi._SIGNATURES['r3dp_sr_warp_input']
    assert restype is _capi._I and len(argtypes) == 13
    if os.path.exists(_capi.LIB_PATH):                                          # built library (python -m real3dportrait_b200.build)
        assert hasattr(_capi.lib(), 'r3dp_sr_warp_input')


def _torso_engine(**kw):
    return engine.FrameEngine(batch=2, device=CPU, hp=dict(syn.WARP_HPARAMS, num_samples_fine=48), torso_model=syn.StubTorsoModel(), **kw)


def test_uint8_frames_are_validated_against_the_effective_mode():
    # a torso head maps sr_mode='fp32' to 'tc', whose last epilogue writes the uint8 frames
    eng = _torso_engine(sr_mode='fp32', out_uint8=True)
    assert eng.torso and eng.head.superresolution.sr_mode == 'tc' and eng.frame_dtype() == torch.uint8
    with pytest.raises(NotImplementedError):                                    # the plain head keeps its fp32 SR
        engine.FrameEngine(batch=2, sr_mode='fp32', device=CPU, out_uint8=True)


def test_step_needs_begin_clip_and_kp_d_belongs_to_the_torso_head():
    planes, cams = torch.zeros(2, 3, 32, 8, 8), torch.zeros(2, 25)
    eng = _torso_engine(sr_mode='tc')
    with pytest.raises(RuntimeError, match='begin_clip'):
        eng.step(planes, cams, kp_d=torch.zeros(2, 68, 3))
    with pytest.raises(RuntimeError, match='begin_clip'):
        eng.prepare([(planes, cams, torch.zeros(2, 4096, 48, 1), None, torch.zeros(2, 68, 3))])
    plain = engine.FrameEngine(batch=2, sr_mode='tc', device=CPU)
    with pytest.raises(ValueError, match='kp_d'):
        plain.step(planes, cams, kp_d=torch.zeros(2, 68, 3))
    with pytest.raises(ValueError, match='torso'):
        plain.begin_clip(torch.zeros(1, 3, 512, 512), torch.zeros(1, 3, 512, 512), torch.zeros(1, 6, 512, 512), torch.zeros(1, 68, 3))


def test_fuse_mode_v3_runs_eagerly():
    eng = engine.FrameEngine(batch=2, device=CPU, hp=dict(syn.WARP_HPARAMS, htbsr_head_weight_fuse_mode='v3'), torso_model=syn.StubTorsoModel())
    assert eng.eager_reason is not None
    assert _torso_engine().eager_reason is None
