"""CPU-side checks: the C-ABI library loads and exports every declared symbol, the host mirror keeps the reference's
state_dict layout, and the product path refuses to run without CUDA (no silent fallback)."""
import os

import pytest
import torch

import real3dportrait_b200 as r3
from real3dportrait_b200 import _capi, synthetic as syn, build as r3build


def test_library_builds_and_exports_every_declared_symbol():
    path = r3build.build()
    assert os.path.exists(path)
    L = _capi.lib()
    declared = _capi.declared_symbols()
    assert len(declared) >= 17
    missing = [s for s in declared if not hasattr(L, s)]
    assert not missing, missing
    assert set(declared) == set(_capi._SIGNATURES), set(declared) ^ set(_capi._SIGNATURES)
    assert L.r3dp_abi_version() == 3


def test_state_dict_layout_matches_reference_checkpoints():
    # key list == what the REFERENCE modules accepted with strict=True in tests/golden/make_golden.py
    head = r3.RenderHead()
    want = {'decoder.' + k for k in syn.make_decoder_params()} | {'superresolution.' + k for k in syn.make_sr_params()}
    assert set(head.state_dict().keys()) == want
    sd = {'decoder.' + k: v for k, v in syn.make_decoder_params().items()}
    sd.update({'superresolution.' + k: v for k, v in syn.make_sr_params().items()})
    head.load_state_dict(sd, strict=True)
    assert sum(p.numel() for p in head.superresolution.parameters()) == 1649578 - 0  # SURVEY.md §8d: 1 649 578 SR params
    assert sum(p.numel() for p in head.decoder.parameters()) == 4257


def test_no_cpu_fallback():
    with pytest.raises(RuntimeError, match='CUDA tensors only'):
        r3.RaySampler()(torch.eye(4)[None], torch.eye(3)[None], 4)
    planes = torch.zeros(1, 3, 32, 4, 4)
    with pytest.raises(RuntimeError, match='CUDA tensors only'):
        r3.planes_to_channels_last(planes)


def test_unsupported_options_raise():
    ren = r3.ImportanceRenderer()
    dec = r3.OSGDecoder(32, {'decoder_lr_mul': 1, 'decoder_output_dim': 32})
    opts = dict(syn.RENDERING_OPTIONS, ray_start=2.0, ray_end=3.0)
    with pytest.raises(NotImplementedError):
        ren(torch.zeros(1, 3, 32, 4, 4), dec, torch.zeros(1, 4, 3), torch.zeros(1, 4, 3), opts)
    with pytest.raises(NotImplementedError):
        r3.ImportanceRenderer(hp={'triplane_feature_type': 'trigrid_v2', 'enable_rescale_plane_regulation': False})


def test_synthetic_cameras_hit_the_box():
    from oracle import real3d_oracle as orc
    cam = syn.make_cameras(8, seed=1)
    c2w, K = syn.split_camera(cam)
    o, d = orc.gen_rays(c2w, K, 64)
    _, _, valid = orc.auto_limits(o, d, 1.0)
    assert bool(valid.all())


def test_torso_head_state_dict_layout():
    """SuperresolutionHybrid8XDC_Warp (minus the caller-supplied torso_model child) has the reference's keys: the REFERENCE class accepted
    exactly this dict with strict=True in tests/golden/make_golden.py::warp_case."""
    m = r3.SuperresolutionHybrid8XDC_Warp(channels=32, img_resolution=512, sr_num_fp16_res=0, sr_antialias=True, hp=syn.WARP_HPARAMS)
    want = set(syn.make_sr_warp_params())
    assert set(m.state_dict().keys()) == want, set(m.state_dict().keys()) ^ want
    m.load_state_dict(syn.make_sr_warp_params(), strict=True)
    assert sum(p.numel() for p in m.parameters()) == 6532912          # probe of the reference class (without torso_model)
    # the other fuse modes of the reference: v1 has no head/torso fusing children (sr_with_ref.py:36-55), v3 has them all; unknown modes raise as in the reference
    for mode in ('v1', 'v3'):
        mm = r3.SuperresolutionHybrid8XDC_Warp(channels=32, img_resolution=512, sr_num_fp16_res=0, sr_antialias=True,
                                               hp=dict(syn.WARP_HPARAMS, htbsr_head_weight_fuse_mode=mode))
        assert set(mm.state_dict().keys()) == set(syn.make_sr_warp_params(fuse_mode=mode))
    assert not any(k.startswith('head_torso') for k in syn.make_sr_warp_params(fuse_mode='v1'))
    with pytest.raises(NotImplementedError):
        r3.SuperresolutionHybrid8XDC_Warp(channels=32, img_resolution=512, sr_num_fp16_res=0, sr_antialias=True,
                                          hp=dict(syn.WARP_HPARAMS, htbsr_head_weight_fuse_mode='v4'))


def test_gpu_local_cpus_is_a_noop_without_a_gpu_and_restores_affinity():
    """engine.gpu_local_cpus(): anything unexpected (no CUDA device, no sysfs entry) must leave the CPU affinity untouched."""
    import os
    from real3dportrait_b200 import engine
    before = os.sched_getaffinity(0)
    with engine.gpu_local_cpus(0):
        inside = os.sched_getaffinity(0)
    assert os.sched_getaffinity(0) == before and inside <= before


def test_bench_clock_sampler_reports_without_nvml():
    """bench.ClockSampler must come up and summarise even when neither NVML nor nvidia-smi can be reached (CPU container)."""
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location('bench_mod', os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'bench.py'))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    s = bench.ClockSampler(0)
    s.start()
    out = s.summary()
    assert set(out) >= {'sm_mhz', 'sm_max_mhz', 'reasons', 'samples', 'source'} and out['source'] in ('nvml', 'nvidia-smi')
    assert bench.host_threads() >= 1
