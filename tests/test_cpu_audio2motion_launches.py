"""The audio2secc VAE's launch plan and the end-to-end bar, on the host.

* launch_plan's invariants: 42 launches for the released pitch config (1 input pack, 18 r3dp_mf_conv3d, 20 WaveNet layers, split, latent,
  store), 39 for VAEModel at A = 1024 and 13, the same plan whatever the amplitude flags; every conv reads whole 32-channel chunks, packs
  its couts to its tile, keeps the lo halves past the channels it reads and writes, and fits its output rows.
* The discrimination check: forward_folded with every GEMM / conv operand rounded as the kernels read it (split fp16) sits at least 10x
  below E2E_BAR and with every launch reading fp16 operands at least 3x above it; with any one launch of either class reading its hi
  halves alone it sits above SITE_MARGIN x E2E_BAR.  The library's own fp32 accumulation uses most of the bar (E2E_BAR's comment), so
  the end-to-end test alone cannot promise 3x per launch: the per-launch rows of tests/test_gpu_audio2motion_launches.py each assert
  that their hi-only operands break their own bar."""
import pytest
import torch

import audio2motion_reference as ref
from real3dportrait_b200 import PitchContourVAEModel, VAEModel
from real3dportrait_b200 import audio2motion as a2m

CASES = [('pitch', 1024), ('vae', 1024), ('vae', 13)]
SITE_MARGIN = 1.25


def _counts(plan):
    out = {}
    for _, fn, _ in plan:
        out[fn] = out.get(fn, 0) + 1
    return out


@pytest.mark.parametrize('kind,A', CASES)
@pytest.mark.parametrize('B,Tx', [(1, 8), (2, 400), (3, 1032), (1, 30000)])
def test_plan_counts_and_conv_arguments(kind, A, B, Tx):
    plan = ref.launch_plan(kind, A, B, Tx)
    pitch = kind == 'pitch'
    assert len(plan) == (42 if pitch else 39)
    assert _counts(plan) == {'r3dp_a2m_input': 1, 'r3dp_mf_conv3d': 18 if pitch else 15, 'r3dp_a2m_wn_layer': 20, 'r3dp_a2m_split': 1,
                             'r3dp_a2m_latent': 1, 'r3dp_a2m_store': 1}
    assert len({tag for tag, _, _ in plan}) == len(plan)
    T, T4 = Tx // 2, Tx // 8
    for tag, fn, a in plan:
        if fn != 'r3dp_mf_conv3d':
            continue
        xs, xlo, cin, N, D, H, W, kd, kh, kw, up, O, cop, relu, ys, yc0, ylo, f32, split = a
        assert cin % 32 == 0 and split == 1 and up == 0 and D == H == kd == kh == 1 and kw in (1, 3), tag
        tile = 16 if O <= 16 else 32 if O <= 32 else 64 if O <= 64 else 128     # the kernel's cout tile
        assert cop == ref.cop_of(O) and cop % tile == 0 and cop - O < tile, tag
        assert xlo >= cin and xs >= xlo + cin, tag                       # the lo halves sit past every channel read
        if f32:
            assert yc0 + O <= ys, tag
        else:
            assert ylo >= yc0 + O and ys >= ylo + yc0 + O, tag            # the lo halves of the slice sit past the hi halves
        assert (N, W) == ((B, T4 if tag == 'g_pre' else T) if kw == 3 else (1, N * W)), tag
        assert N * W in (B * T, B * T4), tag
        assert relu == (2 if tag in ('enc1', 'penc1') else 0), tag


def test_plan_independent_of_amplitude_flags():
    base = ref.launch_plan('pitch', 1024, 2, 400)
    for hp in ({}, {'use_mouth_amp_embed': True, 'use_eye_amp_embed': True}, {'use_eye_amp_embed': True}):
        assert ref.launch_plan('pitch', 1024, 2, 400, hp) == base
        assert ref.launch_plan('pitch', 13, 2, 400, hp)[1:] != base[1:]     # the feature width shows in enc1 and penc1


def test_plan_tags_cover_folded_forward():
    """Every GEMM / conv launch of the plan is a site of forward_folded and no site is missing from the plan."""
    for kind, A in CASES:
        m = _model(kind, A)
        P = a2m.fold_weights(m)
        batch = ref.make_batch(1, 64, A, seed=1, pitch=kind == 'pitch')
        z = torch.zeros(1, 16, 8)
        out = ref.forward_folded(P, batch, z, 0.2, pitch=kind == 'pitch', operands='split')
        assert torch.isfinite(out).all()
        sites = _sites(kind, A, 1, 64)
        with pytest.raises(AssertionError, match='no launch'):
            ref.forward_folded(P, batch, z, 0.2, pitch=kind == 'pitch', operands='hi', site='split')
        for s in sites:
            ref.forward_folded(P, batch, z, 0.2, pitch=kind == 'pitch', operands='hi', site=s)


def _model(kind, A, seed=11):
    m = PitchContourVAEModel(ref.HP_PITCH, audio_in_dim=A) if kind == 'pitch' else VAEModel(audio_in_dim=A)
    m.load_state_dict(ref.make_params({k: v.shape for k, v in m.state_dict().items()}, seed), strict=True)
    return m


def _sites(kind, A, B, Tx):
    return [tag for tag, fn, _ in ref.launch_plan(kind, A, B, Tx) if fn not in ref.PACK_LAUNCHES]


@pytest.mark.parametrize('kind,A', CASES)
@torch.no_grad()
def test_end_to_end_bar_discriminates_every_launch(kind, A):
    """The released pitch config and VAEModel at both feature widths, seed 11, B = 2, T_x = 400, temperature 0.2: the case of the GPU test."""
    pitch = kind == 'pitch'
    P = a2m.fold_weights(_model(kind, A))
    B, Tx = 2, 400
    batch = ref.make_batch(B, Tx, A, seed=Tx + B, pitch=pitch, mouth_amp=0.45)
    z = torch.randn(B, 16, Tx // 8, generator=torch.Generator().manual_seed(5))
    exact = ref.forward_folded(P, batch, z, 0.2, pitch=pitch)
    scale = float(exact.abs().max())

    def ratio(**k):
        return float((ref.forward_folded(P, batch, z, 0.2, pitch=pitch, **k) - exact).abs().max()) / scale

    split = ratio(operands='split')
    print(f'{kind}{A}: all split {split:.2e} = bar / {ref.E2E_BAR / split:.1f}')
    assert split * 10 <= ref.E2E_BAR
    every = ratio(operands='hi')
    print(f'{kind}{A}: all hi-only {every:.2e} = bar x {every / ref.E2E_BAR:.1f}')
    assert every >= 3 * ref.E2E_BAR
    weak = []
    for site in _sites(kind, A, B, Tx):
        r = ratio(operands='hi', site=site)
        print(f'{kind}{A}: {site} hi-only {r:.2e} = bar x {r / ref.E2E_BAR:.1f}')
        if r < SITE_MARGIN * ref.E2E_BAR:
            weak.append(f'{site}: {r:.2e}')
    assert not weak, 'launches whose lost lo halves the end-to-end bar would not see:\n' + '\n'.join(weak)
