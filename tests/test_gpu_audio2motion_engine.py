"""The reference's audio-driven sequence on the library (INTEGRATION.md): PitchContourVAEModel writes a clip's expression columns straight into
the engine's [id | exp | t | T] rows; the coefficient clip renders frames bit-identical to one fed the same rows built with torch.cat from
forward's output, with and without blink."""
import random

import pytest
import torch

import audio2motion_reference as ref
import secc2plane_reference as sref
import real3dportrait_b200 as r3
from real3dportrait_b200 import engine, synthetic as syn

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
B = 2


@pytest.fixture(scope='module')
def renderer(tmp_path_factory):
    kw = syn.write_bfm_folder(str(tmp_path_factory.mktemp('bfm')), seed=0)
    return r3.SECC_Renderer(512, device=DEV, **kw)


@pytest.fixture(scope='module')
def model():
    m = r3.PitchContourVAEModel(ref.HP_PITCH)
    m.load_state_dict(ref.make_params({k: v.shape for k, v in m.state_dict().items()}, 11), strict=True)
    return m.to(DEV).eval()


def _engine(r, blink):
    bb = r3.SegFormerSECC2PlaneBackbone()
    bb.load_state_dict(sref.make_params({k: v.shape for k, v in bb.state_dict().items()}, 7), strict=True)
    eng = engine.FrameEngine(batch=B, sr_mode='tc', hp={'num_samples_fine': 0}, out_uint8=True, secc2plane=bb.to(DEV).eval(), secc_renderer=r,
                             blink=blink)
    eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_params(seed=5))
    return eng


@pytest.mark.parametrize('blink', [False, True])
@torch.no_grad()
def test_rows_written_in_place_match_rows_from_cat(model, renderer, blink):
    Tx = 16                                                                    # 8 frames: four engine steps of B = 2
    N = Tx // 2
    batch = {k: v.to(DEV) for k, v in ref.make_batch(1, Tx, 1024, seed=21).items()}
    z = torch.randn(1, 16, Tx // 8, generator=torch.Generator().manual_seed(2))
    ident = syn.make_coeffs(1, seed=3)['id'].to(DEV)
    K = 146 if blink else 144
    rows = torch.zeros(N, K, device=DEV)
    rows[:, :80] = ident
    model(batch, {}, train=False, temperature=0.2, z=z, out=rows[:, 80:144])
    exp = model(batch, {}, train=False, temperature=0.2, z=z)[0]
    parts = [ident.expand(N, 80), exp]
    if blink:
        sched = r3.period_blink_schedule(N, rng=random.Random(3)).to(DEV, torch.float32)      # a window from frame 0
        rows[:, 144:] = sched
        parts.append(sched)
    cat = torch.cat(parts, 1)
    assert torch.equal(rows, cat)
    frames = []
    for src in (rows, cat):
        eng = _engine(renderer, blink)
        eng.begin_planes(syn.make_planes(1).to(DEV), coeff_src=src[:1, :144].contiguous())
        out = []
        for s in range(N // B):
            cams = syn.make_cameras(B, seed=40 + s).to(DEV)
            u_c, _ = syn.make_jitter(B, 4096, 48, 0, seed=140 + s)
            out.append(eng.step(None, cams, u_c.to(DEV), coeff=src[s * B:(s + 1) * B].contiguous()).clone())
        frames.append(torch.stack(out))
    assert torch.equal(frames[0], frames[1])
