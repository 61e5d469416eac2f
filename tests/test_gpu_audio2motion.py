"""PitchContourVAEModel / VAEModel forward on the GPU against the float64 restatement (tests/audio2motion_reference.py, itself pinned to the
reference's own outputs): T_x from 8 to 30000 (ten minutes of audio at 50 Hz features), temperatures 0 and 0.2, mouth_amp 0.45, blink
ids on, a masked tail, and `out=` into a strided slice of [id | exp | t | T] rows with the other columns untouched.  End-to-end bar:
max |err| <= E2E_BAR max |exp| = 2e-5 max |exp| (audio2motion_reference.E2E_BAR; DESIGN.md, "Audio-to-motion"): the float64 emulation of
split operands sits more than 10x below it, with any one launch reading its fp16 hi halves alone above it (tests/
test_cpu_audio2motion_launches.py).  Also: the seeded draw, the rejected inputs that need the device, and the peak memory of a
30000-frame forward."""
import pytest
import torch

import audio2motion_reference as ref
from real3dportrait_b200 import PitchContourVAEModel, VAEModel

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
TOL = ref.E2E_BAR


def _model(kind, A, seed=11):
    m = PitchContourVAEModel(ref.HP_PITCH, audio_in_dim=A) if kind == 'pitch' else VAEModel(audio_in_dim=A)
    sd = ref.make_params({k: v.shape for k, v in m.state_dict().items()}, seed)
    m.load_state_dict(sd, strict=True)
    return m.to(DEV).eval(), sd


@pytest.fixture(scope='module')
def models():
    return {('pitch', 1024): _model('pitch', 1024), ('vae', 1024): _model('vae', 1024), ('vae', 13): _model('vae', 13)}


def _clear_of_bin_edges(batch):
    """Frames whose f0 sits within 1e-3 of a pitch-bin rounding edge (where an fp32 log one ulp apart picks the neighbouring bin; the bins
    themselves are tested in test_gpu_audio2motion_kernels.py) are set unvoiced."""
    v = ref.f0_mel_scaled64(batch['f0']).clamp(1, 255) + 0.5
    fr = v - v.floor()
    batch['f0'][(fr < 1e-3) | (fr > 1 - 1e-3)] = 0.0
    return batch


def _to(batch, dev):
    return {k: v.to(dev) for k, v in batch.items()}


@pytest.mark.parametrize('Tx', [8, 64, 400, 3000, 30000])
@pytest.mark.parametrize('temperature', [0.0, 0.2])
@pytest.mark.parametrize('case', [('pitch', 1024), ('vae', 1024), ('vae', 13)])
@torch.no_grad()
def test_forward_matches_float64(models, case, temperature, Tx):
    kind, A = case
    m, sd = models[case]
    B = 1 if Tx >= 3000 else 2
    batch = _clear_of_bin_edges(ref.make_batch(B, Tx, A, seed=Tx + B, pitch=kind == 'pitch', mouth_amp=0.45))
    torch.manual_seed(5)
    z_ref = torch.distributions.Normal(0, 1).sample([B, 16, Tx // 8])
    sd64 = {k: v.to(DEV) for k, v in sd.items()}
    want = ref.forward(sd64, _to(batch, DEV), z_ref.to(DEV), temperature, pitch=kind == 'pitch')
    torch.manual_seed(5)                                                       # the class draws the same z from the CPU generator
    ret = {}
    got = m(_to(batch, DEV), ret, train=False, temperature=temperature)
    assert got.shape == (B, Tx // 2, 64) and got.dtype == torch.float32 and got.is_cuda
    assert ret['pred'] is got and ret['mask'] is not None
    scale = float(want.abs().max())
    err = float((got.double() - want).abs().max())
    print(f'{kind}{A} T_x={Tx} temperature={temperature}: max |err| / max |exp| = {err / scale:.3e} (bar {TOL:.0e})')
    assert err <= TOL * scale, (err / scale)
    # z= replaces the draw
    got_z = m(_to(batch, DEV), {}, temperature=temperature, z=z_ref.to(DEV))
    assert torch.equal(got_z, got)


@pytest.mark.parametrize('kind', ['pitch', 'vae'])
@torch.no_grad()
def test_out_into_strided_rows(models, kind):
    m, _ = models[(kind, 1024)]
    B, Tx = 2, 400
    T = Tx // 2
    batch = _to(ref.make_batch(B, Tx, 1024, seed=3, pitch=kind == 'pitch'), DEV)
    z = torch.randn(B, 16, Tx // 8, generator=torch.Generator().manual_seed(1))
    want = m(batch, {}, temperature=0.2, z=z)
    rows = torch.randn(B * T, 146, device=DEV)
    before = rows.clone()
    ret = {}
    got = m(batch, ret, temperature=0.2, z=z, out=rows[:, 80:144])
    assert got.data_ptr() == rows.data_ptr() + 4 * 80 and ret['pred'] is got
    assert torch.equal(rows[:, 80:144], want.reshape(B * T, 64))
    assert torch.equal(rows[:, :80], before[:, :80]) and torch.equal(rows[:, 144:], before[:, 144:])


@torch.no_grad()
def test_rejected_inputs_on_device(models):
    m, _ = models[('pitch', 1024)]
    base = _to(ref.make_batch(1, 64, 1024, seed=2), DEV)
    for bad in (float('nan'), -700.5):
        b = dict(base)
        b['f0'] = base['f0'].clone()
        b['f0'][0, 10] = bad
        with pytest.raises(ValueError, match='f0'):
            m(b, {})
    b = dict(base)
    b['blink'] = base['blink'].clone()
    b['blink'][0, 3] = 2
    with pytest.raises(ValueError, match='blink'):
        m(b, {})
    b = dict(base)
    b['audio'] = base['audio'].cpu()
    with pytest.raises(RuntimeError, match='CUDA'):
        m(b, {})
    rows = torch.zeros(32, 146, device=DEV)
    with pytest.raises(ValueError, match='out'):
        m(base, {}, out=rows[:16, 80:144])
    # f0 = -700 exactly is accepted (log(0) = -inf -> bin 1), as the reference accepts it
    b = dict(base)
    b['f0'] = base['f0'].clone()
    b['f0'][0, 10] = -700.0
    assert torch.isfinite(m(b, {})).all()


@torch.no_grad()
def test_peak_memory_ten_minutes(models):
    m, _ = models[('pitch', 1024)]
    batch = _to(ref.make_batch(1, 30000, 1024, seed=9), DEV)
    m(batch, {})                                                               # weights folded and packed
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = m(batch, {})
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    # the largest live set is the decoder: its cond_layer output (T x 2048 fp32), the WaveNet's three fp32 T x 256 streams and its split
    # output, about 180 MB at T = 15000
    print(f'peak extra memory at T_x = 30000: {peak / 2**20:.1f} MiB')
    assert peak < 256 * 2**20
    assert out.shape == (1, 15000, 64)
