"""Generate tests/golden/audio2motion_small.npz by running the REFERENCE's own PitchContourVAEModel (hubert, use_mouth_amp_embed) and
VAEModel (hubert and mfcc) (modules/audio2motion/vae.py) on seeded parameters and inputs, in float64 on the CPU, with train=False.

    R3DP_REFERENCE=<reference checkout> python tests/golden/make_golden_audio2motion.py

utils.commons.hparams is shimmed by a dict (tests/audio2motion_reference.py).  Every parameter and buffer is replaced by the seeded set of
make_params (post included: the reference zero-initialises it, which would make the flow an identity) and loaded with strict=True.  The
reference draws its prior noise with prior_dist.sample, which returns float32 whatever the model's dtype: the draw is recorded under
torch.manual_seed(seed) and fed to the float64 run as float64 (through a patched sample).

Stored per case `<name>_<Tx>_<B>_<t>`: the expression rows of every fourth frame (`out`, float32) and the draw (`z`, float32); per class the state_dict keys and
shapes (`keys_<cls>`, `shapes_<cls>`); the seeds."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if not os.environ.get('R3DP_REFERENCE'):
    sys.exit('set R3DP_REFERENCE to a checkout of the reference project')
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import audio2motion_reference as ref  # noqa: E402

PARAM_SEED, INPUT_SEED, NOISE_SEED = 11, 12, 13
CASES = [('pitch', 1024), ('vae', 1024), ('vae', 13)]
TEMPS = (1.0, 0.2)


def main():
    torch.set_grad_enabled(False)
    Pitch, Vae = ref.reference_classes(os.environ['R3DP_REFERENCE'])
    store = {'param_seed': np.int64(PARAM_SEED), 'input_seed': np.int64(INPUT_SEED), 'noise_seed': np.int64(NOISE_SEED)}
    for kind, A in CASES:
        m = Pitch(ref.HP_PITCH, audio_in_dim=A) if kind == 'pitch' else Vae(audio_in_dim=A)
        m.eval()
        sd = m.state_dict()
        name = f'{kind}{A}'
        store[f'keys_{name}'] = np.array(list(sd.keys()))
        store[f'shapes_{name}'] = np.array([','.join(map(str, v.shape)) for v in sd.values()])
        m.load_state_dict(ref.make_params({k: v.shape for k, v in sd.items()}, PARAM_SEED), strict=True)
        m.double()
        for Tx in (64, 400):
            for B in (1, 2):
                for ti, temp in enumerate(TEMPS):
                    batch = ref.make_batch(B, Tx, A, INPUT_SEED + Tx + B, pitch=kind == 'pitch')
                    torch.manual_seed(NOISE_SEED + ti)
                    z = m.vae.prior_dist.sample([B, 16, Tx // 8])
                    orig = m.vae.prior_dist.sample
                    m.vae.prior_dist.sample = lambda shape, z=z: z.double()
                    b64 = {k: (v.double() if v.is_floating_point() else v) for k, v in batch.items()}
                    out = m(b64, {}, train=False, temperature=temp)
                    m.vae.prior_dist.sample = orig
                    key = f'{name}_{Tx}_{B}_{ti}'
                    store[f'out_{key}'] = out[:, ::4].float().numpy()
                    store[f'z_{key}'] = z.float().numpy()
    out = os.path.join(HERE, 'audio2motion_small.npz')
    np.savez_compressed(out, **store)
    print(out, os.path.getsize(out), 'bytes')


if __name__ == '__main__':
    main()
