"""Generate tests/golden/blink_secc.npz by running the REFERENCE's own blink_eye_for_secc (inference/edit_secc.py:47-129) on SECC images of
the synthetic head (synthetic.make_bfm) rendered by tests/secc_render_reference.py.

    R3DP_REFERENCE=<reference checkout> python tests/golden/make_golden_blink.py

cv2 and imageio are not needed: edit_secc.py and utils/commons/image_utils.py import them at the top but blink_eye_for_secc calls neither, so
empty stand-ins go into sys.modules first.  scikit-learn (the reference's k-d trees) is needed.

Images: `img<k>_q` uint8 [3,S,S] are the input's 8-bit codes; the input itself is their bin centres, x = (q + 0.5) / 127.5 - 1 in fp32
(blink_reference.encode), whose quantisation is q.  Every case (t, T) of image k stores its output as the pixels that differ from the input
codes: `img<k>_t<t>_T<T>_idx` (uint32 flat indices, row-major) and `..._q` (uint8 [3,n]), lossless (the rest of the output is the input's
codes).  Cases: t = 0 (T = 8), and t = 1, T // 2, T - 1 for T = 8, 10, 12; p = -4/T**2 * t**2 + 4/T * t as real3d_infer.py computes it."""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get('R3DP_REFERENCE')
if not REF:
    sys.exit('set R3DP_REFERENCE to a checkout of the reference project')
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, ROOT)

import blink_reference as bref  # noqa: E402
import secc_render_reference as sref  # noqa: E402
from real3dportrait_b200 import synthetic as syn  # noqa: E402

# (size, exp seed, yaw): two expressions and a yaw at 512^2, one at 224^2
IMAGES = [(512, 1, 0.0), (512, 2, 0.0), (512, 3, 0.3), (224, 4, 0.0)]
CASES = [(0, 8)] + [(t, T) for T in (8, 10, 12) for t in (1, T // 2, T - 1)]


def reference_blink():
    for name in ('cv2', 'imageio'):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.path.insert(0, REF)
    from inference.edit_secc import blink_eye_for_secc
    return blink_eye_for_secc


def render_q(m, S, seed, yaw):
    c = syn.make_coeffs(1, seed=seed, yaw=yaw)
    cpu = {k: v.double().numpy() for k, v in c.items()}
    v = sref.vertices(m, cpu['id'], cpu['exp'], cpu['euler'], cpu['trans'])
    _, secc, _ = sref.render(v, m['faces'], m['ncc'], S)
    return bref.quantise(secc[0].astype(np.float32)).astype(np.uint8)


def main():
    import tempfile
    blink = reference_blink()
    with tempfile.TemporaryDirectory() as d:
        kw = syn.write_bfm_folder(d, seed=0)
        m = sref.load(kw['bfm_folder'], kw['ncc_path'], kw['eye_faces'])
    out = {'cases': np.array(CASES, dtype=np.int32), 'images': np.array(IMAGES, dtype=np.float64)}
    for k, (S, seed, yaw) in enumerate(IMAGES):
        q = render_q(m, S, seed, yaw)
        out[f'img{k}_q'] = q
        x = torch.from_numpy(bref.encode(q))
        assert (bref.quantise(x.numpy()) == q).all()
        for t, T in CASES:
            y = blink(x.clone(), bref.schedule_p(t, T)).numpy()
            qo = bref.codes(y)
            assert (bref.dequantise(qo) == y).all()
            idx = np.nonzero((qo != q).any(0).reshape(-1))[0].astype(np.uint32)
            out[f'img{k}_t{t}_T{T}_idx'] = idx
            out[f'img{k}_t{t}_T{T}_q'] = qo.reshape(3, -1)[:, idx].astype(np.uint8)
            print(f'image {k} ({S}^2) t={t} T={T}: {len(idx)} pixels changed')
    path = os.path.join(HERE, 'blink_secc.npz')
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
