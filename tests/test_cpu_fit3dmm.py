"""The 3DMM fit on the CPU: the float64 restatement (tests/fit_reference.py) against the fixture made with the reference's own
fit_3dmm_for_a_image / fit_3dmm_for_a_video (tests/golden/make_golden_fit.py), the BFM and mediapipe-index loader, and Fit3DMM's argument
checks (every shape error before a device error)."""
import os

import numpy as np
import pytest
import torch

import fit_reference as fref
from real3dportrait_b200 import synthetic as syn
from real3dportrait_b200.fit3dmm import Fit3DMM, load_mp468_index

NAMES = ('id', 'exp', 'euler', 'trans')


@pytest.fixture(scope='module')
def bfm_dir(tmp_path_factory):
    return syn.write_bfm_folder(str(tmp_path_factory.mktemp('bfm')), seed=0, mp468=True)['bfm_folder']


def fixture_cases(golden):
    z = golden('fit_small')
    k = 0
    while f'c{k}_meta' in z:
        pre = f'c{k}_'
        T, video = (int(v) for v in z[pre + 'meta'][:2])
        yield k, T, bool(video), z[pre + 'lms'].numpy(), {n: z[pre + n].numpy() for n in NAMES}, z[pre + 'dev'].numpy()
        k += 1


def test_restatement_matches_the_reference(golden, bfm_dir):
    """Within the reference's own float32 deviation, recorded per case and output (the GPU tests' bar is built from it), which is small
    against the outputs in every case: an ill-conditioned fit would make that bar say little."""
    m = fref.load(bfm_dir)
    seen = set()
    for k, T, video, lms, ref, dev in fixture_cases(golden):
        assert lms.shape == (T, 478, 2) and ref['exp'].shape == (T, 64) and ref['id'].shape == (1, 80)
        want = fref.fit(m, lms, 512, video=video)
        for i, n in enumerate(NAMES):
            err = np.abs(want[n] - ref[n].astype(np.float64)).max()
            assert err <= dev[i] * (1 + 1e-9) + 1e-12, (k, n, err, dev[i])
            assert dev[i] <= 1e-4 * max(1.0, np.abs(want[n]).max()), (k, n, 'an ill-conditioned case', dev[i])
        seen.add((T, video))
    assert {(1, False), (1, True), (2, True), (50, True), (51, True), (120, True)} <= seen


def test_weights_match_the_reference_files():
    w_img, w_vid = fref.weights(False), fref.weights(True)
    assert (w_img[fref.UNMATCHED] == 0).all() and (w_vid[fref.UNMATCHED] == 0).all()
    assert w_img[33] == 5 and w_img[61] == 2 and w_img[78] == 2 and w_img[1] == 1
    assert w_vid[33] == 3 and w_vid[161] == 20 and w_vid[61] == 5 and w_vid[78] == 5
    from real3dportrait_b200.fit3dmm import _weights
    assert np.array_equal(_weights(False)[:468], w_img) and np.array_equal(_weights(True)[:468], w_vid)
    assert not _weights(True)[468:].any()


def test_loader(bfm_dir, tmp_path):
    raw = np.load(os.path.join(bfm_dir, 'index_mp468_from_mesh35709.npy'))
    assert raw.shape == (468,) and (raw[list(syn.MP_UNMATCHED)] == -1).all() and (raw >= 0).sum() == 460
    f = Fit3DMM(bfm_dir, device='cpu')
    idx = f.index.numpy()
    assert (idx[list(syn.MP_UNMATCHED)] == 0).all() and np.array_equal(idx[raw >= 0], raw[raw >= 0])
    m = fref.load(bfm_dir)
    basis = f.basis.numpy().reshape(8, 3, 64, 144).transpose(0, 2, 1, 3).reshape(512, 3, 144)
    assert np.array_equal(basis[:468], m['basis'].astype(np.float32)) and not basis[468:].any()
    mean = f.mean_shape.numpy().reshape(8, 3, 64).transpose(0, 2, 1).reshape(512, 3)
    assert np.array_equal(mean[:468], m['mean'].astype(np.float32)) and not mean[468:].any()
    with pytest.raises(FileNotFoundError, match='BFM_model_front.mat'):
        Fit3DMM(str(tmp_path), device='cpu')
    d = syn.write_bfm_folder(str(tmp_path / 'no_index'), seed=0)['bfm_folder']
    with pytest.raises(FileNotFoundError, match='index_mp468'):
        Fit3DMM(d, device='cpu')
    np.save(os.path.join(d, 'index_mp468_from_mesh35709.npy'), raw[:400])
    with pytest.raises(ValueError, match='400 entries'):
        load_mp468_index(d, 35700)
    np.save(os.path.join(d, 'index_mp468_from_mesh35709.npy'), np.full(468, 40000))
    with pytest.raises(ValueError, match='indexes vertex'):
        load_mp468_index(d, 35700)


def test_argument_validation(bfm_dir):
    f = Fit3DMM(bfm_dir, device='cpu')
    good = torch.zeros(3, 478, 2)
    for bad in (torch.zeros(3, 470, 2), torch.zeros(0, 468, 2), torch.zeros(3, 468, 3), torch.zeros(468, 2), np.zeros((3, 468, 2))):
        with pytest.raises(ValueError, match='lms'):
            f.fit_video(bad)
    for bad in (torch.zeros(2, 468, 2), torch.zeros(468, 3), torch.zeros(2, 2, 468, 2)):
        with pytest.raises(ValueError, match='lms'):
            f.fit_image(bad)
    for size in (0, -5, 1.5, True):
        with pytest.raises(ValueError, match='img_size'):
            f.fit_video(good, img_size=size)
    outs = {'id': torch.zeros(1, 80), 'exp': torch.zeros(3, 64), 'euler': torch.zeros(3, 3), 'trans': torch.zeros(3, 3)}
    for k, bad in (('exp', torch.zeros(2, 64)), ('id', torch.zeros(3, 80)), ('trans', torch.zeros(3, 3, dtype=torch.float64))):
        with pytest.raises(ValueError, match=k):
            f.fit_video(good, out={**outs, k: bad})
    with pytest.raises(ValueError, match='keys'):
        f.fit_video(good, out={'id': outs['id']})
    # shapes are right: now the CPU tensors are refused
    with pytest.raises(RuntimeError, match='CUDA'):
        f.fit_video(good)
    with pytest.raises(RuntimeError, match='CUDA'):
        f.fit_image(torch.zeros(468, 2), out={k: v[:1] for k, v in outs.items()})
