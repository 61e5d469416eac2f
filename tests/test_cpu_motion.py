"""Clip motion on the CPU: the float64 restatement (tests/motion_reference.py) against the fixture made with the reference's own code
(tests/golden/make_golden_motion.py), mirror_index, the key points' off-by-one, and ClipMotion's argument checks."""
import numpy as np
import pytest
import torch

import motion_reference as mref
from real3dportrait_b200 import synthetic as syn
from real3dportrait_b200.motion import ClipMotion

NAMES = ('cameras', 'kp_s', 'kp_d')


@pytest.fixture(scope='module')
def bfm_dir(tmp_path_factory):
    return syn.write_bfm_folder(str(tmp_path_factory.mktemp('bfm')), seed=0, keypoints=True)['bfm_folder']


def fixture_cases(golden):
    z = golden('motion_small')
    k = 0
    while f'c{k}_meta' in z:
        pre = f'c{k}_'
        T, P, mp = (int(v) for v in z[pre + 'meta'])
        pose = None if P == 0 else (z[pre + 'pose_euler'].numpy(), z[pre + 'pose_trans'].numpy())
        args = tuple(z[pre + n].numpy() for n in ('id', 'exp', 'src_euler', 'src_trans', 'src_exp')) + (pose, bool(mp))
        yield k, T, args, [z[pre + n].numpy() for n in NAMES], z[pre + 'dev'].numpy()
        k += 1


def test_restatement_matches_the_reference(golden, bfm_dir):
    """Within the reference's own float32 deviation, which REF_DEV bounds on every case (the GPU tests' bar is built from it)."""
    m = mref.load(bfm_dir)
    n = 0
    for k, T, args, ref, dev in fixture_cases(golden):
        want = mref.clip(m, *args)
        for i, name in enumerate(NAMES):
            err = np.abs(want[i] - ref[i].astype(np.float64)).max()
            assert err <= dev[i] * (1 + 1e-9) + 1e-12, (k, name, err, dev[i])
            assert dev[i] <= mref.REF_DEV[i], (k, name, dev[i])
        assert ref[0].shape == (T, 25) and ref[1].shape == (1, 68, 3) and ref[2].shape == (T, 68, 3)
        n += 1
    assert n >= 10
    # the bound is not loose: some case comes within 10 % of it
    devs = np.array([c[4] for c in fixture_cases(golden)])
    assert (devs.max(0) >= 0.9 * np.array(mref.REF_DEV)).all()


def test_fixture_covers_the_clamp_and_mirror_turns(golden):
    Ts, Ps, clamped = set(), set(), 0
    for _, T, args, ref, _ in fixture_cases(golden):
        Ts.add(T)
        Ps.add(0 if args[5] is None else len(args[5][0]))
        clamped += int((np.abs(ref[2][..., :2]) == 1).sum())
    assert {3, 8, 57, 250} <= Ts and 0 in Ps and 1 in Ps and any(1 < P < 57 for P in Ps) and any(P > 250 for P in Ps)
    assert clamped > 0


def test_mirror_index_table():
    assert [mref.mirror_index(i, 3) for i in range(10)] == [0, 1, 2, 2, 1, 0, 0, 1, 2, 2]
    assert [mref.mirror_index(i, 1) for i in range(4)] == [0, 0, 0, 0]
    assert [mref.mirror_index(i, 4) for i in range(12)] == [0, 1, 2, 3, 3, 2, 1, 0, 0, 1, 2, 3]


def test_keypoints_are_read_without_minus_one(golden, bfm_dir):
    """The reference gathers model['keypoints'] as stored: the 0-based landmarks (ParametricFaceModel's - 1) miss its key points."""
    m, m1 = mref.load(bfm_dir), mref.load(bfm_dir, minus_one=True)
    assert (m['keypoints'] == m1['keypoints'] + 1).all()
    for _, _, args, ref, dev in fixture_cases(golden):
        assert np.abs(mref.clip(m1, *args)[1] - ref[1]).max() > 1000 * dev[1]
        assert np.abs(mref.clip(m, *args)[1] - ref[1]).max() <= dev[1] * (1 + 1e-9) + 1e-12


def test_smoothing_rejects_short_clips(bfm_dir):
    with pytest.raises(ValueError):
        mref.smooth_kp(np.zeros((2, 68, 2)))
    cm = ClipMotion(bfm_dir, device='cpu')
    c = syn.make_coeffs(2)
    for T in (1, 2):
        with pytest.raises(ValueError, match='at least 3 frames'):
            cm.clip(c['id'][:1], torch.zeros(T, 64), c['euler'][:1], c['trans'][:1], c['exp'][:1])


def test_clip_motion_argument_checks(bfm_dir, tmp_path):
    cm = ClipMotion(bfm_dir, device='cpu')
    assert cm.basis.shape == (204, 144) and cm.mean_shape.shape == (204,) and cm.n_kp == 68
    c = syn.make_coeffs(5)
    idc, exp, e, t, se = c['id'][:1], c['exp'], c['euler'][:1], c['trans'][:1], c['exp'][:1]
    bad = [((c['id'][:2], exp, e, t, se), {}),                            # id neither [1,80] nor [T,80]
           ((idc, exp[:, :60], e, t, se), {}),                            # exp width
           ((idc, exp, e[:, :2], t, se), {}),                             # src_euler width
           ((idc, exp, e, torch.zeros(2, 3), se), {}),                    # src_trans rows
           ((idc, exp, e, t, exp[:2]), {}),                               # src_exp rows
           ((idc, exp, e, t, se), {'pose': (torch.zeros(0, 3), torch.zeros(0, 3))}),     # P = 0
           ((idc, exp, e, t, se), {'pose': (torch.zeros(4, 3), torch.zeros(3, 3))}),     # P mismatch
           ((idc, exp, e, t, se), {'pose': torch.zeros(4, 3)})]                          # not a pair
    for args, kw in bad:
        with pytest.raises(ValueError):
            cm.clip(*args, **kw)
    with pytest.raises(RuntimeError, match='CUDA'):
        cm.clip(idc, exp, e, t, se)
    with pytest.raises(FileNotFoundError):
        ClipMotion(str(tmp_path), device='cpu')
    import scipy.io
    mat = scipy.io.loadmat(bfm_dir + '/BFM_model_front.mat')
    d = tmp_path / 'nokp'
    d.mkdir()
    scipy.io.savemat(str(d / 'BFM_model_front.mat'), {k: mat[k] for k in ('meanshape', 'idBase', 'exBase')})
    with pytest.raises(KeyError, match='keypoints'):
        ClipMotion(str(d), device='cpu')
    n = mat['meanshape'].size // 3
    for kp in (n, -1):                                                    # key points must index the vertices as stored
        d = tmp_path / f'kp{kp}'
        d.mkdir()
        k = mat['keypoints'].copy()
        k[5] = kp
        scipy.io.savemat(str(d / 'BFM_model_front.mat'), {**{x: mat[x] for x in ('meanshape', 'idBase', 'exBase')}, 'keypoints': k})
        with pytest.raises(ValueError, match='keypoints'):
            ClipMotion(str(d), device='cpu')


def test_synthetic_keypoints_leave_the_bfm_unchanged(tmp_path):
    a = syn.make_bfm(0)
    k = syn.make_keypoints(a)
    b = syn.make_bfm(0)
    assert all(np.array_equal(a[x], b[x]) for x in a)
    assert k.shape == (68, 1) and len(np.unique(k)) == 68 and k.min() >= 1
    P = a['meanshape'].reshape(-1, 3)[k.astype(np.int64)[:, 0] - 1]
    assert (P[:, 2] > 0).all()                                             # the front of the head
    import scipy.io
    kw = syn.write_bfm_folder(str(tmp_path / 'plain'), seed=0)
    assert 'keypoints' not in scipy.io.loadmat(kw['bfm_folder'] + '/BFM_model_front.mat')
