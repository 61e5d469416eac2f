"""Source images without a GPU: the numpy restatement (tests/source_reference.py) against the reference's own outputs in
tests/golden/source_small.npz, the integer blur against cv2, the frame selection, the darkening table, the failure geometries of
extract_background, and every input prepare_source / inpaint_torso / extract_background reject before touching the device."""
import numpy as np
import pytest
import torch

import source_reference as sr
from conftest import GOLDEN
from real3dportrait_b200 import source, synthetic as syn


@pytest.fixture(scope='module')
def z():
    return np.load(f'{GOLDEN}/source_small.npz')


def test_restatement_matches_fixture_torso_and_head(z):
    cases = sr.golden_cases(z)
    assert len(cases) == 7
    for name, img, seg in cases:
        assert np.array_equal(sr.inpaint_torso(img, seg), z[f'{name}.torso']), name
        assert np.array_equal(sr.head_image(img, seg), z[f'{name}.head']), name


def test_fixture_covers_the_edge_cases(z):
    cases = {name: seg for name, _, seg in sr.golden_cases(z)}
    hs = {k: sr.head_sum(v) for k, v in cases.items()}
    assert cases['wrap_torso'][4][0].any() and (hs['wrap_torso'][-1] != 0).any()       # torso on row 0 under head on the last row
    assert cases['wrap_neck'][2][:3].any() and (hs['wrap_neck'][-1] != 0).any()         # (dilated) neck on row 0
    assert not cases['no_torso'][4].any()
    frac = hs['fractional']
    assert ((frac != 0) != (frac > 0.5)).sum() > 1000
    neck = cases['neck_gaps'][2] != 0
    assert any(np.diff(np.nonzero(neck[:, c])[0]).max(initial=1) > 7 for c in range(neck.shape[1]))   # gaps the dilation does not close
    wide, head = cases['wide_neck'][2] != 0, hs['wide_neck'] != 0
    top = [np.nonzero(wide[:, c])[0][0] for c in range(wide.shape[1]) if wide[:, c].any()]
    cols = [c for c in range(wide.shape[1]) if wide[:, c].any()]
    assert any(not head[max(t - 4, 0), c] for t, c in zip(top, cols))                  # neck columns with no head above


def test_restatement_matches_fixture_background(z):
    """Bit-exact except where tied nearest pixels carry different colours; there the reference's colour is one of the tied ones."""
    ties = 0
    for name, img, seg in sr.golden_cases(z):
        got, src, imgs, arg = sr.extract_background(img[None], seg[None])
        ties += sr.check_background(got, z[f'{name}.bg'], src, sr.source_colours(imgs, arg))
    for n in z['bg_frames'].tolist():
        frames, segs = sr.bg_inputs(n)
        got, src, imgs, arg = sr.extract_background(frames, segs)
        ties += sr.check_background(got, z[f'bg{n}'], src, sr.source_colours(imgs, arg))
    assert ties > 0                                     # the fixture does exercise differently coloured ties


def test_restatement_edt_is_exact():
    scipy_nd = pytest.importorskip('scipy.ndimage')
    rng = np.random.default_rng(0)
    for H, W, p in ((37, 91, 0.02), (64, 64, 0.3), (100, 70, 0.001)):
        src = rng.random((H, W)) < p
        src[rng.integers(H), rng.integers(W)] = True
        d2, fr, fc = sr.edt(src)
        want = np.rint(scipy_nd.distance_transform_edt(~src) ** 2).astype(np.int64)
        assert np.array_equal(d2, want)
        assert src[fr, fc].all() and np.array_equal((fr - np.arange(H)[:, None]) ** 2 + (fc - np.arange(W)[None]) ** 2, d2)


def test_integer_blur_matches_cv2():
    cv2 = pytest.importorskip('cv2')
    rng = np.random.default_rng(1)
    for shape in ((512, 512, 3), (37, 91, 3), (64, 200, 3)):
        img = rng.integers(0, 256, shape, dtype=np.uint8)
        assert np.array_equal(sr.blur_u8(img), cv2.GaussianBlur(img, (5, 5), cv2.BORDER_DEFAULT)), shape


@pytest.mark.parametrize('n, interval, count', [(1, 5, 1), (5, 5, 1), (6, 5, 2), (99, 5, 20), (100, 20, 5), (150, 20, 8), (1000, 20, 50),
                                                (9999, 20, 500), (10000, 20, 500), (10001, 20, 501), (25000, 50, 500), (30001, 60, 501)])
def test_frame_selection(n, interval, count):
    assert source.frame_interval(n) == sr.frame_interval(n) == interval
    sel = source.selected_frames(n)
    assert list(sel) == sr.selected(n) and len(sel) == count and sel[0] == 0


def test_darken_table(z):
    tab = source.darken_table(source.NECK_ROWS)
    assert tab.dtype == np.float64 and np.array_equal(tab.view(np.int64), z['tab_neck'].view(np.int64))
    assert np.array_equal(source.darken_table(source.TORSO_ROWS), tab[:source.TORSO_ROWS])


def test_failure_geometries_raise():
    """The two geometries where the reference's NearestNeighbors.fit gets no points raise (sklearn itself, when importable, and the
    restatement): a frame without foreground, and no pixel farther than 10 from the foreground."""
    H, W = 64, 64
    img = np.zeros((1, H, W, 3), np.uint8)
    no_fg = np.zeros((1, 6, H, W), np.float32)
    no_fg[:, 0] = 1
    near = np.zeros((1, 6, H, W), np.float32)
    near[:, 0] = 1
    near[:, 4, ::12, ::12] = 1                          # foreground on a 12-pixel grid: nothing is farther than 10 from it
    near[:, 0, ::12, ::12] = 0
    for seg in (no_fg, near):
        with pytest.raises(ValueError):
            sr.extract_background(img, seg)
    neighbors = pytest.importorskip('sklearn.neighbors')
    with pytest.raises(ValueError):
        neighbors.NearestNeighbors(n_neighbors=1, algorithm='kd_tree').fit(np.zeros((0, 2)))


def _ok(H=64, W=64):
    return torch.zeros(H, W, 3, dtype=torch.uint8), torch.from_numpy(syn.make_segmap(H, W, 0))


@pytest.mark.parametrize('fn', ['prepare_source', 'inpaint_torso'])
def test_rejected_inputs_single(fn):
    f = getattr(source, fn)
    img, seg = _ok()
    bad = [
        (img.float(), seg, ValueError, 'uint8'),
        (img[..., :2], seg, ValueError, 'uint8'),
        (img[None], seg, ValueError, 'uint8'),
        (img.numpy(), seg, ValueError, 'tensor'),
        (img, seg.double(), ValueError, 'float32 or uint8'),
        (img, seg[:5], ValueError, r'\[6, 64, 64\]'),
        (img, seg[None].expand(2, -1, -1, -1), ValueError, r'\[6, 64, 64\]'),
        (img, seg[:, :32], ValueError, r'\[6, 64, 64\]'),
        (torch.zeros(63, 64, 3, dtype=torch.uint8), seg[:, :63], ValueError, r'\[64, 1024\]'),
        (torch.zeros(64, 1025, 3, dtype=torch.uint8), torch.zeros(6, 64, 1025), ValueError, r'\[64, 1024\]'),
        (img, seg, RuntimeError, 'CUDA'),              # CPU tensors: no fallback
        (img, seg.to(torch.uint8)[None], RuntimeError, 'CUDA'),
    ]
    for a, b, exc, msg in bad:
        with pytest.raises(exc, match=msg):
            f(a, b)
    if fn == 'prepare_source':
        with pytest.raises(ValueError, match='bg_img'):
            f(img, seg, bg_img=torch.zeros(1, 3, 32, 64))


def test_rejected_inputs_background():
    img, seg = _ok()
    f = source.extract_background
    for a, b, exc, msg in [
        (img, seg, ValueError, r'\[N,H,W,3\]'),
        (img[None].float(), seg[None], ValueError, 'uint8'),
        (img[None], seg, ValueError, r'\[1, 6, 64, 64\]'),
        (img[None].expand(3, -1, -1, -1), seg[None], ValueError, r'\[3, 6, 64, 64\]'),
        (img[None][:0], seg[None][:0], ValueError, 'uint8 RGB'),
        (img[None], seg[None], RuntimeError, 'CUDA'),
    ]:
        with pytest.raises(exc, match=msg):
            f(a, b)
