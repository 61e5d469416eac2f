"""Source images on the GPU: every output bit-exact against the reference's fixture (extract_background up to differently coloured ties)
and against the numpy restatement on randomised make_segmap maps from 64^2 to 1024^2 and 1 to 150 frames; the EDT's d^2 against scipy and
its tie rule against an all-pairs search; sentinel guards, out=, determinism, CUDA-graph replay, and the two rejected geometries."""
import numpy as np
import pytest
import torch

import source_reference as sr
from launch_harness import guarded, guards_intact
from conftest import GOLDEN
import real3dportrait_b200 as r3
from real3dportrait_b200 import _capi as capi, source, synthetic as syn

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


@pytest.fixture(scope='module')
def z():
    return np.load(f'{GOLDEN}/source_small.npz')


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def test_fixture_bit_exact(z):
    for name, img, seg in sr.golden_cases(z):
        segs = [seg] if name == 'fractional' else [seg, seg.astype(np.uint8)]
        for s in segs:
            out = r3.prepare_source(_t(img), _t(s))
            assert torch.equal(out['ref_torso_img'].cpu(), sr.normalise(z[f'{name}.torso'])), name
            assert torch.equal(out['ref_head_img'].cpu(), sr.normalise(z[f'{name}.head'])), name
            bg = r3.extract_background(_t(img[None]), _t(s[None])).cpu().numpy()
            assert torch.equal(out['bg_img'].cpu(), sr.normalise(bg))
            _, src, imgs, arg = sr.extract_background(img[None], s[None])
            sr.check_background(bg, z[f'{name}.bg'], src, sr.source_colours(imgs, arg))
            assert np.array_equal(r3.inpaint_torso(_t(img), _t(s)[None]).cpu().numpy(), z[f'{name}.torso'])
    for n in z['bg_frames'].tolist():
        frames, segs = sr.bg_inputs(n)
        bg = r3.extract_background(_t(frames), _t(segs)).cpu().numpy()
        got, src, imgs, arg = sr.extract_background(frames, segs)
        assert np.array_equal(bg, got), n
        sr.check_background(bg, z[f'bg{n}'], src, sr.source_colours(imgs, arg))


SIZES = [(64, 64), (96, 200), (333, 128), (512, 512), (1024, 1024), (1024, 700)]


@pytest.mark.parametrize('H, W', SIZES)
def test_random_maps_match_restatement(H, W):
    rng = np.random.default_rng(H * 7 + W)
    for k in range(2):
        kw = {'center': float(rng.uniform(0.35, 0.65)), 'torso_top': float(rng.uniform(0.45, 0.8)), 'torso': bool(rng.random() < 0.8),
              'neck_width': float(rng.uniform(0.0, 0.25)), 'neck_gaps': int(rng.integers(0, 6)), 'fractional': bool(k == 1),
              'roll': int(rng.integers(-H // 2, H // 2)) if rng.random() < 0.5 else 0}
        seed = int(rng.integers(1 << 30))
        img, seg = syn.make_source_image(H, W, seed), syn.make_segmap(H, W, seed, **kw)
        out = r3.prepare_source(_t(img), _t(seg))
        assert torch.equal(out['ref_torso_img'].cpu(), sr.normalise(sr.inpaint_torso(img, seg))), kw
        assert torch.equal(out['ref_head_img'].cpu(), sr.normalise(sr.head_image(img, seg))), kw
        try:
            want = sr.extract_background(img[None], seg[None])[0]
        except ValueError:
            with pytest.raises(ValueError):
                r3.extract_background(_t(img[None]), _t(seg[None]))
            continue
        assert torch.equal(out['bg_img'].cpu(), sr.normalise(want)), kw


@pytest.mark.parametrize('n, H, W', [(1, 64, 96), (4, 128, 64), (7, 80, 80), (37, 96, 128), (100, 64, 64), (150, 112, 72)])
def test_frames_match_restatement(n, H, W):
    frames, segs = sr.bg_inputs(n, H, W, seed=n)
    want = sr.extract_background(frames, segs)[0]
    assert np.array_equal(r3.extract_background(_t(frames), _t(segs)).cpu().numpy(), want)
    assert np.array_equal(r3.extract_background(_t(frames), _t(segs.astype(np.uint8))).cpu().numpy(), want)


def _distance(seg):
    """r3dp_src_bg_distance on one frame -> its d^2 [H,W]."""
    H, W = seg.shape[1:]
    s = _t(seg)
    g = torch.empty(1, H, W, dtype=torch.int16, device=DEV)
    d2, arg = torch.empty(H, W, dtype=torch.int32, device=DEV), torch.empty(H, W, dtype=torch.int32, device=DEV)
    flag = torch.empty(1, dtype=torch.int32, device=DEV)
    p = capi.ptr
    capi.check(capi.lib().r3dp_src_bg_distance(p(s), 0, 0, 1, H, W, p(g, torch.int16), 1, p(d2, torch.int32), p(arg, torch.int32),
                                               p(flag, torch.int32), capi.stream()))
    return d2.cpu().numpy()


def test_edt_exact_and_tie_rule():
    from scipy.ndimage import distance_transform_edt
    rng = np.random.default_rng(3)
    for H, W, p in ((64, 64, 0.01), (200, 150, 0.002), (1024, 1024, 0.0005), (96, 80, 0.3)):
        seg = np.zeros((6, H, W), np.float32)
        fg = rng.random((H, W)) < p
        fg[rng.integers(H), rng.integers(W)] = True
        seg[0] = ~fg
        want = np.rint(distance_transform_edt(~fg) ** 2).astype(np.int64)
        assert np.array_equal(_distance(seg), want), (H, W)
    # the fill's nearest pixel among ties: every pixel of a small image against all pairs, ordered by (d^2, column, row)
    for H, W in ((64, 64), (72, 96)):
        fg = np.zeros((H, W), bool)
        fg[H // 2:] = rng.random((H - H // 2, W)) < 0.03    # scattered foreground: the far set's edge is irregular, with many ties
        fg[-1, 0] = True
        seg = np.zeros((1, 6, H, W), np.float32)
        seg[0, 0] = ~fg
        frame = rng.integers(0, 256, (1, H, W, 3), dtype=np.uint8)
        bg = r3.extract_background(_t(frame), _t(seg)).cpu().numpy()
        far = np.rint(distance_transform_edt(~fg) ** 2) > 100
        ys, xs = np.nonzero(far)
        py, px = np.mgrid[0:H, 0:W]
        d2 = (py.reshape(-1, 1) - ys[None]) ** 2 + (px.reshape(-1, 1) - xs[None]) ** 2
        k = np.argmin(d2 * (1 << 20) + xs[None] * 1024 + ys[None], 1)
        assert (np.sort(d2, 1)[:, 1] == d2.min(1)).sum() > 50          # pixels with tied nearest sources
        assert np.array_equal(bg, frame[0][ys[k], xs[k]].reshape(H, W, 3)), (H, W)


def _guarded(shape, dtype, fill):
    buf, v = guarded(int(np.prod(shape)), dtype, fill=fill, device=DEV)
    return buf, v.view(shape)


def test_sentinels_out_and_determinism(z):
    name, img, seg = sr.golden_cases(z)[0]
    H, W = img.shape[:2]
    bufs, out = {}, {}
    for k in source.OUTPUTS:
        bufs[k], out[k] = _guarded((1, 3, H, W), torch.float32, float('nan'))
    res = r3.prepare_source(_t(img), _t(seg), out=out)
    for k in source.OUTPUTS:
        assert res[k].data_ptr() == out[k].data_ptr()
        assert guards_intact(bufs[k], out[k].numel(), fill=float('nan'))
    ref = {k: v.clone() for k, v in res.items()}
    for _ in range(3):
        again = r3.prepare_source(_t(img), _t(seg))
        assert all(torch.equal(again[k], ref[k]) for k in source.OUTPUTS)
    for fn, args in ((r3.inpaint_torso, (_t(img), _t(seg))), (r3.extract_background, (_t(img[None]), _t(seg[None])))):
        buf, o = _guarded((H, W, 3), torch.uint8, 0xAB)
        assert fn(*args, out=o).data_ptr() == o.data_ptr()
        assert guards_intact(buf, o.numel(), fill=0xAB)
        assert torch.equal(o, fn(*args))
    # bg_img= skips the extraction and is copied into out
    bg = torch.rand(1, 3, H, W, device=DEV)
    res = r3.prepare_source(_t(img), _t(seg), bg_img=bg, out=out)
    assert torch.equal(res['bg_img'], bg) and res['bg_img'].data_ptr() == out['bg_img'].data_ptr()
    assert r3.prepare_source(_t(img), _t(seg), bg_img=bg)['bg_img'] is bg


def test_cuda_graph_replay():
    H, W = 256, 192
    imgs = [syn.make_source_image(H, W, s) for s in (1, 2)]
    segs = [syn.make_segmap(H, W, s, center=0.4 + 0.1 * s) for s in (1, 2)]
    img, seg = _t(imgs[0]), _t(segs[0])
    out = {k: torch.empty(1, 3, H, W, device=DEV) for k in source.OUTPUTS}
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        r3.prepare_source(img, seg, out=out)                  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        r3.prepare_source(img, seg, out=out)
    for i in (1, 0, 1):
        img.copy_(_t(imgs[i]))
        seg.copy_(_t(segs[i]))
        g.replay()
        torch.cuda.synchronize()
        want = r3.prepare_source(_t(imgs[i]), _t(segs[i]))
        assert all(torch.equal(out[k], want[k]) for k in source.OUTPUTS), i


def test_rejected_geometries_and_devices():
    H, W = 64, 64
    img = torch.zeros(1, H, W, 3, dtype=torch.uint8, device=DEV)
    seg = torch.zeros(1, 6, H, W, device=DEV)
    seg[:, 0] = 1
    with pytest.raises(ValueError, match='no foreground'):
        r3.extract_background(img, seg)
    seg[:, 0, ::12, ::12] = 0
    with pytest.raises(ValueError, match='farther than 10'):
        r3.extract_background(img, seg)
    with pytest.raises(ValueError, match='no foreground'):
        r3.prepare_source(img[0], torch.ones(6, H, W, device=DEV))
    with pytest.raises(ValueError, match='out'):
        r3.prepare_source(img[0], seg[0], out={k: torch.empty(1, 3, H, W, device=DEV) for k in source.OUTPUTS[:2]})
    with pytest.raises(ValueError, match='out'):
        r3.inpaint_torso(img[0], seg[0], out=torch.empty(H, W, 3, device=DEV))
