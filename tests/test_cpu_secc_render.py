"""SECC renderer without a GPU: the float64 oracle (tests/secc_render_reference.py) on hand-made meshes with known answers, the loader and host
logic of SECC_Renderer, and the oracle's speed at the size the GPU tests use."""
import os
import time

import numpy as np
import pytest
import torch

import secc_render_reference as ref
from real3dportrait_b200 import secc_render as sr, synthetic as syn

S = 8


def ndc(u, v, z):
    """Pixel coordinates (column u, row v; centres at integers, exact in binary at S = 8) and z -> the oracle's (x_ndc, y_ndc, z)."""
    return [ref.pixel_ndc(u, S), ref.pixel_ndc(v, S), z]


def raster(verts, faces, slack=0.0):
    v = np.array(verts, np.float64)
    pairs = ref.raster_pairs(v, np.array(faces), S, slack)
    face, _ = ref.resolve(pairs, S)
    return face.reshape(S, S), pairs


def test_pixel_centres_are_exact():
    assert ref.pixel_ndc(0, S) == 1 - 1 / 8 and ref.pixel_ndc(7, S) == -1 + 1 / 8
    assert ref.pixel_ndc(np.arange(S), S).tolist() == [(S - 1 - 2 * c) / S for c in range(S)]


def test_shared_edge_through_centres_leaves_them_uncovered():
    # a square split along its diagonal, which passes through the centres (k, k); the outer edges lie between centres
    verts = [ndc(-0.5, -0.5, 9), ndc(4.5, -0.5, 9), ndc(4.5, 4.5, 9), ndc(-0.5, 4.5, 9)]
    face, _ = raster(verts, [[0, 1, 2], [0, 2, 3]])
    for k in range(5):
        assert face[k, k] == -1
    assert face[0, 3] == 0 and face[3, 0] == 1               # above the diagonal: face 0 (rows are v), below: face 1
    assert (face[:5, :5] >= 0).sum() == 25 - 5 and (face[5:] == -1).all() and (face[:, 5:] == -1).all()


def test_face_behind_the_camera_is_skipped():
    tri = [ndc(0, 0, -1), ndc(6, 0, -2), ndc(0, 6, -0.5)]
    face, pairs = raster(tri, [[0, 1, 2]])
    assert (face == -1).all() and pairs['face'].size == 0


def test_pixel_with_negative_pz_is_skipped():
    # one vertex behind the camera: the corrected barycentrics are all positive at some centres of the bounding box, with pz < 0 there
    verts = [ndc(1, 5, -1), ndc(0, 0, 2), ndc(6, 7, 2)]
    face, pairs = raster(verts, [[0, 1, 2]])
    neg = (pairs['w'] > 0).all(1) & (pairs['pz'] < 0)
    assert neg.any()
    assert not pairs['covered'][neg].any()
    assert (face.reshape(-1)[pairs['pix'][neg]] == -1).all()


def test_zero_area_face_is_skipped():
    face, pairs = raster([ndc(0, 0, 9), ndc(3, 3, 9), ndc(6, 6, 9)], [[0, 1, 2]])
    assert (face == -1).all() and pairs['face'].size == 0


def test_back_face_is_drawn():
    tri = [ndc(0.5, 0.5, 9), ndc(6.5, 0.5, 9), ndc(0.5, 6.5, 9)]
    f_ccw, _ = raster(tri, [[0, 1, 2]])
    f_cw, _ = raster(tri, [[0, 2, 1]])
    assert (f_ccw >= 0).sum() > 0 and np.array_equal(f_ccw >= 0, f_cw >= 0)


def test_nearer_face_wins_and_ties_go_to_the_lower_index():
    far = [ndc(0.5, 0.5, 9), ndc(6.5, 0.5, 9), ndc(0.5, 6.5, 9)]
    near = [ndc(0.5, 0.5, 8), ndc(6.5, 0.5, 8), ndc(0.5, 6.5, 8)]
    face, _ = raster(far + near, [[0, 1, 2], [3, 4, 5]])
    assert set(np.unique(face).tolist()) == {-1, 1}
    face, _ = raster(near + far, [[3, 4, 5], [0, 1, 2]])
    assert set(np.unique(face).tolist()) == {-1, 1}
    # an exact tie: the same triangle listed twice, and a third face elsewhere as face 0
    other = [ndc(7, 7, 9), ndc(7.4, 7, 9), ndc(7, 7.4, 9)]
    face, _ = raster(far + other, [[3, 4, 5], [0, 1, 2], [0, 1, 2]])
    assert set(np.unique(face).tolist()) == {-1, 1}


def test_face_zero_is_background_in_image_zero_only():
    verts = np.array([[ndc(0.5, 0.5, 9), ndc(6.5, 0.5, 9), ndc(0.5, 6.5, 9), ndc(6.5, 6.5, 9)]] * 2)
    ncc = np.full((4, 3), 0.5)
    mask, secc, face = ref.render(verts, np.array([[0, 1, 2], [1, 3, 2]]), ncc, S)
    f0 = face[0] == 0
    assert f0.any() and (face[1] == 0).any()
    assert (mask[0, 0][f0] == 0).all() and (secc[0][:, f0] == -1).all()
    assert (mask[1, 0][face[1] == 0] == 1).all() and np.allclose(secc[1][:, face[1] == 0], 0.0)
    assert (mask[0, 0][face[0] == 1] == 1).all()


# ---- loader and host logic ----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def bfm_dir(tmp_path_factory):
    d = str(tmp_path_factory.mktemp('bfm'))
    bfm = syn.make_bfm(0)
    return bfm, syn.write_bfm_folder(d, bfm)


def test_loader(bfm_dir):
    bfm, kw = bfm_dir
    m = sr.load_bfm(kw['bfm_folder'], kw['ncc_path'], kw['eye_faces'])
    tri0 = bfm['tri'].astype(np.int64) - 1                       # the file holds 1-based indices
    eyes = set((np.concatenate([bfm['right_eye'], bfm['left_eye']]) - 1).tolist())
    assert len(eyes) == bfm['right_eye'].size + bfm['left_eye'].size            # disjoint lists
    keep = [i for i in range(tri0.shape[0]) if i not in eyes]
    assert np.array_equal(m['faces'], tri0[keep]) and m['faces'].min() == 0
    assert np.array_equal(m['faces'][0], tri0[0])                               # face 0 survives the eye removal
    mean = bfm['meanshape'].reshape(-1, 3)
    assert np.abs(mean.mean(0)).max() > 1e-2                                    # the file's mean is off-centre ...
    assert np.abs(m['mean'].astype(np.float64).mean(0)).max() < 1e-6           # ... the loaded one is recentred
    assert np.allclose(m['mean'], mean - mean.mean(0), atol=1e-6)
    assert m['ncc'].shape == (mean.shape[0], 3)
    r = sr.SECC_Renderer(device='cpu', **kw)
    assert r.rasterize_size == 224 and abs(r.fov - 2 * np.degrees(np.arctan(112 / 1015))) < 1e-12
    assert r.basis.shape == (3 * mean.shape[0], 144) and r.basis.dtype == torch.float32
    assert torch.equal(r.basis[:, :80], torch.from_numpy(bfm['idBase'].astype(np.float32)))
    assert torch.equal(r.basis[:, 80:], torch.from_numpy(bfm['exBase'].astype(np.float32)))
    assert r.face_buf.dtype == torch.int32 and r.n_faces == len(keep) and r.ncc.shape == (mean.shape[0], 4)
    assert all(t.is_contiguous() for t in (r.basis, r.mean_shape, r.face_buf, r.ncc))       # the kernels take dense buffers
    kb = r.key_buffer(2, 8)
    assert (kb == -1).all() and kb.shape == (2, 8, 8)
    r.to('cpu')
    r.float()
    assert r.key_buffer(2, 8) is kb and r.graph_buffers(2, 8)[4] is kb      # a .to() frees no buffer a captured graph may write
    with pytest.raises(RuntimeError, match='CUDA'):
        r(torch.zeros(1, 80), torch.zeros(1, 64), torch.zeros(1, 3), torch.zeros(1, 3))


def test_missing_files(bfm_dir, tmp_path):
    _, kw = bfm_dir
    with pytest.raises(FileNotFoundError, match='BFM_model_front.mat'):
        sr.SECC_Renderer(device='cpu', **dict(kw, bfm_folder=str(tmp_path)))
    with pytest.raises(FileNotFoundError, match='ncc_code'):
        sr.SECC_Renderer(device='cpu', **dict(kw, ncc_path=os.path.join(str(tmp_path), 'ncc_code.npy')))
    with pytest.raises(FileNotFoundError, match='eye face list'):
        sr.SECC_Renderer(device='cpu', **dict(kw, eye_faces=(kw['eye_faces'][0], str(tmp_path / 'x.npy'))))


def test_btc_reshape():
    x = torch.arange(2 * 3 * 5, dtype=torch.float32).reshape(2, 3, 5)
    (flat,) = sr.flatten_btc(x)
    assert torch.equal(flat, x.reshape(6, 5))
    y = torch.arange(6 * 3 * 4 * 4, dtype=torch.float32).reshape(6, 3, 4, 4)
    out = sr.unflatten_btc(y, (2, 3))
    assert out.shape == (2, 3, 3, 4, 4)
    for n in range(2):
        for t in range(3):
            assert torch.equal(out[n, :, t], y[n * 3 + t])       # '(n t) c h w -> n c t h w'
    assert sr.unflatten_btc(y, None) is y


def test_oracle_speed_at_512_batch_4(bfm_dir):
    _, kw = bfm_dir
    m = ref.load(kw['bfm_folder'], kw['ncc_path'], kw['eye_faces'])
    c = syn.make_coeffs(4, seed=3, yaw=0.6)
    t0 = time.perf_counter()
    v = ref.vertices(m, c['id'].numpy(), c['exp'].numpy(), c['euler'].numpy(), c['trans'].numpy())
    mask, secc, face = ref.render(v, m['faces'], m['ncc'], 512)
    dt = time.perf_counter() - t0
    print(f'oracle: 512^2, B=4, {m["faces"].shape[0]} faces: {dt:.1f} s')
    assert dt < 30
    cover = mask.mean()
    assert 0.3 < cover < 0.95, cover                              # the head fills most of the image
    assert np.abs(v[..., :2]).max() < 1.0
    assert (face[0] == 0).sum() > 0                               # face 0 is visible in image 0
