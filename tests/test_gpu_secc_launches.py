"""Every launch of the SECC renderer (r3dp_secc_vertices, r3dp_secc_raster + r3dp_secc_resolve) and of blink (r3dp_secc_blink) at the
arguments the engine and the class pass, and at the edges each entry point accepts, against float64 (tests/secc_launch_reference.py) or,
for blink, bit for bit against the numpy restatement (tests/blink_reference.py, tie = 'lowest').  Every output sits between sentinel guards:
every element written, nothing outside it, the key buffer left empty.

* VERTEX_ROWS  the engine's rows (euler = trans = NULL, id and exp read from one row at stride 144 or 146, exp at row + n_id), the class's
               (separate id / exp tensors, pose given), separate tensors of other widths, a K sweep on random bases, B across the 32-frame
               tile, N around the 8-vertex block, and euler angles beyond +-pi; bar: vertex_bar.
* RASTER_ROWS  synthetic heads at S from 1 to 1024 (the engine's S = 512 without the mask, which must equal the launch with it bit for bit),
               coarse meshes at 2048 / 4096, heads partly off screen, near and behind the camera and turned by +-pi/2 and pi;
               hand-placed vertex buffers (secc_launch_reference.hand_scenes) with exact face maps; bar: check_raster.
* BLINK_ROWS   the engine's launch (rows at stride 146 read from column 144), the drop-in, S at the ends of 64..1024 and around powers of two,
               B = 33 and 200, hand-made eye holes that touch the prior regions' limits, a large blink list, and the control edges.
* test_secc_launches_have_rows  records the launches of begin_planes(coeff_src=), an engine step (blink False / True), forward and the drop-in,
               requires them to equal secc_launch_reference.launch_plan, and every launch to have a row here (and every engine / class row
               to be launched)."""
import ctypes
import math

import numpy as np
import pytest
import torch

import blink_reference as bref
import secc2plane_reference as s2p_ref
import secc_launch_reference as lr
import secc_render_reference as ref
from launch_harness import Recorder, assert_plan, assert_rows, guarded, guards_intact, untouched
import real3dportrait_b200 as r3
from real3dportrait_b200 import _capi as capi, engine, synthetic as syn

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
TAN = ref.TAN_HALF
N_BFM = 150 * 238


@pytest.fixture(scope='module')
def bfm(tmp_path_factory):
    kw = syn.write_bfm_folder(str(tmp_path_factory.mktemp('bfm')), seed=0)
    return kw, ref.load(kw['bfm_folder'], kw['ncc_path'], kw['eye_faces'])


@pytest.fixture(scope='module')
def coarse(tmp_path_factory):
    """A 16 x 24 head (384 vertices) for S = 2048 / 4096, where the float64 oracle and one thread per face loop over large boxes."""
    kw = syn.write_bfm_folder(str(tmp_path_factory.mktemp('coarse')), bfm=syn.make_bfm(seed=1, rows=16, cols=24))
    return kw, ref.load(kw['bfm_folder'], kw['ncc_path'], kw['eye_faces'])


_RENDERERS = {}


def renderer(kw, S):
    key = (kw['bfm_folder'], S)
    if key not in _RENDERERS:
        _RENDERERS[key] = r3.SECC_Renderer(S, device=DEV, **kw)
    return _RENDERERS[key]


# ---- r3dp_secc_vertices --------------------------------------------------------------------------------------------------------------------
# (tag, basis: 'bfm' | 'rand', N, n_id, n_exp, B, layout: 'row' (one [B, W] tensor, exp at row + n_id, W = ids = exps) | 'split' (id [B, ids],
#  exp [B, exps]), W / (ids, exps), pose: None (NULL) | yaw amplitude | 'wild' (euler beyond +-pi))
VERTEX_ROWS = [
    ('engine-144-B4', 'bfm', N_BFM, 80, 64, 4, 'row', 144, None),
    ('engine-144-B1', 'bfm', N_BFM, 80, 64, 1, 'row', 144, None),
    ('engine-146-B4', 'bfm', N_BFM, 80, 64, 4, 'row', 146, None),
    ('rows-146-B1', 'bfm', N_BFM, 80, 64, 1, 'row', 146, None),
    ('forward-B4', 'bfm', N_BFM, 80, 64, 4, 'split', (80, 64), 0.6),
    ('split-84-100', 'bfm', N_BFM, 80, 64, 3, 'split', (84, 100), 0.6),
    ('wild-euler', 'bfm', N_BFM, 80, 64, 4, 'split', (80, 64), 'wild'),
] + [(f'K-{a}+{e}', 'rand', 2000, a, e, 5, 'row', a + e + 3, 0.6) for a, e in ((0, 4), (4, 0), (1, 3), (80, 64), (124, 128), (128, 128))] \
  + [(f'B{B}', 'bfm', N_BFM, 80, 64, B, 'row', 144, 0.6) for B in (1, 31, 32, 33, 64, 65)] \
  + [(f'N{N}', 'rand', N, 80, 64, 5, 'row', 144, 0.6) for N in (1, 7, 8, 9)]


def vertex_signature(row):
    tag, _, N, n_id, n_exp, B, layout, W, pose = row
    ids, exps = (W, W) if layout == 'row' else W
    return 'r3dp_secc_vertices', (N, n_id, n_exp, ids, exps, B, 10.0, ctypes.c_float(TAN).value), (pose is not None,) * 2


def _rand_basis(N, K, seed):
    g = np.random.default_rng(seed)
    mean = g.uniform(-0.6, 0.6, (N, 3)).astype(np.float32)
    basis = (0.01 * g.standard_normal((3 * N, K))).astype(np.float32)
    return basis, mean


def _pose(B, pose, seed):
    if pose is None:
        return None, None
    g = torch.Generator().manual_seed(seed)
    if pose == 'wild':
        e = torch.tensor([[3 * math.pi + 0.1, -3 * math.pi - 0.1, 2.5 * math.pi], [-3 * math.pi - 0.1, 3 * math.pi + 0.1, -math.pi],
                          [math.pi, -math.pi / 2, 3 * math.pi + 0.1], [1.0, 2.0, -3 * math.pi - 0.1]])[:B]
    else:
        e = (torch.rand(B, 3, generator=g) * 2 - 1) * pose * torch.tensor([0.2, 1.0, 0.2])
    return e, 0.02 * torch.randn(B, 3, generator=g)


def _launch_vertices(basis, mean, N, n_id, n_exp, id_t, ids, exp_p, exps, euler, trans, B):
    """r3dp_secc_vertices into a buffer between guards: every element written, nothing else, w = 0."""
    big, verts = guarded(B * N * 4, torch.float32, device=DEV)
    p = capi.ptr
    capi.check(capi.lib().r3dp_secc_vertices(p(basis), p(mean), N, n_id, n_exp, p(id_t), ids, exp_p, exps, p(euler), p(trans), B, 10.0, TAN,
                                             p(verts), capi.stream()))
    torch.cuda.synchronize()
    assert guards_intact(big, B * N * 4), 'vertices: written outside the output'
    assert not bool(untouched(verts).any()), 'vertices: an element was not written'
    v = verts.view(B, N, 4)
    assert bool((v[..., 3] == 0).all())
    return v


@pytest.mark.parametrize('row', VERTEX_ROWS, ids=[r[0] for r in VERTEX_ROWS])
def test_vertices_vs_float64(bfm, row):
    tag, kind, N, n_id, n_exp, B, layout, W, pose = row
    K = n_id + n_exp
    if kind == 'bfm':
        _, m = bfm
        basis = np.concatenate([m['id_base'], m['exp_base']], 1).astype(np.float32)
        mean = m['mean'].astype(np.float32)
    else:
        basis, mean = _rand_basis(N, K, seed=K + N)
        m = {'id_base': basis[:, :n_id].astype(np.float64), 'exp_base': basis[:, n_id:].astype(np.float64), 'mean': mean.astype(np.float64)}
    basis_t, mean_t = torch.from_numpy(np.ascontiguousarray(basis)).to(DEV), torch.from_numpy(mean.reshape(-1).copy()).to(DEV)
    g = torch.Generator().manual_seed(B * 7 + K)
    euler, trans = _pose(B, pose, seed=B + K)
    euler_d, trans_d = (None if euler is None else euler.to(DEV)), (None if trans is None else trans.to(DEV))
    if layout == 'row':
        rows = torch.randn(B, W, generator=g).to(DEV)
        id_t, ids, exps = rows, W, W
        exp_p = ctypes.c_void_p(rows.data_ptr() + 4 * n_id)                # the engine's exp pointer: row + n_id
        idv, expv = rows[:, :n_id], rows[:, n_id:K]
    else:
        ids, exps = W
        id_t, exp_t = torch.randn(B, ids, generator=g).to(DEV), torch.randn(B, exps, generator=g).to(DEV)
        exp_p = capi.ptr(exp_t)
        idv, expv = id_t[:, :n_id], exp_t[:, :n_exp]
    got = _launch_vertices(basis_t, mean_t, N, n_id, n_exp, id_t, ids, exp_p, exps, euler_d, trans_d, B).cpu().double().numpy()
    v, bar = lr.vertex_bar(m, {'id': idv, 'exp': expv, 'euler': euler, 'trans': trans})
    err = np.abs(got[..., :3] - v)
    ratio = float((err / bar).max())
    print(f'vertices {tag}: max |err| xy {err[..., :2].max():.2e} z {err[..., 2].max():.2e}; worst err/bar {ratio:.3f}')
    assert ratio <= 1.0, f'{tag}: err/bar {ratio:.3f}'


# ---- r3dp_secc_raster + r3dp_secc_resolve --------------------------------------------------------------------------------------------------
def _raster(verts, N, faces, ncc4, B, S, drop_face0, with_mask):
    """raster then resolve, the key buffer read back between them; every output between guards.  -> (face [B,S,S], secc, mask or None)."""
    L, p, st = capi.lib(), capi.ptr, capi.stream()
    F = faces.shape[0]
    kbig, keys = guarded(B * S * S, torch.int64, device=DEV)
    keys.fill_(-1)
    capi.check(L.r3dp_secc_raster(p(verts), N, p(faces, torch.int32), F, B, S, p(keys, torch.int64), st))
    kimg = keys.clone()
    sbig, secc = guarded(B * 3 * S * S, torch.float32, device=DEV)
    mbig, mask = guarded(B * S * S, torch.float32, device=DEV) if with_mask else (None, None)
    capi.check(L.r3dp_secc_resolve(p(verts), N, p(faces, torch.int32), p(ncc4), B, S, int(drop_face0), p(keys, torch.int64), p(secc),
                                   p(mask), st))
    torch.cuda.synchronize()
    assert bool((keys == -1).all()), 'resolve leaves the key buffer empty'
    assert guards_intact(kbig, B * S * S), 'keys: written outside the output'
    assert guards_intact(sbig, B * 3 * S * S), 'secc: written outside the output'
    assert not bool(untouched(secc).any()), 'secc: an element was not written'
    if with_mask:
        assert guards_intact(mbig, B * S * S), 'mask: written outside the output'
        assert not bool(untouched(mask).any()), 'mask: an element was not written'
    k = kimg.cpu().numpy().view(np.uint64)
    face = np.where(k == np.uint64(2 ** 64 - 1), -1, (k & np.uint64(0xffffffff)).astype(np.int64)).reshape(B, S, S)
    return face, secc.view(B, 3, S, S), (mask.view(B, 1, S, S) if with_mask else None)


# (tag, mesh: 'bfm' | 'coarse', S, B, pose: None (engine: NULL) | yaw amplitude | name of a POSES entry, drop_face0, mask)
POSES = {
    'offscreen': ([[0, 0.3, 0], [0, -0.3, 0.1]], [[0.95, 0, 0], [0, -1.05, 0.2]]),      # a third of the head or more beyond x / y = -+1
    'near': ([[0, 0.2, 0]], [[0, 0, 9.0]]),                                          # z from 0.3 to 1.7: faces far beyond NDC +-1.5
    'behind': ([[0, 0, 0]], [[0, 0, 12.0]]),                                         # z < 0 everywhere: all culled
    'turned': ([[math.pi / 2, 0, 0], [-math.pi / 2, 0, 0], [0, math.pi / 2, 0], [0, -math.pi / 2, 0], [0, 0, math.pi / 2],
                [0, 0, -math.pi / 2], [math.pi, 0, 0], [0, math.pi, 0], [0, 0, math.pi]], [[0, 0, 0]] * 9),
}
RASTER_ROWS = [
    ('engine-512-B4', 'bfm', 512, 4, None, 1, False),
    ('engine-512-B1', 'bfm', 512, 1, None, 1, False),
    ('class-224-B4', 'bfm', 224, 4, 0.6, 1, True),
    ('drop0-512-B2', 'bfm', 512, 2, 0.6, 0, True),
] + [(f'S{S}', 'bfm', S, 2, 0.6, 1, True) for S in (1, 2, 3, 8, 64, 511, 513, 1023, 1024)] \
  + [(f'coarse-S{S}', 'coarse', S, 1, 0.6, 1, True) for S in (2048, 4096)] \
  + [(f'{k}', 'bfm', 128 if k == 'near' else 256, len(POSES[k][0]), k, 1, True) for k in POSES]


def raster_signatures(row, N, F):
    tag, _, S, B, _, drop, mask = row
    return ('r3dp_secc_raster', (N, F, B, S), ()), ('r3dp_secc_resolve', (N, B, S, drop), (mask,))


@pytest.mark.parametrize('row', RASTER_ROWS, ids=[r[0] for r in RASTER_ROWS])
def test_raster_resolve_vs_float64(bfm, coarse, row):
    tag, mesh, S, B, pose, drop, with_mask = row
    kw, m = bfm if mesh == 'bfm' else coarse
    r = renderer(kw, S)
    c = syn.make_coeffs(B, seed=S + B)
    if pose is None:
        euler = trans = None
    elif isinstance(pose, str):
        euler, trans = torch.tensor(POSES[pose][0], dtype=torch.float32), torch.tensor(POSES[pose][1], dtype=torch.float32)
    else:
        c = syn.make_coeffs(B, seed=S + B, yaw=pose)
        euler, trans = c['euler'], c['trans']
    coeff = torch.cat([c['id'], c['exp']], 1).to(DEV)
    verts = _launch_vertices(r.basis, r.mean_shape, r.n_verts, r.n_id, r.n_exp, coeff, 144, ctypes.c_void_p(coeff.data_ptr() + 4 * r.n_id),
                             144, None if euler is None else euler.to(DEV), None if trans is None else trans.to(DEV), B)
    face, secc, mask = _raster(verts, r.n_verts, r.face_buf, r.ncc, B, S, drop, with_mask)
    # the other mask form of the same launch: secc equal bit for bit
    _, secc2, mask2 = _raster(verts, r.n_verts, r.face_buf, r.ncc, B, S, drop, not with_mask)
    assert torch.equal(secc.view(torch.int32), secc2.view(torch.int32)), f'{tag}: secc depends on whether the mask is written'
    mask = mask if with_mask else mask2
    v, bar = lr.vertex_bar(m, {'id': c['id'], 'exp': c['exp'], 'euler': euler, 'trans': trans})
    st = lr.check_raster(m, v, lr.raster_err(v, bar), S, face, secc.cpu().double().numpy(), mask.cpu().double().numpy(), f'raster {tag}', drop)
    if pose == 'behind':
        assert (face == -1).all() and bool((secc == -1).all())
    if pose == 'near':
        assert np.abs(v[..., :2]).max() > 1.5 and (face >= 0).mean() > 0.5         # faces beyond the cull, covering the screen
    if pose == 'offscreen':
        assert v[0, :, 0].min() < -1.2 and 0.05 < (face[0] >= 0).mean()
    if tag.startswith('engine'):
        # the class's render() on the same rows launches exactly this
        _, sr = r.render(coeff)
        assert torch.equal(sr, secc)
    assert st['decisive'] > 0.5 * B * S * S


@pytest.mark.parametrize('scene', lr.hand_scenes(), ids=[s['name'] for s in lr.hand_scenes()])
def test_raster_hand_placed(scene):
    S, v, faces = scene['S'], scene['v'], scene['faces']
    N = v.shape[1]
    v4 = np.zeros((1, N, 4), np.float32)
    v4[..., :3] = v
    ncc4 = np.zeros((N, 4), np.float32)
    ncc4[:, :3] = scene['ncc']
    verts = torch.from_numpy(v4).to(DEV)
    f_t = torch.from_numpy(faces.astype(np.int32)).to(DEV)
    face, secc, mask = _raster(verts, N, f_t, torch.from_numpy(ncc4).to(DEV), 1, S, scene['drop_face0'], True)
    want = lr.expected_faces(scene)
    assert np.array_equal(face[0], want), f'{scene["name"]}: {(face[0] != want).sum()} pixels differ from the exact face map'
    for rc in scene['empty']:
        assert face[0][rc] == -1, (scene['name'], rc)
    for rc in scene['covered']:
        assert face[0][rc] >= 0, (scene['name'], rc)
    m = {'faces': faces, 'ncc': scene['ncc']}
    lr.check_raster(m, v, np.zeros((1, 2)), S, face, secc.cpu().double().numpy(), mask.cpu().double().numpy(), f'hand {scene["name"]}',
                    scene['drop_face0'])


# ---- r3dp_secc_blink -----------------------------------------------------------------------------------------------------------------------
def _face_img(S, holes):
    """Hand-made [3,S,S] codes: (1 + r % 250, 1 + c % 250, 200) on the face, 0 in each hole rows [r0, r1) x cols [c0, c1)."""
    r, c = np.mgrid[0:S, 0:S]
    q = np.stack([1 + r % 250, 1 + c % 250, np.full((S, S), 200)]).astype(np.int64)
    for r0, r1, c0, c1 in holes:
        q[:, r0:r1, c0:c1] = 0
    return bref.encode(q)


def edge_images(S):
    """Eye holes touching the prior regions' limits: rows S/4 and S/2 - 1, columns S/4, S/2 - 1, S/2 and 3S/4 - 1."""
    a, h, t = S // 4, S // 2, (S // 4) * 3
    k = max(2, S // 32)
    return [_face_img(S, [(a, h, a, h), (a, h, h, t)]),                                   # both prior regions entirely holes
            _face_img(S, [(a, a + k, a, a + 2 * k), (a, a + k, t - 2 * k, t)]),           # top row, outer columns
            _face_img(S, [(h - k, h, h - 2 * k, h), (h - k, h, h, h + 2 * k)])]           # bottom row, the two middle columns


def _want(x, p):
    """The restatement of one image under control p (None = untouched) -> (fp32 image, faulted)."""
    if p is None:
        return x, False
    try:
        return bref.blink(x, p, tie='lowest')[0], False
    except ValueError:
        return x, True


def _launch_blink(x, p=None, rows=ctypes.c_void_p(0), stride=0):
    """r3dp_secc_blink on x [B,3,S,S] (numpy fp32) between guards (images and scratch); p: float64 [B], or rows: the device pointer of the
    (t, T) columns of fp32 rows at the given stride."""
    B, S = x.shape[0], x.shape[-1]
    big, secc = guarded(x.size, torch.float32, device=DEV)
    secc.copy_(torch.from_numpy(x).reshape(-1))
    n = int(capi.lib().r3dp_secc_blink_scratch_bytes(B, S))
    sc_big = torch.full((n + 2 * 4096,), 0xA5, dtype=torch.uint8, device=DEV)
    off = (-(sc_big.data_ptr() + 4096)) % 256
    sc = sc_big[4096 + off:4096 + off + n]
    faults = torch.zeros(1, dtype=torch.int32, device=DEV)
    p_t = None if p is None else torch.tensor(p, dtype=torch.float64, device=DEV)
    capi.check(capi.lib().r3dp_secc_blink(capi.ptr(secc), B, S, capi.ptr(p_t, torch.float64), rows, stride,
                                          capi.ptr(sc, torch.uint8), capi.ptr(faults, torch.int32), capi.stream()))
    torch.cuda.synchronize()
    assert guards_intact(big, x.size), 'blink images: written outside the output'
    assert bool((sc_big[:4096 + off] == 0xA5).all()) and bool((sc_big[4096 + off + n:] == 0xA5).all()), 'blink: written outside the scratch'
    return secc.view(x.shape).cpu().numpy(), int(faults.item())


def _check_blink(tag, x, ctl):
    """ctl: list of per-image controls, each ('p', p) or ('rows', t, T); one launch per form present.  Bit for bit against the restatement."""
    B = x.shape[0]
    forms = {c[0] for c in ctl}
    assert len(forms) == 1
    if forms == {'p'}:
        ps = [c[1] for c in ctl]
        got, faults = _launch_blink(x, p=ps)
        want_p = [bref.p_control(p) for p in ps]
    else:
        rows = torch.zeros(B, 146)
        for b, c in enumerate(ctl):
            rows[b, 144], rows[b, 145] = c[1], c[2]
        rows = rows.to(DEV)
        got, faults = _launch_blink(x, rows=ctypes.c_void_p(rows.data_ptr() + 4 * 144), stride=146)   # the engine's launch: stride 146, column 144
        want_p = [bref.rows_control(c[1], c[2]) for c in ctl]
    n_fault, blinked = 0, 0
    for b in range(B):
        want, fault = _want(x[b], want_p[b])
        n_fault += fault
        blinked += want_p[b] is not None and not fault
        assert np.array_equal(got[b].view(np.uint32), want.view(np.uint32)), \
            f'{tag} image {b} control {ctl[b]} (p {want_p[b]}): {(got[b].view(np.uint32) != want.view(np.uint32)).sum()} values differ'
    assert faults == n_fault, f'{tag}: {faults} faults counted, {n_fault} expected'
    print(f'blink {tag}: B={B} S={x.shape[-1]}, {blinked} edited, {n_fault} faults, bit-exact')


def _rendered(kw, S, B, seed):
    r = renderer(kw, S)
    c = syn.make_coeffs(B, seed=seed, yaw=0.3)
    return r.render(torch.cat([c['id'], c['exp']], 1).to(DEV), c['euler'].to(DEV), c['trans'].to(DEV))[1].cpu().numpy()


MENU = [('rows', 3, 8), ('rows', 0, 0), ('rows', 5, 10), ('rows', 0, 8), ('rows', 11, 12), ('rows', 1, 9)]
#: the control edges (SECC_Renderer.blink's docstring; bref.rows_control / p_control): one image each
ROW_EDGES = [(0.5, 8.0), (2.7, 8.9), (7.9, 8.0), (0.5, 0.7), (1.5, 1.7), (8, 8), (9, 8), (0, 1), (3, 4096), (3, 4097), (4095, 4096),
             (-1, 8), (-0.5, 8), (3, -8), (float('nan'), 8), (3, float('nan')), (float('inf'), 8), (3, float('inf')), (float('-inf'), 8),
             (3, float('-inf')), (4, 8)]
P_EDGES = [-0.0, float('nan'), 1.0, float(np.nextafter(1.0, 2.0)), 5e-324, -1.0, 0.5, float('inf')]
# (tag, S, B, images, controls)
BLINK_ROWS = [
    ('engine-512-B4', 512, 4, 'rendered', [('rows', 2, 8), ('rows', 0, 0), ('rows', 6, 12), ('rows', 4, 8)]),
    ('drop-in-512', 512, 1, 'rendered', [('p', 0.5)]),
] + [(f'S{S}', S, 3, 'rendered', [('rows', 3, 8), ('rows', 5, 10), ('rows', 0, 0)]) for S in (64, 65, 127, 128, 1023, 1024)] \
  + [(f'S{S}-p', S, 2, 'rendered', [('p', 0.44), ('p', 1.0)]) for S in (64, 1024)] \
  + [(f'B{B}-S64', 64, B, 'rendered', [MENU[b % len(MENU)] for b in range(B)]) for B in (33, 200)] \
  + [(f'edges-S{S}-{f}', S, 3, 'edge', [('p', 0.5)] * 3 if f == 'p' else [('rows', 1, 8), ('rows', 5, 10), ('rows', 3, 12)])
     for S in (64, 1024) for f in ('p', 'rows')] \
  + [('large-list-S1024', 1024, 1, 'large', [('p', 1.0)]),
     ('control-rows', 128, len(ROW_EDGES), 'good', [('rows', t, T) for t, T in ROW_EDGES]),
     ('control-p', 128, len(P_EDGES), 'good', [('p', p) for p in P_EDGES])]


def blink_signature(row):
    tag, S, B, _, ctl = row
    return lr.blink_row(B, S, 0 if ctl[0][0] == 'p' else 146, ctl[0][0] == 'p')


@pytest.mark.parametrize('row', BLINK_ROWS, ids=[r[0] for r in BLINK_ROWS])
def test_blink_vs_restatement(bfm, row):
    tag, S, B, kind, ctl = row
    kw, _ = bfm
    if kind == 'rendered':
        x = _rendered(kw, S, B, seed=S * 3 + B)
    elif kind == 'edge':
        x = np.stack(edge_images(S))
    elif kind == 'large':
        x = _face_img(S, [(S // 4 + 8, S // 2 - 8, S // 4 + 16, S // 2 - 4), (S // 4 + 8, S // 2 - 8, S // 2 + 4, 3 * (S // 4) - 16)])[None]
    else:
        one = _face_img(S, [(S // 4 + 6, S // 4 + 14, S // 4 + 4, S // 4 + 20), (S // 4 + 8, S // 4 + 15, S // 2 + 6, S // 2 + 22)])
        x = np.stack([one] * B)
    if tag == 'drop-in-512':
        out = r3.blink_eye_for_secc(torch.from_numpy(x[0]).to(DEV), ctl[0][1])
        want, _ = _want(x[0], ctl[0][1])
        assert np.array_equal(out.cpu().numpy().view(np.uint32), want.view(np.uint32))
    _check_blink(tag, x, ctl)


def test_drop_in_control_edges(bfm):
    """blink_eye_for_secc on the p edges: outside [0, 1] (NaN included) raises; -0.0, 1.0 and 5e-324 edit as the restatement does."""
    x = _face_img(128, [(40, 48, 36, 52), (40, 47, 70, 86)])
    img = torch.from_numpy(x).to(DEV)
    for p in P_EDGES:
        if bref.p_control(p) is None:
            with pytest.raises(ValueError):
                r3.blink_eye_for_secc(img, p)
        else:
            got = r3.blink_eye_for_secc(img, p).cpu().numpy()
            assert np.array_equal(got.view(np.uint32), bref.blink(x, p)[0].view(np.uint32)), p


# ---- the recorded launches -----------------------------------------------------------------------------------------------------------------
class _SeccCalls(Recorder):
    """Records every SECC renderer / blink launch as its secc_launch_reference signature."""

    def __init__(self, lib):
        super().__init__(lib, lr.LAUNCHES.__contains__)

    def record(self, name, args):
        return lr.signature(name, args, capi._SIGNATURES[name][1])


def _backbone(seed=7):
    bb = r3.SegFormerSECC2PlaneBackbone()
    bb.load_state_dict(s2p_ref.make_params({k: v.shape for k, v in bb.state_dict().items()}, seed), strict=True)
    return bb.to(DEV).eval()


def _table_rows(N, F):
    """{signature: row tag} of every table above."""
    out = {}
    for row in VERTEX_ROWS:
        out.setdefault(vertex_signature(row), row[0])
    for row in RASTER_ROWS:
        for s in raster_signatures(row, N, F):
            out.setdefault(s, row[0])
    for row in BLINK_ROWS:
        out.setdefault(blink_signature(row), row[0])
    return out


@torch.no_grad()
def test_secc_launches_have_rows(bfm):
    kw, _ = bfm
    r = renderer(kw, 512)
    r224 = r3.SECC_Renderer(device=DEV, **kw)
    N, F = r.n_verts, r.n_faces
    engines = {}
    for blink in (False, True):
        eng = engine.FrameEngine(batch=4, sr_mode='tc', hp={'num_samples_fine': 0}, out_uint8=True, secc2plane=_backbone(), secc_renderer=r,
                                 blink=blink, use_graph=False)
        eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_params(seed=5))
        engines[blink] = eng
    c = syn.make_coeffs(4, seed=3, yaw=0.3)
    cs = torch.cat([c['id'][:1], c['exp'][:1]], 1).to(DEV)
    cano = syn.make_planes(1, seed=1).to(DEV)
    cams = syn.make_cameras(4, seed=2).to(DEV)
    u_c = syn.make_jitter(4, 4096, 48, 0, seed=3)[0].to(DEV)
    img = r.render(cs)[1][0].clone()
    torch.cuda.synchronize()
    recorded = []

    def run(shape, fn, **kw_plan):
        rec.calls.clear()
        fn()
        torch.cuda.synchronize()
        got = list(rec.calls)
        assert_plan(got, lr.launch_plan(shape, N, F, r.tan_half, **kw_plan), shape)
        recorded.extend((shape, s) for s in got)

    with _SeccCalls(capi.lib()) as rec:
        for blink, eng in engines.items():
            rows = torch.cat([c['id'], c['exp']] + ([torch.tensor([[1., 8.], [0., 0.], [5., 10.], [3., 9.]])] if blink else []), 1).to(DEV)
            run('begin_planes', lambda: eng.begin_planes(cano, coeff_src=cs))
            run('step_blink' if blink else 'step', lambda: eng.step(None, cams, u_c, coeff=rows), B=4)
        run('forward', lambda: r224(*(c[k].to(DEV) for k in ('id', 'exp', 'euler', 'trans'))), B=4)
        run('blink_eye_for_secc', lambda: r3.blink_eye_for_secc(img, 0.5), img_size=512)
    table = _table_rows(N, F)
    missing = [f'{shape}: {s}' for shape, s in recorded if s not in table]
    launched = {s for _, s in recorded}
    prod = ('engine', 'forward', 'class', 'drop-in')
    stale = [f'{tag}: {s}' for s, tag in table.items() if tag.startswith(prod) and s not in launched]
    assert_rows(missing, stale, 'the engine / class')
