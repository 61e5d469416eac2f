"""The SECC launch checking code on the CPU (tests/secc_launch_reference.py, tests/blink_reference.py):
  - launch_plan's rows are well formed, and the tables of tests/test_gpu_secc_launches.py cover the production rows
  - check_raster accepts a float32 numpy simulation of the raster rules on the hand-placed meshes, and the exact face maps reject the same
    simulation with the tie going to the higher face or without the pz < 0 skip
  - the restatement's blink control rule agrees with schedule_p and with SECC_Renderer.blink's docstring on every control edge."""
import ctypes
import math

import numpy as np
import pytest

import blink_reference as bref
import secc_launch_reference as lr
import secc_render_reference as ref

F32 = np.float32
N_BFM, F_BFM = 150 * 238, 70389


# ---- launch_plan ---------------------------------------------------------------------------------------------------------------------------
SHAPES = ('begin_planes', 'step', 'step_blink', 'forward', 'blink_eye_for_secc')


def _plan(shape):
    return lr.launch_plan(shape, N_BFM, F_BFM, ref.TAN_HALF, img_size=512)


def test_launch_plan_rows_are_well_formed():
    from real3dportrait_b200 import _capi as capi
    for shape in SHAPES:
        plan = _plan(shape)
        assert plan, shape
        for fn, vals, nonnull in plan:
            types = capi._SIGNATURES[fn][1]
            n_vals = sum(t is not capi._P for t in types)
            assert len(vals) == n_vals and len(nonnull) == len(lr.OPTIONAL[fn]), (shape, fn)
            assert all(types[i] is capi._P for i in lr.OPTIONAL[fn])
            assert all(isinstance(v, int) or ctypes.c_float(v).value == v for v in vals), (shape, fn, vals)
    bp, st, sb = _plan('begin_planes'), _plan('step'), _plan('step_blink')
    assert [r[0] for r in bp] == ['r3dp_secc_vertices', 'r3dp_secc_raster', 'r3dp_secc_resolve'] * 2
    assert bp[0][1][:6] == (N_BFM, 80, 64, 144, 144, 1) and bp[0][2] == (False, False) and bp[2][2] == (False,)
    assert st[0][1][3:6] == (144, 144, 4) and sb[0][1][3:6] == (146, 146, 4)
    assert sb[-1] == ('r3dp_secc_blink', (4, 512, 146), (False, True)) and len(sb) == len(st) + 1
    fw = _plan('forward')
    assert fw[0][1][3:5] == (80, 64) and fw[0][2] == (True, True) and fw[1][1][3] == 224 and fw[2][2] == (True,)
    assert _plan('blink_eye_for_secc') == [('r3dp_secc_blink', (1, 512, 0), (True, False))]
    # a recorded call maps onto the same form
    args = [None, None, N_BFM, 80, 64, ctypes.c_void_p(16), 146, ctypes.c_void_p(16 + 320), 146, ctypes.c_void_p(0), ctypes.c_void_p(0), 4,
            10.0, ref.TAN_HALF, None, None]
    assert lr.signature('r3dp_secc_vertices', args, capi._SIGNATURES['r3dp_secc_vertices'][1]) == sb[0]


def test_tables_cover_the_plan():
    gpu = pytest.importorskip('test_gpu_secc_launches')
    table = gpu._table_rows(N_BFM, F_BFM)
    for shape in SHAPES:
        for s in _plan(shape):
            assert s in table, f'{shape}: {s} has no table row'
    # and every production row of the tables is in the plan
    planned = {s for shape in SHAPES for s in _plan(shape)}
    prod = [(s, tag) for s, tag in table.items() if tag.startswith(('engine', 'forward', 'class', 'drop-in'))]
    assert prod and all(s in planned for s, _ in prod), [tag for s, tag in prod if s not in planned]


# ---- check_raster on a float32 simulation --------------------------------------------------------------------------------------------------
def _edge(px, py, ax, ay, bx, by):
    return (px - ax) * (by - ay) - (py - ay) * (bx - ax)


def simulate(scene, tie='low', pz_skip=True):
    """The raster and resolve rules in float32, one face at a time over its bounding box: -> (face [1,S,S], secc [1,3,S,S] float64)."""
    S, v, faces, ncc = scene['S'], scene['v'][0].astype(F32), scene['faces'], scene['ncc'].astype(F32)
    eps = F32(1e-8)
    pix = (F32(-1) + (F32(2) * (S - 1 - np.arange(S)).astype(F32) + F32(1)) / F32(S)).astype(F32)
    best = np.full((S, S), np.inf, F32)
    face = np.full((S, S), -1, np.int64)
    wsave = np.zeros((S, S, 3), F32)

    def bary(px, py, a, b, c):
        area = _edge(c[0], c[1], a[0], a[1], b[0], b[1]) + eps
        b0, b1, b2 = _edge(px, py, b[0], b[1], c[0], c[1]) / area, _edge(px, py, c[0], c[1], a[0], a[1]) / area, \
            _edge(px, py, a[0], a[1], b[0], b[1]) / area
        t0, t1, t2 = b0 * b[2] * c[2], a[2] * b1 * c[2], a[2] * b[2] * b2
        den = np.maximum(t0 + t1 + t2, eps)
        return t0 / den, t1 / den, t2 / den

    for f, (i0, i1, i2) in enumerate(faces):
        a, b, c = v[i0], v[i1], v[i2]
        A = _edge(a[0], a[1], b[0], b[1], c[0], c[1])
        if max(a[2], b[2], c[2]) < 0 or -eps <= A <= eps:
            continue
        xs, ys = np.array([a[0], b[0], c[0]]), np.array([a[1], b[1], c[1]])
        if not (xs.max() >= -1.5 and xs.min() <= 1.5 and ys.max() >= -1.5 and ys.min() <= 1.5):
            continue
        cols = np.nonzero((pix <= xs.max()) & (pix >= xs.min()))[0]
        rows = np.nonzero((pix <= ys.max()) & (pix >= ys.min()))[0]
        if not cols.size or not rows.size:
            continue
        py, px = np.meshgrid(pix[rows], pix[cols], indexing='ij')
        w0, w1, w2 = bary(px, py, a, b, c)
        pz = w0 * a[2] + w1 * b[2] + w2 * c[2]
        cov = (w0 > 0) & (w1 > 0) & (w2 > 0)
        if pz_skip:
            cov &= ~(pz < 0)
        pz = np.abs(pz)
        sub = best[np.ix_(rows, cols)]
        win = cov & ((pz < sub) | ((pz == sub) & (tie == 'high')))
        rr, cc = np.nonzero(win)
        best[rows[rr], cols[cc]] = pz[rr, cc]
        face[rows[rr], cols[cc]] = f
        wsave[rows[rr], cols[cc]] = np.stack([w0[rr, cc], w1[rr, cc], w2[rr, cc]], -1)
    secc = np.full((3, S, S), -1.0)
    hit = (face >= 0) & ~((face == 0) & bool(scene['drop_face0']))
    fv = faces[np.maximum(face, 0)]
    col = (wsave[..., None] * ncc[fv]).sum(2, dtype=F32)
    secc[:, hit] = (F32(2) * col[hit] - F32(1)).T
    return face[None], secc[None]


def _check(scene, face, secc):
    m = {'faces': scene['faces'], 'ncc': scene['ncc']}
    want = lr.expected_faces(scene)
    assert np.array_equal(face[0], want), f'{scene["name"]}: {(face[0] != want).sum()} pixels differ from the exact face map'
    lr.check_raster(m, scene['v'], np.zeros((1, 2)), scene['S'], face, secc, None, scene['name'], scene['drop_face0'])


@pytest.mark.parametrize('scene', lr.hand_scenes(), ids=[s['name'] for s in lr.hand_scenes()])
def test_check_raster_accepts_the_float32_rules(scene):
    face, secc = simulate(scene)
    for rc in scene['empty']:
        assert face[0][rc] == -1
    for rc in scene['covered']:
        assert face[0][rc] >= 0
    _check(scene, face, secc)


@pytest.mark.parametrize('mutant', [{'tie': 'high'}, {'pz_skip': False}], ids=['tie-to-higher-face', 'no-pz-skip'])
def test_hand_placed_meshes_reject_raster_mutants(mutant):
    failed = []
    for scene in lr.hand_scenes():
        face, secc = simulate(scene, **mutant)
        try:
            _check(scene, face, secc)
        except AssertionError:
            failed.append(scene['name'])
    assert failed, f'no hand-placed mesh tells {mutant} apart'


# ---- the blink control rule ----------------------------------------------------------------------------------------------------------------
NAN, INF = float('nan'), float('inf')
# (t, T) -> the docstring's answer: None (untouched) or p = schedule_p(int(t), int(T))
ROW_EDGES = {(0.5, 8.0): 0.0, (2.7, 8.9): bref.schedule_p(2, 8), (7.9, 8.0): bref.schedule_p(7, 8), (0.5, 0.7): None, (1.5, 1.7): None,
             (8, 8): None, (9, 8): None, (0, 1): 0.0, (3, 4096): bref.schedule_p(3, 4096), (3, 4097): None,
             (4095, 4096): bref.schedule_p(4095, 4096), (-1, 8): None, (-0.5, 8): None, (3, -8): None, (NAN, 8): None, (3, NAN): None,
             (INF, 8): None, (3, INF): None, (-INF, 8): None, (3, -INF): None, (4, 8): 1.0, (0, 0): None}


def test_rows_control_rule():
    for (t, T), want in ROW_EDGES.items():
        got = bref.rows_control(t, T)
        assert (got is None) == (want is None) and (want is None or got == want), ((t, T), got, want)
    # integer rows of the period schedule: exactly schedule_p, in Python's evaluation order
    for T in range(1, 13):
        for t in range(T):
            assert bref.rows_control(float(t), float(T)) == bref.schedule_p(t, T) == -4 / T ** 2 * t ** 2 + 4 / T * t
        assert bref.rows_control(float(T), float(T)) is None
    assert bref.schedule_p(3, 4096) > 0 and bref.rows_control(3, 4097) is None
    # the GPU table runs every one of these edges
    gpu = pytest.importorskip('test_gpu_secc_launches')
    assert {(float(t), float(T)) for t, T in gpu.ROW_EDGES} >= {(float(t), float(T)) for t, T in ROW_EDGES if not (t == 0 and T == 0)} - \
        {(a, b) for a, b in ROW_EDGES if math.isnan(a) or math.isnan(b)}


def test_p_control_rule():
    assert bref.p_control(-0.0) == 0.0 and math.copysign(1, bref.p_control(-0.0)) == -1     # p = -0.0: edited as p = 0 (quantised)
    assert bref.p_control(NAN) is None and bref.p_control(float(np.nextafter(1.0, 2.0))) is None and bref.p_control(-1e-300) is None
    assert bref.p_control(1.0) == 1.0 and bref.p_control(5e-324) == 5e-324 and bref.p_control(INF) is None
    x = bref.encode(np.full((3, 64, 64), 150))
    assert np.array_equal(bref.blink(x, -0.0)[1], bref.blink(x, 0.0)[1])
