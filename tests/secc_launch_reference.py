"""Checking code of the SECC renderer's kernels (r3dp_secc_vertices / _raster / _resolve) and blink (r3dp_secc_blink), shared by the tests:

  vertex_bar    float64 vertices and their fp32 error bound: gamma_{K+1} sum |terms| of the K-term dot product, propagated through the pose
                and the projection
  raster_err    per frame, the NDC error of x / y and the relative error of z that the raster check allows (from vertex_bar, or 0 for vertices
                placed by hand)
  check_raster  the kernel's face map and images against the float64 oracle (secc_render_reference): decisive pixels take the oracle's face,
                ambiguous ones a face the oracle finds within delta (or none), values within value_bar where the faces agree
  launch_plan   the (entry point, non-pointer arguments, which optional pointers are non-null) rows of each call shape of SECC_Renderer,
                FrameEngine and blink_eye_for_secc, written from their contract; a recorded-launch test holds it to what the code launches
numpy only."""
from __future__ import annotations

import ctypes

import numpy as np

import secc_render_reference as ref
from launch_harness import given

U = 2.0 ** -24
CAMERA_DISTANCE = 10.0
#: the optional pointer arguments of each launch (positions in the C argument list): NULL or not is part of a launch's row
OPTIONAL = {'r3dp_secc_vertices': (9, 10), 'r3dp_secc_raster': (), 'r3dp_secc_resolve': (9,), 'r3dp_secc_blink': (3, 4)}
LAUNCHES = tuple(OPTIONAL)


def gamma(n):
    return n * U / (1 - n * U)


def _np(x, B=None, n=3):
    if x is None:
        return None
    if hasattr(x, 'detach'):
        x = x.detach().cpu().double().numpy()
    return np.asarray(x, np.float64)


def vertex_bar(m, c):
    """c: id [B,n_id], exp [B,n_exp], euler / trans [B,3] or None (zero pose, as the kernel reads NULL) as tensors or arrays ->
    (float64 vertices [B,N,3] (x_ndc, y_ndc, z_view), their fp32 error bound [B,N,3])."""
    idv, expv = _np(c['id']), _np(c['exp'])
    B = idv.shape[0]
    euler, trans = _np(c.get('euler')), _np(c.get('trans'))
    euler = np.zeros((B, 3)) if euler is None else euler
    t = np.zeros((B, 3)) if trans is None else trans
    s, terms = ref.shape(m, idv, expv)
    K = idv.shape[1] + expv.shape[1]
    e_s = gamma(K + 1) * terms
    R = ref.rotation(euler)
    e_r = 8 * U + 2 * U * np.abs(euler).max()                           # sincospif of x / pi: argument and result rounding, 2-3 factor products
    aR = np.abs(R)
    e_v = np.einsum('bij,bnj->bni', aR, e_s) + e_r * np.abs(s).sum(-1, keepdims=True) \
        + gamma(3) * (np.einsum('bij,bnj->bni', aR, np.abs(s)) + np.abs(t)[:, None])
    v = ref.vertices(m, idv, expv, euler, t)
    z = v[..., 2]
    e_z = e_v[..., 2] + U * np.abs(z)
    rel = e_z / np.abs(z) + 3 * U
    tz = np.abs(z) * ref.TAN_HALF
    e_x = e_v[..., 0] / tz + np.abs(v[..., 0]) * rel
    e_y = e_v[..., 1] / tz + np.abs(v[..., 1]) * rel
    return v, np.stack([e_x, e_y, e_z], -1)


def raster_err(v, bar):
    """Per frame [B,2]: the largest x / y vertex error (NDC) and the largest relative z error."""
    return np.stack([bar[..., :2].max((1, 2)), (bar[..., 2] / np.abs(v[..., 2])).max(1)], 1)


def value_bar(m, vb, f, d_ndc):
    """Per pixel and channel, the fp32 bar of secc for winning faces f [n] of one frame (vertices vb [N,3]) with vertex error d_ndc:
    |dw_i| <= (d_ndc 2 perimeter / |A| + 4u) (zmax / zmin)^2 for each barycentric, times 2 spread(ncc) as sum_i dw_i ~ 0, + 12u of rounding.
    -> (bar [n,3], the faces' NCC codes [n,3 verts,3 ch])."""
    fv = m['faces'][f]
    P = vb[fv]                                                          # [n,3 verts,3]
    A = np.abs((P[:, 0, 0] - P[:, 1, 0]) * (P[:, 2, 1] - P[:, 1, 1]) - (P[:, 0, 1] - P[:, 1, 1]) * (P[:, 2, 0] - P[:, 1, 0]))
    per = sum(np.hypot(*(P[:, i, :2] - P[:, (i + 1) % 3, :2]).T) for i in range(3))
    zr = (P[:, :, 2].max(1) / P[:, :, 2].min(1)) ** 2
    dw = 3 * (d_ndc * 2 * per / A + 4 * U) * zr
    ncc = m['ncc'][fv]
    return 2 * dw[:, None] * (ncc.max(1) - ncc.min(1)) + 12 * U, ncc


def check_raster(m, v, err, S, face, secc, mask, label, drop_face0=True):
    """m: faces [F,3] and ncc [N,3]; v [B,N,3] float64 vertices; err [B,2] (raster_err; zeros for exact hand-placed vertices); face [B,S,S]
    the kernel's winning face per pixel (-1 none), secc [B,3,S,S], mask [B,1,S,S] or None, float64.  Asserts the bars; returns the stats."""
    faces = m['faces']
    B = v.shape[0]
    stats = {'decisive': 0, 'ambiguous': 0, 'value_ratio': 0.0, 'value_err': 0.0}
    for b in range(B):
        d_ndc = 2 * err[b, 0] + 4 * U                                  # vertex error + the pixel centre's rounding
        d_px = d_ndc * S / 2 + 1e-6
        d_z = err[b, 1] + 16 * U
        pairs = ref.raster_pairs(v[b], faces, S, slack_px=4 * d_px)
        f_ref, w_ref = ref.resolve(pairs, S)
        near = pairs['dist'] > -d_px
        cov = pairs['covered'].astype(bool)[near]
        pix, pf, ppz, pd = pairs['pix'][near].astype(np.int64), pairs['face'][near].astype(np.int64), pairs['pz'][near], pairs['dist'][near]
        # the winner's own pair
        win = f_ref[pix] == pf
        wpz = np.full(S * S, np.inf)
        wd = np.full(S * S, -np.inf)
        wpz[pix[win & cov]] = ppz[win & cov]
        wd[pix[win & cov]] = pd[win & cov]
        amb = np.zeros(S * S, bool)
        amb[pix[~win & ~(ppz > wpz[pix] * (1 + d_z))]] = True           # another face within delta and not clearly farther
        amb |= (f_ref >= 0) & (wd <= d_px)                              # the centre is within delta of the winner's boundary
        amb |= (f_ref < 0) & np.isin(np.arange(S * S), pix)             # no winner, but a face comes within delta
        got = face[b].reshape(-1)
        dec = ~amb
        bad = dec & (got != f_ref)
        assert not bad.any(), f'{label} b={b}: {bad.sum()} decisive pixels differ, e.g. {np.nonzero(bad)[0][:5]}'
        ai = np.nonzero(amb)[0]
        if ai.size:
            allowed = np.unique(pix.astype(np.int64) * (faces.shape[0] + 1) + pf)
            ga = got[ai]
            ok = (ga == -1) | np.isin(ai.astype(np.int64) * (faces.shape[0] + 1) + ga, allowed)
            assert ok.all(), f'{label} b={b} pixel {ai[~ok][0]}: face {ga[~ok][0]}'
        stats['decisive'] += int(dec.sum())
        stats['ambiguous'] += int(amb.sum())
        # values where the faces agree
        same = np.nonzero((got == f_ref) & (f_ref >= 0))[0]
        vbar, ncc = value_bar(m, v[b], f_ref[same], d_ndc)
        col = (w_ref[same][:, :, None] * ncc).sum(1)
        drop = (b == 0) & (f_ref[same] == 0) & bool(drop_face0)          # the packed face 0: background
        want = np.where(drop[:, None], -1.0, 2 * col - 1)
        gotv = secc[b].reshape(3, -1)[:, same].T
        err_v = np.abs(gotv - want)
        stats['value_ratio'] = max(stats['value_ratio'], float((err_v / vbar).max(initial=0)))
        stats['value_err'] = max(stats['value_err'], float(err_v.max(initial=0)))
        assert (err_v <= vbar).all(), f'{label} b={b}: value error {err_v.max():.2e}'
        bg = (got < 0) | ((b == 0) & (got == 0) & bool(drop_face0))
        assert (secc[b].reshape(3, -1)[:, bg] == -1).all(), f'{label} b={b}: background secc is not -1'
        if mask is not None:
            assert (mask[b, 0].reshape(-1)[bg] == 0).all() and (mask[b, 0].reshape(-1)[~bg] == 1).all(), f'{label} b={b}: mask'
    print(f'{label}: decisive {stats["decisive"]}, ambiguous {stats["ambiguous"]}, secc max |err| {stats["value_err"]:.2e}, '
          f'worst err/bar {stats["value_ratio"]:.3f}')
    return stats


# ---- launch rows ----------------------------------------------------------------------------------------------------------------------------
def signature(fn, args, types):
    """A call of one of LAUNCHES -> (entry point, its non-pointer arguments with floats rounded to fp32 as the C side receives them, the
    non-NULL flags of its optional pointers).  types: the entry point's ctypes argument types (capi._SIGNATURES[fn][1])."""
    vals = tuple(ctypes.c_float(a).value if t is ctypes.c_float else a for a, t in zip(args, types) if t is not ctypes.c_void_p)
    nonnull = tuple(given(args[i]) for i in OPTIONAL[fn])
    return fn, vals, nonnull


def render_rows(N, F, n_id, n_exp, ids, exps, B, S, pose, drop_face0, with_mask, tan_half):
    """The three launches of one SECC_Renderer call (render() or forward())."""
    tan = ctypes.c_float(tan_half).value
    return [('r3dp_secc_vertices', (N, n_id, n_exp, ids, exps, B, CAMERA_DISTANCE, tan), (pose, pose)),
            ('r3dp_secc_raster', (N, F, B, S), ()),
            ('r3dp_secc_resolve', (N, B, S, int(drop_face0)), (with_mask,))]


def blink_row(B, S, stride, with_p):
    """One r3dp_secc_blink call: p per image (stride 0) or (t, T) rows at a row stride."""
    return ('r3dp_secc_blink', (B, S, stride), (with_p, not with_p))


def launch_plan(shape, N, F, tan_half, n_id=80, n_exp=64, B=4, S=None, img_size=None):
    """The launch rows of one call shape, in launch order:
      'begin_planes'        FrameEngine.begin_planes(coeff_src=c [1, n_id + n_exp]): render(c), then render of c with exp zeroed; zero pose
                            (euler = trans = NULL), rows at stride n_id + n_exp with exp at row + n_id, size S (the renderer's, 512 for the engine)
      'step', 'step_blink'  one FrameEngine step at batch B: render(coeff) as above at B (rows [id | exp], or [id | exp | t | T] at stride
                            n_id + n_exp + 2 with blink=True), then with blink=True one r3dp_secc_blink on the batch's (t, T) columns
      'forward'             SECC_Renderer.forward(id, exp, euler, trans) at batch B: separate id / exp tensors (strides n_id, n_exp), pose and mask
                            given, size S (224 by default, 2 x 112)
      'blink_eye_for_secc'  the drop-in on one [3, img_size, img_size] image: p given, no rows"""
    K = n_id + n_exp
    if shape == 'begin_planes':
        return render_rows(N, F, n_id, n_exp, K, K, 1, S or 512, False, True, False, tan_half) * 2
    if shape in ('step', 'step_blink'):
        W = K + (2 if shape == 'step_blink' else 0)
        rows = render_rows(N, F, n_id, n_exp, W, W, B, S or 512, False, True, False, tan_half)
        return rows + ([blink_row(B, S or 512, W, False)] if shape == 'step_blink' else [])
    if shape == 'forward':
        return render_rows(N, F, n_id, n_exp, n_id, n_exp, B, S or 224, True, True, True, tan_half)
    if shape == 'blink_eye_for_secc':
        return [blink_row(1, img_size, 0, True)]
    raise ValueError(shape)


# ---- hand-placed meshes -------------------------------------------------------------------------------------------------------------------
def _scene(name, S, verts, faces, drop_face0=0, empty=(), covered=()):
    v = np.asarray(verts, np.float64)
    assert (v.astype(np.float32).astype(np.float64) == v).all(), f'{name}: vertices must be exact in fp32'
    n = v.shape[0]
    ncc = ((np.arange(3 * n).reshape(n, 3) * 7919) % 97 / 96.0).astype(np.float32).astype(np.float64)   # distinct codes per vertex
    return {'name': name, 'S': S, 'v': v[None], 'faces': np.asarray(faces, np.int64), 'ncc': ncc, 'drop_face0': drop_face0,
            'empty': list(empty), 'covered': list(covered)}


def hand_scenes():
    """Vertex buffers placed by hand in NDC (x, y, z_view), exact in binary at power-of-two S, so every raster decision is exact: the expected
    face map is the float64 oracle's, and 'empty' / 'covered' list pixels (r, c) whose answer is known by construction.
      edge        a square split along its diagonal, which passes through the pixel centres (r, r): covered by neither face
      cull        faces touching x = +-1.5 / y = +-1.5 from inside and just beyond, and one screen-filling face with vertices on the limit
      z0          a face with one vertex behind the camera (z = -1): its covered centres have pz < 0 and are skipped
      sliver      two 2-wide slivers through a row of pixel centres at S = 4096: |A| = 2^-26 (> 1e-8, rasterised) and 2^-27 (culled)
      subpixel    a face between four pixel centres: covers none
      tie         faces 1 and 2 coincide (same positions, distinct vertices and codes) at pz = 2 over face 0 at pz = 3; face 3 behind all:
                  the lower index wins every tied pixel"""
    out = []
    sq = [(-0.75, -0.75, 2), (0.75, -0.75, 2), (0.75, 0.75, 2), (-0.75, 0.75, 2)]
    out.append(_scene('edge', 8, sq, [(0, 1, 2), (0, 2, 3)], empty=[(r, r) for r in range(1, 7)], covered=[(1, 2), (2, 1), (6, 5)]))
    e = 2.0 ** -22
    cull = [(1.5, -0.5, 2), (2.5, -0.5, 2), (2.0, 0.5, 2),                       # xmin = 1.5: kept, covers no centre
            (1.5 + e, -0.5, 2), (2.5, -0.5, 2), (2.0, 0.5, 2),                   # beyond: culled
            (-2.5, 0.5, 2), (-1.5, 0.5, 2), (-2.0, -0.5, 2),                     # xmax = -1.5
            (-0.5, 1.5 + e, 2), (0.5, 1.5 + e, 2), (0.0, 2.5, 2),                # ymin just beyond 1.5
            (-1.5, -1.5, 4), (1.5, -1.5, 4), (0.0, 1.5, 4)]                      # on the limits: kept, covers most of the screen
    out.append(_scene('cull', 16, cull, [(0, 1, 2), (3, 4, 5), (6, 7, 8), (9, 10, 11), (12, 13, 14)], covered=[(8, 8), (15, 1)]))
    z0 = [(0.0, 0.0, -1), (0.75, 0.375, 1), (-0.375, -0.75, 1), (0.5, 0.75, 2), (0.875, 0.75, 2), (0.875, 0.875, 2)]
    out.append(_scene('z0', 16, z0, [(0, 1, 2), (3, 4, 5)], empty=[(5, 5), (6, 6), (7, 7)]))
    y0, y1 = 2.0 ** -12 - 2.0 ** -35, -2.0 ** -12 - 2.0 ** -35
    sl = [(1.0, y0, 1), (-1.0, y0, 1), (0.0, y0 + 2.0 ** -27, 1), (1.0, y1, 1), (-1.0, y1, 1), (0.0, y1 + 2.0 ** -28, 1)]
    out.append(_scene('sliver', 4096, sl, [(0, 1, 2), (3, 4, 5)], covered=[(2047, 2047), (2047, 2048), (2047, 100)],
                      empty=[(2048, 2047), (2048, 2048), (2046, 2047)]))
    sub = [(-0.0625, -0.0625, 2), (0.0625, -0.0625, 2), (0.0, 0.0625, 2)]
    out.append(_scene('subpixel', 8, sub, [(0, 1, 2)], empty=[(r, c) for r in (3, 4) for c in (3, 4)]))
    tie = [(0.875, -0.875, 3), (-0.875, -0.875, 3), (0.0, 0.875, 3),
           (0.5, -0.5, 2), (-0.5, -0.5, 2), (0.0, 0.5, 2), (0.5, -0.5, 2), (-0.5, -0.5, 2), (0.0, 0.5, 2),
           (1.0, -1.0, 5), (-1.0, -1.0, 5), (0.0, 1.0, 5)]
    for drop in (0, 1):
        out.append(_scene(f'tie-drop{drop}', 16, tie, [(0, 1, 2), (3, 4, 5), (6, 7, 8), (9, 10, 11)], drop_face0=drop,
                          covered=[(8, 8), (9, 6)]))
    return out


def expected_faces(scene):
    """The float64 oracle's face map [S, S] of a hand-placed scene (exact: every decision is exact in binary)."""
    S = scene['S']
    f, _ = ref.resolve(ref.raster_pairs(scene['v'][0], scene['faces'], S), S)
    return f.reshape(S, S)
