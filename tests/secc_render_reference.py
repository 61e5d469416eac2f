"""Float64 restatement of the reference's SECC renderer (deep_3drecon/secc_renderer.py with ParametricFaceModel and MeshRenderer on pytorch3d's
MeshRasterizer), written from their sources; the checker of r3dp_secc_* and SECC_Renderer.  numpy only.

  shape     s = idBase id + exBase exp + mean (mean recentred at load)                          bfm.py:78-81, 102-115
  pose      v = (Rz Ry Rx) s + trans, z = 10 - z                                                  bfm.py:204-243, 260-270
  camera    x negated (mesh_renderer.py:69-71); x_ndc = x / (z tan(fov/2)), y_ndc likewise, z stays the view z
  pixels    row r, column c at NDC (1 - (2c+1)/S, 1 - (2r+1)/S)
  faces     skipped if max z < 0 or |A| <= 1e-8 (A the signed edge-function area); b_i = edge_i / (A + 1e-8);
            w_i = b_i z_j z_k / max(sum, 1e-8); covered iff all w_i > 0; pz = sum w_i z_i, skipped if pz < 0; nearest pz wins, ties to the lower face
  image     secc = 2 mask sum_i w_i ncc_i - 1; mask = packed face index > 0 (face 0 of image 0 of a call is background)"""
from __future__ import annotations

import numpy as np

EPS = 1e-8
TAN_HALF = 112.0 / 1015.0          # tan(fov / 2) with fov = 2 atan(center / focal)


def load(bfm_folder, ncc_path, eye_faces):
    """The reference's files -> float64 mean [N,3] (recentred as the reference does, in float32), bases [3N,K], faces [F,3] 0-based, ncc [N,3]."""
    import os
    from scipy.io import loadmat
    m = loadmat(os.path.join(bfm_folder, 'BFM_model_front.mat'))
    mean = m['meanshape'].astype(np.float32).reshape(-1, 3)
    mean = (mean - np.mean(mean, axis=0, keepdims=True)).astype(np.float64)
    tri = m['tri'].astype(np.int64) - 1
    drop = set()
    for p in eye_faces:
        drop.update((np.load(p).astype(np.int64) - 1).tolist())
    faces = np.array([t for i, t in enumerate(tri) if i not in drop])
    ncc = np.load(ncc_path).astype(np.float64).T
    return {'mean': mean, 'id_base': m['idBase'].astype(np.float32).astype(np.float64),
            'exp_base': m['exBase'].astype(np.float32).astype(np.float64), 'faces': faces, 'ncc': ncc}


def rotation(euler):
    """euler [B,3] -> R = Rz Ry Rx [B,3,3] (v = R s; the reference's rot is R^T on row vectors)."""
    x, y, z = (np.asarray(euler, np.float64)[:, i] for i in range(3))
    o, n = np.ones_like(x), np.zeros_like(x)
    rx = np.stack([o, n, n, n, np.cos(x), -np.sin(x), n, np.sin(x), np.cos(x)], 1).reshape(-1, 3, 3)
    ry = np.stack([np.cos(y), n, np.sin(y), n, o, n, -np.sin(y), n, np.cos(y)], 1).reshape(-1, 3, 3)
    rz = np.stack([np.cos(z), -np.sin(z), n, np.sin(z), np.cos(z), n, n, n, o], 1).reshape(-1, 3, 3)
    return rz @ ry @ rx


def shape(bfm, id, exp):
    """-> s [B,N,3] and the sum of |terms| of each component [B,N,3] (for the fp32 error bar)."""
    id, exp = np.asarray(id, np.float64), np.asarray(exp, np.float64)
    s = id @ bfm['id_base'].T + exp @ bfm['exp_base'].T + bfm['mean'].reshape(1, -1)
    a = np.abs(id) @ np.abs(bfm['id_base']).T + np.abs(exp) @ np.abs(bfm['exp_base']).T + np.abs(bfm['mean']).reshape(1, -1)
    B = s.shape[0]
    return s.reshape(B, -1, 3), a.reshape(B, -1, 3)


def vertices(bfm, id, exp, euler=None, trans=None):
    """-> [B,N,3] (x_ndc, y_ndc, z_view) float64."""
    s, _ = shape(bfm, id, exp)
    B = s.shape[0]
    R = rotation(np.zeros((B, 3)) if euler is None else euler)
    t = np.zeros((B, 3)) if trans is None else np.asarray(trans, np.float64)
    v = np.einsum('bij,bnj->bni', R, s) + t[:, None]
    z = 10.0 - v[..., 2]
    return np.stack([-v[..., 0] / (z * TAN_HALF), v[..., 1] / (z * TAN_HALF), z], -1)


def pixel_ndc(i, S):
    return 1.0 - (2.0 * np.asarray(i, np.float64) + 1.0) / S


def _edge(px, py, ax, ay, bx, by):
    return (px - ax) * (by - ay) - (py - ay) * (bx - ax)


def raster_pairs(v, faces, S, slack_px=0.0):
    """Every (pixel, face) pair of one frame whose pixel centre lies in the face's bounding box widened by slack_px, for the faces that pass
    the culls.  -> dict of flat arrays: pix (r*S + c), face, pz, covered (the rules above), dist (signed distance of the centre to the nearest
    edge in pixels, > 0 inside), w [n,3] (corrected barycentrics)."""
    v = np.asarray(v, np.float64)
    faces = np.asarray(faces)
    a, b, c = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
    A = _edge(a[:, 0], a[:, 1], b[:, 0], b[:, 1], c[:, 0], c[:, 1])
    zmax = np.maximum(np.maximum(a[:, 2], b[:, 2]), c[:, 2])
    keep = np.nonzero(~(zmax < 0) & ~((A <= EPS) & (A >= -EPS)))[0]
    xs, ys = np.stack([a[keep, 0], b[keep, 0], c[keep, 0]]), np.stack([a[keep, 1], b[keep, 1], c[keep, 1]])
    sl = 2.0 * slack_px / S
    xmin, xmax, ymin, ymax = xs.min(0) - sl, xs.max(0) + sl, ys.min(0) - sl, ys.max(0) + sl
    # column c has x = 1 - (2c+1)/S: columns inside [xmin, xmax]
    c0 = np.clip(np.ceil((S * (1 - xmax) - 1) / 2), 0, S).astype(np.int64)
    c1 = np.clip(np.floor((S * (1 - xmin) - 1) / 2), -1, S - 1).astype(np.int64)
    r0 = np.clip(np.ceil((S * (1 - ymax) - 1) / 2), 0, S).astype(np.int64)
    r1 = np.clip(np.floor((S * (1 - ymin) - 1) / 2), -1, S - 1).astype(np.int64)
    nw, nh = c1 - c0 + 1, r1 - r0 + 1
    ok = (nw > 0) & (nh > 0)
    keep, c0, r0, nw, nh = keep[ok], c0[ok], r0[ok], nw[ok], nh[ok]
    out = {k: [] for k in ('pix', 'face', 'pz', 'covered', 'dist', 'w')}
    if keep.size == 0:
        return {k: np.zeros((0, 3) if k == 'w' else 0) for k in out}
    for dy in range(int(nh.max())):
        for dx in range(int(nw.max())):
            sel = np.nonzero((nh > dy) & (nw > dx))[0]
            if sel.size == 0:
                continue
            f = keep[sel]
            r, cc = r0[sel] + dy, c0[sel] + dx
            px, py = pixel_ndc(cc, S), pixel_ndc(r, S)
            fa, fb, fc = a[f], b[f], c[f]
            e0 = _edge(px, py, fb[:, 0], fb[:, 1], fc[:, 0], fc[:, 1])
            e1 = _edge(px, py, fc[:, 0], fc[:, 1], fa[:, 0], fa[:, 1])
            e2 = _edge(px, py, fa[:, 0], fa[:, 1], fb[:, 0], fb[:, 1])
            area = _edge(fc[:, 0], fc[:, 1], fa[:, 0], fa[:, 1], fb[:, 0], fb[:, 1]) + EPS
            b0, b1, b2 = e0 / area, e1 / area, e2 / area
            t0, t1, t2 = b0 * fb[:, 2] * fc[:, 2], fa[:, 2] * b1 * fc[:, 2], fa[:, 2] * fb[:, 2] * b2
            den = np.maximum(t0 + t1 + t2, EPS)
            w = np.stack([t0 / den, t1 / den, t2 / den], 1)
            pz = (w * np.stack([fa[:, 2], fb[:, 2], fc[:, 2]], 1)).sum(1)
            sgn = np.sign(A[f])
            lens = [np.hypot(fc[:, 0] - fb[:, 0], fc[:, 1] - fb[:, 1]), np.hypot(fa[:, 0] - fc[:, 0], fa[:, 1] - fc[:, 1]),
                    np.hypot(fb[:, 0] - fa[:, 0], fb[:, 1] - fa[:, 1])]
            dist = np.min(np.stack([sgn * e / np.maximum(l, 1e-300) for e, l in zip((e0, e1, e2), lens)]), 0) * (S / 2)
            inbox = (px <= xs.max(0)[ok][sel]) & (px >= xs.min(0)[ok][sel]) & (py <= ys.max(0)[ok][sel]) & (py >= ys.min(0)[ok][sel])
            covered = inbox & (w > 0).all(1) & ~(pz < 0)
            out['pix'].append(r * S + cc); out['face'].append(f); out['pz'].append(pz)
            out['covered'].append(covered); out['dist'].append(dist); out['w'].append(w)
    return {k: np.concatenate(v_) for k, v_ in out.items()}


def resolve(pairs, S):
    """Nearest covered pz per pixel, ties to the lower face -> face [S*S] (-1 empty), w [S*S,3]."""
    face = np.full(S * S, -1, np.int64)
    w = np.zeros((S * S, 3))
    cov = np.nonzero(pairs['covered'])[0]
    if cov.size:
        o = cov[np.lexsort((pairs['face'][cov], pairs['pz'][cov], pairs['pix'][cov]))]
        first = np.ones(o.size, bool)
        first[1:] = pairs['pix'][o][1:] != pairs['pix'][o][:-1]
        o = o[first]
        face[pairs['pix'][o]] = pairs['face'][o]
        w[pairs['pix'][o]] = pairs['w'][o]
    return face, w


def render(verts, faces, ncc, S):
    """verts [B,N,3] (vertices()), faces [F,3], ncc [N,3] -> mask [B,1,S,S], secc [B,3,S,S], face [B,S,S] (the pix_to_face of each image)."""
    B = verts.shape[0]
    faces = np.asarray(faces)
    masks, seccs, fs = [], [], []
    for b in range(B):
        f, w = resolve(raster_pairs(verts[b], faces, S), S)
        hit = f >= 0
        col = np.zeros((S * S, 3))
        vi = faces[np.maximum(f, 0)]
        col[hit] = (w[hit, :, None] * ncc[vi[hit]]).sum(1)
        m = hit & ~((b == 0) & (f == 0))                 # pix_to_face > 0 on the packed index
        masks.append(m.reshape(1, S, S).astype(np.float64))
        seccs.append((2 * m[:, None] * col - 1).T.reshape(3, S, S))
        fs.append(f.reshape(S, S))
    return np.stack(masks), np.stack(seccs), np.stack(fs)
