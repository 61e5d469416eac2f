"""A numpy restatement of the source images (DESIGN.md, "Source images"), written from the semantics rather than from the reference's code:
per-column torso and neck inpainting, cv2's 5x5 GaussianBlur(sigma 4) as its exact integer form, the head image, and extract_background
through an exact squared EDT with the library's tie rule (nearest source by smallest column, then smallest row)."""
import json

import numpy as np
import torch

from real3dportrait_b200 import synthetic as syn

TORSO_ROWS, NECK_ROWS, PUSH_DOWN = 9, 53, 4
BLUR_TAPS = np.array([48, 53, 54, 53, 48], np.int64)


def _seg6(seg):
    seg = np.asarray(seg)
    return (seg[0] if seg.ndim == 4 else seg).astype(np.float32)


def head_sum(seg):
    s = _seg6(seg)
    return (s[1] + s[3]) + s[5]                                      # float32, in that order


def blur_u8(img):
    """cv2.GaussianBlur(img, (5, 5), 4) on uint8 [H,W,3]: taps along rows, then columns, reflect-101 borders, one rounding."""
    x = img.astype(np.int64)
    p = np.pad(x, ((0, 0), (2, 2), (0, 0)), mode='reflect')         # numpy's 'reflect' is reflect-101
    h = sum(BLUR_TAPS[k] * p[:, k:k + x.shape[1]] for k in range(5))
    p = np.pad(h, ((2, 2), (0, 0), (0, 0)), mode='reflect')
    v = sum(BLUR_TAPS[k] * p[k:k + x.shape[0]] for k in range(5))
    return ((v + (1 << 15)) >> 16).astype(np.uint8)


def darken(v, scale):
    return np.floor(v.astype(np.float64) * scale).astype(np.uint8)


def inpaint_torso(img, seg, tab_torso=None, tab_neck=None):
    """The torso image: head zeroed, per column the darkened upward copies of the top torso pixel (9 rows) and of the dilated neck's
    anchor (53 rows, written after), the blur at the neck copies, zero outside dilated neck | torso | both copies."""
    s = _seg6(seg)
    H, W = s.shape[1:]
    tab_torso = 0.98 ** np.arange(TORSO_ROWS) if tab_torso is None else tab_torso
    tab_neck = 0.98 ** np.arange(NECK_ROWS) if tab_neck is None else tab_neck
    head = head_sum(s) != 0
    neck, torso = s[2] != 0, s[4] != 0
    dil = np.zeros_like(neck)
    for d in range(-3, 4):                                           # rows r-3 .. r+3, nothing outside the image
        lo, hi = max(0, -d), min(H, H - d)
        dil[lo:hi] |= neck[lo + d:hi + d]
    out = img.copy()
    out[head] = 0
    keep = dil | torso
    neck_px = np.zeros((H, W), bool)
    for c in range(W):
        rows = np.nonzero(torso[:, c])[0]
        if rows.size and head[rows[0] - 1, c]:                     # row -1 is row H-1, as numpy indexes
            r = rows[0]
            for k in range(TORSO_ROWS):
                out[r - k, c] = darken(img[r, c], tab_torso[k])
                keep[r - k, c] = True
    for c in range(W):
        rows = np.nonzero(dil[:, c])[0]
        if rows.size and head[rows[0] - 1, c]:
            a = rows[0] + min(rows.size - 1, PUSH_DOWN)
            for k in range(NECK_ROWS):
                out[a - k, c] = darken(img[a, c], tab_neck[k])
                keep[a - k, c] = True
                neck_px[a - k, c] = True
    b = blur_u8(out)
    out[neck_px] = b[neck_px]
    out[~keep] = 0
    return out


def head_image(img, seg):
    out = img.copy()
    out[~(head_sum(seg) > 0.5)] = 0
    return out


def normalise(u8):
    """The reference's ((torch.tensor(u8) - 127.5) / 127.5) as [1,3,H,W] float32."""
    return ((torch.from_numpy(np.ascontiguousarray(u8)) - 127.5) / 127.5).float().unsqueeze(0).permute(0, 3, 1, 2).contiguous()


def frame_interval(n):
    return 5 if n < 100 else 20 if n < 10000 else n // 500


def selected(n):
    i = frame_interval(n)
    return list(range(0, n, i)) if n > i else [0]


def edt(src, rows_per_chunk=8):
    """Exact squared distance of every pixel to the nearest True pixel of src [H,W], and that pixel (row, col): among equidistant ones the
    smallest column, then the smallest row.  Column pass, then a brute-force min over all columns per row (argmin keeps the first)."""
    H, W = src.shape
    big = 1 << 20
    r = np.arange(H)[:, None]
    up = np.where(src, r, -big)
    up = np.maximum.accumulate(up, 0)                                # nearest source at or above
    dn = np.where(src, r, 2 * big)
    dn = np.minimum.accumulate(dn[::-1], 0)[::-1]                    # nearest source at or below
    use_up = (r - up) <= (dn - r)
    near = np.where(use_up, up, dn)                                  # the upper one on a tie
    g2 = np.where(np.abs(near - r) < big // 2, (near - r).astype(np.int64) ** 2, np.int64(1) << 40)
    d2 = np.empty((H, W), np.int64)
    fc = np.empty((H, W), np.int64)
    dx2 = (np.arange(W)[:, None] - np.arange(W)[None]).astype(np.int64) ** 2   # [x, u]
    for r0 in range(0, H, rows_per_chunk):
        cand = dx2[None] + g2[r0:r0 + rows_per_chunk, None, :]      # [rows, x, u]
        u = np.argmin(cand, 2)
        fc[r0:r0 + rows_per_chunk] = u
        d2[r0:r0 + rows_per_chunk] = np.take_along_axis(cand, u[..., None], 2)[..., 0]
    fr = np.take_along_axis(near, fc, 1)
    return d2, fr, fc


def background_distances(segs):
    """Per selected frame in order: max over frames of d^2 to the frame's non-bg pixels, and the first frame attaining it."""
    best = arg = None
    for i, s in enumerate(segs):
        fg = _seg6(s)[0] == 0
        if not fg.any():
            raise ValueError('a frame without a foreground pixel')
        d2 = edt(fg)[0]
        if best is None:
            best, arg = d2, np.zeros(d2.shape, np.int64)
        else:
            arg = np.where(d2 > best, i, arg)
            best = np.maximum(best, d2)
    return best, arg


def extract_background(frames, segs):
    """frames [N,H,W,3] uint8, segs [N,6,H,W] -> the background uint8 [H,W,3] and the fill's source mask (d^2 > 100)."""
    sel = selected(len(frames))
    best, arg = background_distances([segs[i] for i in sel])
    src = best > 100
    if not src.any():
        raise ValueError('no background pixel')
    _, fr, fc = edt(src)
    imgs = np.stack([frames[i] for i in sel])
    arg = arg.copy()
    if src[0, 0]:                    # the reference's assignment through the [HW,1] mask's nonzero tuple also writes pixel 0, last write wins
        arg[0, 0] = arg.reshape(-1)[np.nonzero(src.reshape(-1))[0][-1]]
    return imgs[arg[fr, fc], fr, fc], src, imgs, arg


def tied_colours(colour_of_source, src, p):
    """The colours of every source pixel nearest to pixel p = (row, col)."""
    H, W = src.shape
    r, c = p
    ys, xs = np.nonzero(src)
    d2 = (ys - r) ** 2 + (xs - c) ** 2
    m = d2 == d2.min()
    return {tuple(int(v) for v in colour_of_source[y, x]) for y, x in zip(ys[m], xs[m])}


# ---- the fixture's inputs (tests/golden/make_golden_source.py) ------------------------------------------------------------------------
BG_FRAMES = [1, 5, 6, 100, 150]
BG_H, BG_W = 96, 128


def case_inputs(H, W, seed, kw):
    return syn.make_source_image(H, W, seed), syn.make_segmap(H, W, seed, **kw)


def bg_inputs(n, H=BG_H, W=BG_W, seed=7):
    """n frames of a portrait that sways left and right, each with its own image."""
    frames = np.stack([syn.make_source_image(H, W, 100 + i) for i in range(n)])
    segs = np.stack([syn.make_segmap(H, W, seed, center=0.5 + 0.2 * np.sin(0.7 * i)) for i in range(n)])
    return frames, segs


def golden_cases(z):
    """[(name, img, seg)] of the fixture's torso / head / single-frame background cases."""
    return [(c['name'], *case_inputs(c['H'], c['W'], c['seed'], c['kw'])) for c in json.loads(str(z['cases']))]


def check_background(got, want, src, colour_of_source):
    """got == want except where want's colour is one of the tied nearest sources' colours; returns the number of such pixels."""
    bad = np.nonzero((got != want).any(-1))
    for p in zip(*bad):
        assert tuple(int(v) for v in want[p]) in tied_colours(colour_of_source, src, p), p
    return len(bad[0])


def source_colours(imgs, arg):
    H, W = arg.shape
    return imgs[arg, np.arange(H)[:, None], np.arange(W)[None]]
