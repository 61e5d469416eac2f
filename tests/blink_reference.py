"""A numpy restatement of blink_eye_for_secc (inference/edit_secc.py:47-129), written from the spec in DESIGN.md ("SECC blink"):

  quantise  q = trunc(((x + 1) / 2) * 255) in fp32; the output is q / 127.5 - 1 in fp32 wherever no blink rewrites it; p == 0 stops here
  face      every channel's q != 0
  coarse    ~face inside the prior eye regions: rows [H//4, H//2), left [W//4, W//2), right [W//2, W//4*3)
  box       rows [min_h - 4, max_h + 4) x each eye's coarse columns [cmin - 4, cmax + 4) (half-open)
  er        face & box minus every pixel within distance 5 (dy^2 + dx^2 <= 25) of a coarse pixel;  eye = box & ~er
  columns   n, mean = sum rows / n, min (99999 when empty), max (-99999) of eye, in float64
  blink     eye & (row <= p mean + (1-p) min  |  row >= p mean + (1-p) max)
  fill      each blinked pixel takes the q of its nearest er pixel (the reference aliases its face mask to the eroded one)
  raises    ValueError when coarse, either eye's half of it, er or the blink set is empty

blink(x, p) returns (out fp32 [3,H,W], q_out int [3,H,W], ties, info): ties maps each blinked pixel's flat index to the flat indices of all
its nearest er pixels (the reference's k-d tree picks any of them; tie='lowest', the kernel's rule, takes the first).  p32 rounds p to
fp32 first (only to show why the kernel keeps p in double)."""
import numpy as np

F32 = np.float32


def quantise(x):
    x = np.asarray(x, dtype=F32)
    return np.trunc(((x + F32(1)) / F32(2)) * F32(255)).astype(np.int64)


def dequantise(q):
    return np.asarray(q).astype(F32) / F32(127.5) - F32(1)


def codes(y):
    """An output image (q / 127.5 - 1 in fp32) -> its codes q (exact: the 256 outputs are distinct)."""
    return np.rint((np.asarray(y, dtype=np.float64) + 1) * 127.5).astype(np.int64)


def encode(q):
    """uint8 codes -> fp32 images whose quantisation is exactly q (the centre of each code's bin)."""
    return ((np.asarray(q).astype(F32) + F32(0.5)) / F32(127.5) - F32(1)).astype(F32)


def schedule_p(t, T):
    return -4 / T ** 2 * t ** 2 + 4 / T * t


def rows_control(t, T):
    """The control of an image given by an fp32 row (t, T) (SECC_Renderer.blink's docstring, DESIGN.md "SECC blink"): None (untouched)
    unless 0 <= t < T <= 4096 and int(t) < int(T); else p = schedule_p(int(t), int(T)) in double."""
    t, T = float(np.float32(t)), float(np.float32(T))
    if not (T > 0 and t >= 0 and t < T and T <= 4096):
        return None
    ti, Ti = int(t), int(T)
    return None if ti >= Ti else schedule_p(ti, Ti)


def p_control(p):
    """The control of an image given by a double p: None (untouched) unless 0 <= p <= 1 (so NaN is untouched and -0.0 is p = 0)."""
    p = float(p)
    return p if 0.0 <= p <= 1.0 else None


def _disk_dilate(m, radius=5):
    H, W = m.shape
    pad = np.zeros((H + 2 * radius, W + 2 * radius), dtype=bool)
    pad[radius:radius + H, radius:radius + W] = m
    out = np.zeros_like(m)
    for dy in range(-radius, radius + 1):
        for dx in range(-radius, radius + 1):
            if dy * dy + dx * dx <= radius * radius:
                out |= pad[radius + dy:radius + dy + H, radius + dx:radius + dx + W]
    return out


def blink(x, p, tie='lowest', p32=False, fill_from='er'):
    if not 0.0 <= p <= 1.0:
        raise ValueError('close_eye_percent outside [0, 1]')
    q = quantise(x)
    C, H, W = q.shape
    info = {}
    if p == 0:
        return dequantise(q), q, {}, info
    if p32:
        p = float(F32(p))
    face = (q != 0).all(0)
    rows, cols = np.mgrid[0:H, 0:W]
    in_rows = (rows >= H // 4) & (rows < H // 2)
    left = in_rows & (cols >= W // 4) & (cols < W // 2)
    right = in_rows & (cols >= W // 2) & (cols < W // 4 * 3)
    coarse = ~face & (left | right)
    if not (coarse & left).any() or not (coarse & right).any():
        raise ValueError('no non-face pixel in a prior eye region')
    rr = np.nonzero(coarse.any(1))[0]
    min_h, max_h = rr.min(), rr.max()
    box = np.zeros((H, W), dtype=bool)
    for half in (left, right):
        cc = np.nonzero((coarse & half).any(0))[0]
        box[min_h - 4:max_h + 4, cc.min() - 4:cc.max() + 4] = True
    af = face & box
    er = af & ~_disk_dilate(coarse)
    if not er.any():
        raise ValueError('no face pixel left around the eyes')
    eye = ~er & box
    n = eye.sum(0)
    mean = np.where(eye, rows, 0).sum(0) / np.clip(n, 1, H)
    mn = np.where(eye, rows, 99999).min(0)
    mx = np.where(eye, rows, -99999).max(0)
    lo = p * mean + (1 - p) * mn
    hi = p * mean + (1 - p) * mx
    bl = eye & ((rows <= lo) | (rows >= hi))
    if not bl.any():
        raise ValueError('no pixel to blink')
    info.update(face=face, coarse=coarse, box=box, er=er, eye=eye, blink=bl, lo=lo, hi=hi)
    src_set = er if fill_from == 'er' else af
    E = np.stack(np.nonzero(src_set), 1)                           # row-major order
    Bp = np.stack(np.nonzero(bl), 1)
    q_out = q.copy()
    ties = {}
    for s in range(0, len(Bp), 512):
        b = Bp[s:s + 512]
        d2 = ((b[:, None, :] - E[None, :, :]) ** 2).sum(-1)
        best = d2.min(1)
        for k in range(len(b)):
            cand = np.nonzero(d2[k] == best[k])[0]
            src = E[cand[0]] if tie == 'lowest' else E[cand[-1]]
            q_out[:, b[k, 0], b[k, 1]] = q[:, src[0], src[1]]
            ties[int(b[k, 0] * W + b[k, 1])] = E[cand, 0] * W + E[cand, 1]
    return dequantise(q_out), q_out, ties, info


def equal_outside_ties(q_got, q_ref_in, q_want, ties):
    """q_got [3,H,W] equals q_want everywhere except at tied blink pixels, where it must be the input q of one of the tied candidates.
    Returns the number of tied pixels whose value differs from q_want."""
    C, H, W = q_want.shape
    diff = np.nonzero((q_got != q_want).any(0).reshape(-1))[0]
    flat_in = q_ref_in.reshape(C, -1)
    got = q_got.reshape(C, -1)
    for i in diff:
        cand = ties.get(int(i))
        assert cand is not None and len(cand) > 1, f'pixel {divmod(int(i), W)} differs and is not a tied blink pixel'
        assert any((flat_in[:, j] == got[:, i]).all() for j in cand), f'pixel {divmod(int(i), W)} takes no tied candidate'
    return len(diff)
