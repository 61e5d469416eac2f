"""The SECC blink restatement (tests/blink_reference.py) against the reference's own output (tests/golden/blink_secc.npz), on hand-made images
with known answers, and period_blink_schedule against real3d_infer.py's window rule."""
import os
import random

import numpy as np
import pytest

import blink_reference as bref
from real3dportrait_b200.secc_render import period_blink_schedule

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'blink_secc.npz')
S = 64


def test_restatement_against_reference_fixture():
    g = np.load(GOLD)
    cases = [tuple(int(v) for v in c) for c in g['cases']]
    tied = 0
    for k in range(len(g['images'])):
        q = g[f'img{k}_q'].astype(np.int64)
        x = bref.encode(q)
        for t, T in cases:
            want = q.copy().reshape(3, -1)
            idx = g[f'img{k}_t{t}_T{T}_idx']
            want[:, idx] = g[f'img{k}_t{t}_T{T}_q']
            _, q_out, ties, _ = bref.blink(x, bref.schedule_p(t, T), tie='lowest')
            assert (t == 0) == (len(idx) == 0)
            tied += bref.equal_outside_ties(q_out, q, want.reshape(q.shape), ties)
    assert tied > 0                                                   # the tie rule is exercised (the k-d tree breaks ties its own way)


def _face(holes=((22, 26, 20, 28), (22, 26, 36, 44)), size=S):
    """A size^2 image: face codes (1 + row, 1 + col, 200) everywhere, background (0) in each hole rows [r0, r1) x cols [c0, c1)."""
    r, c = np.mgrid[0:size, 0:size]
    q = np.stack([1 + r, 1 + c, np.full((size, size), 200)]).astype(np.int64)
    for r0, r1, c0, c1 in holes:
        q[:, r0:r1, c0:c1] = 0
    return q


def test_quantise_and_p_zero():
    q = _face()
    x = bref.encode(q)
    out, q_out, ties, _ = bref.blink(x, 0.0)
    assert (q_out == q).all() and not ties
    assert out.dtype == np.float32 and (out == q.astype(np.float32) / np.float32(127.5) - np.float32(1)).all()
    assert (bref.quantise(np.float32([-1.0, 1.0, 0.0])) == [0, 255, 127]).all()


def test_box_is_half_open():
    _, _, _, info = bref.blink(bref.encode(_face()), 0.5)
    box = info['box']
    # coarse rows 22..25 -> box rows [18, 29); left columns 20..27 -> [16, 31); right 36..43 -> [32, 47)
    assert box[18, 16] and box[28, 30] and box[18, 32] and box[28, 46]
    assert not box[17, 20] and not box[29, 20] and not box[20, 15] and not box[20, 31] and not box[20, 47]


def test_erosion_boundary_is_inclusive_at_5():
    _, _, _, info = bref.blink(bref.encode(_face()), 0.5)
    er = info['er']
    # nearest coarse pixel of (r, c) above the left hole's top row 22 at column 24: distance 22 - r
    assert not er[17, 24]                                             # d^2 = 25: eroded
    assert er[18, 16] and not er[18, 20]                              # (18,16) -> (22,20): 16 + 16 = 32 kept; (18,20): 16 eroded
    r0 = 22
    assert not er[r0 - 5, 24] and (r0 - 5 - 4 < 18 or er[r0 - 6, 24])
    # a pixel at (dy, dx) = (3, 4) from the hole's corner (d^2 = 25) is eroded; (4, 4) (d^2 = 32) is kept
    assert not er[26 + 2, 28 + 3] if 28 + 3 < 31 else True
    assert not er[22 - 3, 20 - 4] and er[22 - 4, 20 - 4]


def test_zero_channel_is_not_face():
    q = _face(holes=((22, 26, 20, 28),))                              # no hole on the right: the reference raises
    with pytest.raises(ValueError):
        bref.blink(bref.encode(q), 0.5)
    q[2, 24, 40] = 0                                                  # one channel of one right-hand pixel quantises to 0
    _, q_out, _, info = bref.blink(bref.encode(q), 0.5)
    assert info['coarse'][24, 40] and info['box'][20, 36]


def test_fill_comes_from_the_eroded_set():
    x = bref.encode(_face())
    _, q_er, ties, info = bref.blink(x, 1.0)
    _, q_af, _, _ = bref.blink(x, 1.0, fill_from='af')
    # a blinked pixel in the hole takes a pixel more than 5 px from every hole pixel; filling from the uneroded set takes the hole's rim
    assert info['blink'][22, 24]
    # the face codes are (1 + row, 1 + col, 200): each fill names its source pixel
    src_er, src_af = (q_er[0, 22, 24] - 1, q_er[1, 22, 24] - 1), (q_af[0, 22, 24] - 1, q_af[1, 22, 24] - 1)
    assert info['er'][src_er] and not info['er'][src_af] and info['box'][src_af]
    assert (src_er[0] - 22) ** 2 + (src_er[1] - 24) ** 2 > (src_af[0] - 22) ** 2 + (src_af[1] - 24) ** 2
    assert not np.array_equal(q_er, q_af)


def test_double_p_decides_a_threshold_row():
    """A column whose eye pixels are rows [a, b] blinks row r when r <= p mean + (1 - p) a: at (t, T) = (2, 10) with a = 28, b = 53 (a
    hole over rows [32, 51) at 128^2), row 36 sits on that threshold up to its last rounding, and an fp32 copy of p leaves it open.
    (A column of one eye pixel always blinks: its two thresholds are equal.)"""
    x = bref.encode(_face(holes=((32, 51, 40, 50), (32, 51, 72, 82)), size=128))
    p = bref.schedule_p(2, 10)
    assert float(np.float32(p)) != p
    _, _, _, i64 = bref.blink(x, p)
    _, _, _, i32 = bref.blink(x, p, p32=True)
    assert np.nonzero(i64['eye'][:, 45])[0].tolist() == list(range(28, 54))
    assert i64['blink'][36, 45] and not i32['blink'][36, 45]


@pytest.mark.parametrize('kind', ['no-left', 'no-right', 'no-coarse', 'no-er'])
def test_raise_cases(kind):
    # 'no-er': a blank frame; the box's corners lie (4, 4) from the nearest coarse pixel (d^2 = 32), so only non-face corners empty er
    holes = {'no-left': ((22, 26, 36, 44),), 'no-right': ((22, 26, 20, 28),), 'no-coarse': (), 'no-er': ((0, S, 0, S),)}[kind]
    x = bref.encode(_face(holes))
    with pytest.raises(ValueError):
        bref.blink(x, 0.5)
    bref.blink(x, 0.0)                                                # p = 0 only quantises: never raises
    with pytest.raises(ValueError):
        bref.blink(x, 1.5)


def test_period_schedule():
    n = 300
    s = period_blink_schedule(n, rng=random.Random(7))
    draws = random.Random(7)
    Ts = [draws.randint(8, 12) for _ in range(3)]                    # frames 0, 125, 250 draw in order
    assert s.dtype.is_floating_point is False and s.shape == (n, 2)
    for i, T in zip((0, 125, 250), Ts):
        assert [tuple(v) for v in s[i:i + T].tolist()] == [(t, T) for t in range(T)]
        assert (s[i + T:i + T + 1, 1] == 0).all()
    assert int((s[:, 1] > 0).sum()) == sum(Ts)
    # the last frame never blinks; a window that reaches it stops there
    s2 = period_blink_schedule(130, rng=random.Random(1))
    T2 = random.Random(1).randint(8, 12)
    T2b = (lambda r: (r.randint(8, 12), r.randint(8, 12)))(random.Random(1))[1]
    assert s2[125:129, 1].tolist() == [T2b] * 4 and s2[129].tolist() == [0, 0]
    assert s2[0:T2, 0].tolist() == list(range(T2))
    # the module's random, seeded, gives the same windows
    random.seed(11)
    a = period_blink_schedule(260)
    random.seed(11)
    assert a.tolist() == period_blink_schedule(260, rng=random.Random(11)).tolist()
    with pytest.raises(ValueError):
        period_blink_schedule(10, fps=2, period=5)
