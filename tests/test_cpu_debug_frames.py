"""The 'concat_debug' restatement (tests/debug_frames_reference.py) against frames the reference's own forward_secc2video wrote
(tests/golden/debug_frames.npz), and the readings the fixture must reject: a float32-only conversion, and copying the source bytes and q."""
import os

import numpy as np
import pytest
import torch

from debug_frames_reference import S, concat_debug_reference, full_inputs

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'debug_frames.npz')
KEYS = ('ref_bytes', 'secc', 'image_raw', 'image_depth', 'image')


def case(name):
    d = np.load(GOLDEN)
    return full_inputs({k: d[f'{name}.{k}'] for k in KEYS}), torch.from_numpy(d[f'{name}.frames'])


def run(t, **kw):
    return concat_debug_reference(t['ref_gt_img'], t['drv_secc'], t['image_raw'], t['image_depth'], t['image'], **kw)


@pytest.mark.parametrize('name', ['quirks', 'flat'])
def test_restatement_matches_reference_frames(name):
    t, frames = case(name)
    assert frames.shape == (t['image'].shape[0], S, 5 * S, 3) and frames.dtype == torch.uint8
    assert torch.equal(run(t), frames)


def test_constant_depth_gives_byte_zero():
    _, frames = case('flat')
    assert int(frames[:, :, 3 * S:4 * S].max()) == 0


def _panel_misses(a, b):
    return [int((a[:, :, p * S:(p + 1) * S] != b[:, :, p * S:(p + 1) * S]).sum()) for p in range(5)]


def test_float32_conversion_fails_on_fixture():
    t, frames = case('quirks')
    miss = _panel_misses(run(t, float32_only=True), frames)
    print('float32-only bytes wrong per panel:', miss)
    assert miss[1] > 0 and miss[2] > 0 and miss[4] > 0, miss       # panel 0 differs only through the conversion of 127 source bytes


def test_copied_bytes_fail_on_fixture():
    t, frames = case('quirks')
    miss = _panel_misses(run(t, copy_bytes=True, ref_bytes=t['ref_bytes']), frames)
    print('copied source bytes / q: bytes wrong per panel:', miss)
    assert miss[0] > 0 and miss[1] > 0 and miss[2:] == [0, 0, 0], miss


def test_fixture_covers_the_quirks():
    t, frames = case('quirks')
    src = torch.as_tensor(t['ref_bytes'])
    assert len(torch.unique(src)) == 256
    p0 = frames[:, :, :S].to(torch.int16)
    assert bool((p0 == src.to(torch.int16) - 1).any()) and bool((p0 == src.to(torch.int16)).any())  # source bytes both kept and lowered
    d = t['image_depth']
    assert int(d.flatten(1).min(1).values.argmin()) != int(d.flatten(1).max(1).values.argmax())     # min and max in different frames
    assert float(t['drv_secc'].min()) < -1
