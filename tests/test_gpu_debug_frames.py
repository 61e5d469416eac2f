"""The 'concat_debug' panel kernels (r3dp_debug_panels, r3dp_debug_depth_panel) and concat_debug_frames on the GPU, bit for bit against the
CPU restatement of real3d_infer.py:494-521 (tests/debug_frames_reference.py) and the reference-generated fixture: seeded random and adversarial
inputs, B = 1 and 4, clips that are not a multiple of the batch, strided destinations inside canaries, and constant depth."""
import os

import numpy as np
import pytest
import torch

import real3dportrait_b200 as r3
from real3dportrait_b200 import debug_frames as dbg
from debug_frames_reference import S, byte_boundaries, concat_debug_reference, full_inputs, quirk_inputs, secc_boundaries

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'debug_frames.npz')
KEYS = ('ref_bytes', 'secc', 'image_raw', 'image_depth', 'image')


def _ref(t):
    return concat_debug_reference(t['ref_gt_img'], t['drv_secc'], t['image_raw'], t['image_depth'], t['image'])


def _dev(t):
    return [t[k].to(DEV) for k in ('ref_gt_img', 'drv_secc', 'image_raw', 'image_depth', 'image')]


def _random(N, seed, adversarial=False):
    """Full-resolution random inputs (no 8 x 8 structure in panels 0, 1 and 4); adversarial: the quirk values scattered among them."""
    g = torch.Generator().manual_seed(seed)
    t = {'ref_gt_img': ((torch.randint(0, 256, (1, 3, S, S), generator=g).float() - 127.5) / 127.5),
         'drv_secc': torch.rand(N, 3, S, S, generator=g) * 2.2 - 1.1, 'image_raw': torch.rand(N, 3, 64, 64, generator=g) * 2.4 - 1.2,
         'image_depth': torch.rand(N, 1, 64, 64, generator=g) * 0.5 + 2.0, 'image': torch.rand(N, 3, S, S, generator=g) * 2 - 1}
    if adversarial:
        for k, vals in (('drv_secc', secc_boundaries()), ('image', byte_boundaries()), ('image_raw', byte_boundaries())):
            flat = t[k].view(-1)
            idx = torch.randperm(flat.numel(), generator=g)[:len(vals) * 4]
            flat[idx] = torch.from_numpy(np.tile(vals, 4))
    return t


@pytest.mark.parametrize('name', ['quirks', 'flat'])
def test_concat_debug_frames_equals_fixture(name):
    d = np.load(GOLDEN)
    t = full_inputs({k: d[f'{name}.{k}'] for k in KEYS})
    got = r3.concat_debug_frames(*_dev(t))
    assert got.dtype == torch.uint8 and got.shape == (3, S, 5 * S, 3) and got.is_cuda
    assert torch.equal(got.cpu(), torch.from_numpy(d[f'{name}.frames']))


@pytest.mark.parametrize('N,seed,adv', [(1, 0, False), (4, 1, False), (4, 2, True), (7, 3, True)])
def test_concat_debug_frames_equals_restatement(N, seed, adv):
    t = _random(N, seed, adv)
    assert torch.equal(r3.concat_debug_frames(*_dev(t)).cpu(), _ref(t))


def test_quirk_inputs_at_full_batch():
    t = full_inputs(quirk_inputs(4, 9))
    assert torch.equal(r3.concat_debug_frames(*_dev(t)).cpu(), _ref(t))


@pytest.mark.parametrize('B', [1, 4])
@pytest.mark.parametrize('aligned', [True, False])
def test_entry_points_in_batches_into_a_strided_clip(B, aligned):
    """A clip of 7 frames written B frames at a time by r3dp_debug_panels into strips sliced from a wider buffer (row pitch 7680 + pad, a
    frame gap, an odd start when not aligned), then r3dp_debug_depth_panel over the whole clip: every strip byte is written, nothing else."""
    N = 7
    t = _random(N, 11 + B, adversarial=True)
    ref_gt, secc, raw, depth, image = _dev(t)
    pad = 16 if aligned else 5
    rows = S + 3                                                       # 3 spare rows per frame
    canary = 0xA5
    buf = torch.full((N * rows * (5 * S * 3 + pad) + 64,), canary, dtype=torch.uint8, device=DEV)
    off = 8 if aligned else 3
    pitch, fstride = 5 * S * 3 + pad, rows * (5 * S * 3 + pad)
    clip = buf[off:off + (N - 1) * fstride + (S - 1) * pitch + 5 * S * 3].as_strided((N, S, 5 * S, 3), (fstride, pitch, 3, 1))
    feat = raw.permute(0, 2, 3, 1).reshape(N, 4096, 3).contiguous()
    # the render's real layout has more than 3 channels: pad the features to 32 with values the kernel must not read
    feat32 = torch.cat([feat, torch.full((N, 4096, 29), float('nan'), device=DEV)], -1).contiguous()
    for b0 in range(0, N, B):
        n = min(B, N - b0)
        dbg.debug_panels(ref_gt, secc[b0:b0 + n].contiguous(), feat32[b0:b0 + n].contiguous(), image[b0:b0 + n].contiguous(), clip[b0:b0 + n])
    dbg.depth_panel(depth.contiguous(), clip)
    torch.cuda.synchronize()
    assert torch.equal(clip.cpu(), _ref(t))
    mask = torch.ones(buf.numel(), dtype=torch.bool)
    idx = torch.arange(N * S * 5 * S * 3).view(N, S, 5 * S * 3)
    pos = off + (idx // (S * 5 * S * 3)) * fstride + ((idx // (5 * S * 3)) % S) * pitch + idx % (5 * S * 3)
    mask[pos.view(-1)] = False
    assert bool((buf.cpu()[mask] == canary).all()), 'a byte outside the strips was written'


def test_panels_leave_panel_3_and_depth_panel_leaves_the_rest():
    t = _random(2, 21)
    ref_gt, secc, raw, depth, image = _dev(t)
    out = torch.full((2, S, 5 * S, 3), 7, dtype=torch.uint8, device=DEV)
    dbg.debug_panels(ref_gt, secc, raw.permute(0, 2, 3, 1).reshape(2, 4096, 3).contiguous(), image, out)
    assert bool((out[:, :, 3 * S:4 * S] == 7).all()) and bool((out[:, :, :3 * S] != 7).any())
    out2 = torch.full_like(out, 7)
    dbg.depth_panel(depth.contiguous(), out2)
    assert bool((out2[:, :, :3 * S] == 7).all()) and bool((out2[:, :, 4 * S:] == 7).all())


@pytest.mark.parametrize('F', [1, 3])
def test_constant_depth_gives_byte_zero(F):
    t = _random(F, 30 + F)
    t['image_depth'][:] = 2.5
    got = r3.concat_debug_frames(*_dev(t)).cpu()
    assert int(got[:, :, 3 * S:4 * S].max()) == 0
    assert torch.equal(got, _ref(t))


def test_single_frame_depth_and_nan():
    t = _random(1, 40)
    assert torch.equal(r3.concat_debug_frames(*_dev(t)).cpu(), _ref(t))
    t['image_depth'][0, 0, 3, 3] = float('nan')                        # torch's min / max propagate NaN: the whole panel is byte 0
    got = r3.concat_debug_frames(*_dev(t)).cpu()
    assert int(got[:, :, 3 * S:4 * S].max()) == 0 and torch.equal(got, _ref(t))


def test_graph_capture_and_guards():
    t = _random(2, 50)
    ref_gt, secc, raw, depth, image = _dev(t)
    out = torch.empty(2, S, 5 * S, 3, dtype=torch.uint8, device=DEV)
    r3.concat_debug_frames(ref_gt, secc, raw, depth, image, out=out)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        r3.concat_debug_frames(ref_gt, secc, raw, depth, image, out=out)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.cpu(), _ref(t))
    with pytest.raises(ValueError):
        r3.concat_debug_frames(ref_gt, secc[:, :, :256, :256].contiguous(), raw, depth, image)
    with pytest.raises(ValueError):
        dbg.debug_panels(ref_gt, secc, raw.permute(0, 2, 3, 1).reshape(2, 4096, 3).contiguous(), image, out[:, :, :S])
    with pytest.raises(ValueError):
        dbg.depth_panel(depth.contiguous(), out.cpu())
