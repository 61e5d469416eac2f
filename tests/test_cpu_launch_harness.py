"""The shared launch-test helpers (tests/launch_harness.py) on CPU tensors: guards report a stray or a missed write, split / join round-trip,
launch_signature rounds to fp32, the recorder records only what it selects and always restores the C API, conv3d puts a plan row's
arguments at their C positions, and the plan assertions name what differs."""
import ctypes

import pytest
import torch

import launch_harness as lh
from real3dportrait_b200 import _capi as capi


@pytest.mark.parametrize('dtype', [torch.float16, torch.float32, torch.uint8, torch.int64])
@pytest.mark.parametrize('where', ['head', 'tail'])
def test_write_into_a_guard_is_reported(dtype, where):
    buf, y = lh.guarded(10, dtype, device='cpu')
    assert lh.guards_intact(buf, 10) and bool(lh.untouched(y).all())
    buf[lh.GUARD - 1 if where == 'head' else lh.GUARD + 10] = 0
    assert not lh.guards_intact(buf, 10)


def test_fill_value_is_compared_by_bits():
    buf, y = lh.guarded(5, torch.float32, fill=float('nan'), device='cpu')
    assert lh.guards_intact(buf, 5, fill=float('nan'))
    buf[0] = -float('nan')                                      # still NaN, other bits
    assert not lh.guards_intact(buf, 5, fill=float('nan'))


@pytest.mark.parametrize('split', [False, True])
def test_missed_element_of_a_slice_is_reported(split):
    vs, c0, n, lo, rows = 16, 2, 3, 8, 4
    buf, y = lh.guarded(rows * vs, torch.float16, device='cpu')
    mask = lh.inside(vs, c0, n, lo, split, device='cpu')
    assert int(mask.sum()) == n * (2 if split else 1)
    yv = y.view(rows, vs)
    yv[:, mask] = 1.0
    lh.assert_written(buf, y, vs, mask, 'full')
    last = (lo if split else 0) + c0 + n - 1                    # the last element of the slice (of its lo half when split)
    lh.bits(yv)[rows - 1, last] = lh.SENTINEL[torch.float16][1]
    with pytest.raises(AssertionError, match='not written'):
        lh.assert_written(buf, y, vs, mask, 'missed')
    yv[rows - 1, last] = 1.0
    yv[0, c0 + n] = 1.0
    with pytest.raises(AssertionError, match='outside its channels'):
        lh.assert_written(buf, y, vs, mask, 'stray')


def test_split_join_round_trip():
    g = torch.Generator().manual_seed(0)
    h = (torch.randn(64, 8, generator=g) * 100).half().float()
    v = torch.where(h.abs() < 1, torch.ones_like(h), h) * (1 + 2.0 ** -12)   # hi + lo with both halves normal fp16: a split pair exactly
    hi, lo = lh.split(v)
    y = torch.cat([hi, lo], -1)
    assert torch.equal(lh.join(y, 0, 8, 8), v.double())
    assert torch.equal(lh.split_cat(v), y)
    assert torch.equal(lh.join(y, 2, 3, 8, split=False), hi[:, 2:5].double())
    lh.check_split_layout(y)


def test_launch_signature_rounds_to_fp32():
    fn, a = lh.launch_signature('f', [3, 0.1, True])
    assert fn == 'f' and a == (3, ctypes.c_float(0.1).value, True) and a[1] != 0.1


class _FakeLib:
    def r3dp_a(self, *args):
        return sum(args)

    def r3dp_b(self, *args):
        return -1


def test_recorder_passes_through_records_selected_and_restores():
    lib, ptr = capi._lib, capi.ptr
    with lh.Recorder(_FakeLib(), lambda n: n == 'r3dp_a', ptrs=True) as rec:
        assert capi._lib is rec and capi.ptr == rec.ptr
        assert capi._lib.r3dp_a(1, 2) == 3 and capi._lib.r3dp_b(5) == -1
    assert rec.calls == [('r3dp_a', (1, 2))]
    assert capi._lib is lib and capi.ptr is ptr
    with pytest.raises(RuntimeError):
        with lh.Recorder(_FakeLib(), lambda n: True) as rec:
            capi._lib.r3dp_b(1)
            raise RuntimeError('the body fails')
    assert rec.calls == [('r3dp_b', (1,))]
    assert capi._lib is lib and capi.ptr is ptr


def test_given_treats_null_and_zero_as_absent():
    assert not lh.given(None) and not lh.given(ctypes.c_void_p(0)) and not lh.given(ctypes.c_void_p(None)) and not lh.given(0)
    assert lh.given(ctypes.c_void_p(64)) and lh.given(64)


class _Conv3dLib:
    def r3dp_mf_conv3d(self, *args):
        return 0


def test_conv3d_argument_order_and_call_signature(monkeypatch):
    """conv3d puts a plan row's arguments, overrides included, at their C positions: recorded and read back through call_signature."""
    row = tuple(range(101, 120))                                # xs .. split, all distinct
    x, res, y = (ctypes.c_void_p(a) for a in (0x1000, 0x2000, 0x3000))
    monkeypatch.setattr(capi, 'stream', lambda: ctypes.c_void_p(0x4000))
    with lh.Recorder(_Conv3dLib(), lambda n: True) as rec:
        lh.conv3d(row, x, None, None, res, y, N=7, W=9)
        lh.conv3d(row, x, None, None, None, y)
    (fn, a), (_, b) = rec.calls
    assert fn == 'r3dp_mf_conv3d' and len(a) == len(capi._SIGNATURES[fn][1])
    assert (a[0].value, a[4].value, a[5].value, a[6].value, a[18].value, a[24].value) == (0x1000, None, None, 0x2000, 0x3000, 0x4000)
    want = dict(zip(lh.CONV3D_ARGS, row), N=7, W=9)
    assert lh.call_signature(fn, a, (6,)) == (fn, tuple(want[k] for k in lh.CONV3D_ARGS) + (True,))
    assert lh.call_signature(fn, b, (6,)) == (fn, row + (False,))


def test_plan_and_row_assertions_name_the_difference():
    lh.assert_plan([('f', (1,)), ('g', (2,))], [('f', (1,)), ('g', (2,))], 'same')
    with pytest.raises(AssertionError, match=r"where: the module launches \('h', \(3,\)\) not in launch_plan, which has \('g', \(2,\)\)"):
        lh.assert_plan([('f', (1,)), ('h', (3,))], [('f', (1,)), ('g', (2,))], 'where')
    with pytest.raises(AssertionError, match='order differs'):
        lh.assert_plan([('g', (2,)), ('f', (1,))], [('f', (1,)), ('g', (2,))], 'where')
    lh.assert_rows([], [], 'the model')
    with pytest.raises(AssertionError, match='the model launches without a float64 row:\nB=2: f'):
        lh.assert_rows(['B=2: f'], [], 'the model')
    with pytest.raises(AssertionError, match='rows the model no longer launches:\nrow 3'):
        lh.assert_rows([], ['row 3'], 'the model')
