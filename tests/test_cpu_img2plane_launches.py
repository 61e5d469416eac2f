"""img2plane_reference.launch_plan on the host: its launch count from the block counts, its buffer flow, the channel slices of the two
concatenation buffers and the tensor-core route, at every backbone scale and H = 16, 32, 144, 512; the hand-written conv-class tables of
tests/test_gpu_img2plane_conv_classes.py against the 512^2 plan; and the CPU emulation that shows why the end-to-end bar of
tests/test_gpu_img2plane.py stays at 3e-3 max|ref| (DESIGN.md, Canonical plane backbone -> Bars)."""
import pytest
import torch
import torch.nn.functional as F

import img2plane_reference as ref
from real3dportrait_b200.img2plane import Img2PlaneModel

SIZES = [16, 32, 144, 512]
SCALES = ['small', 'standard', 'large']
CAT_WIDTH = {'cat1280': 1280, 'cat448': 448}


@pytest.mark.parametrize('scale', SCALES)
@pytest.mark.parametrize('H', SIZES)
def test_launch_count(H, scale):
    plan = ref.launch_plan(H, 2, scale)
    nlow, ntri = ref.SCALES[scale]
    assert len(plan) == ref.launch_count(H, scale) == 116 + 9 * nlow + 12 * ntri + 3 * (1 if H % 256 == 0 else 2)
    per_fn = {}
    for launch in plan:
        per_fn[launch.fn] = per_fn.get(launch.fn, 0) + 1
    assert per_fn['r3dp_ip_attention'] == per_fn['r3dp_sp_dwconv_gelu'] == nlow + ntri
    assert per_fn['r3dp_sp_layernorm'] == 2 + 2 * nlow - 1 + 2 + 3 * ntri - 1
    assert sum(per_fn.values()) == len(plan)


def test_launch_count_512_standard():
    assert len(ref.launch_plan(512, 4)) == 176
    assert len(ref.launch_plan(512, 1)) == 176


@pytest.mark.parametrize('scale', SCALES)
@pytest.mark.parametrize('H', SIZES)
def test_every_buffer_is_written_before_it_is_read(H, scale):
    """Every read finds its buffer written by an earlier launch, and every channel of a concatenation slice it reads covered by the union of
    the slices written before it."""
    written = {'img'}
    filled = {b: [False] * w for b, w in CAT_WIDTH.items()}
    for launch in ref.launch_plan(H, 3, scale):
        for role, (b, c0, c1) in launch.reads.items():
            assert b in written, f'{launch.tag}: reads {b} ({role}) before any launch writes it'
            if b in filled:
                assert all(filled[b][c0:c1]), f'{launch.tag}: reads {b}[{c0}:{c1}] before all of it is written'
        for role, (b, c0, c1) in launch.writes.items():
            written.add(b)
            if b in filled:
                filled[b][c0:c1] = [True] * (c1 - c0)
    assert 'planes' in written


@pytest.mark.parametrize('H', SIZES)
def test_concatenation_slices_tile_their_buffers(H):
    plan = ref.launch_plan(H, 1)
    for cat, width in CAT_WIDTH.items():
        slices = sorted((c0, c1) for launch in plan for b, c0, c1 in launch.writes.values() if b == cat)
        assert slices[0][0] == 0 and slices[-1][1] == width, (cat, slices)
        for (a0, a1), (b0, b1) in zip(slices, slices[1:]):
            assert a1 == b0, f'{cat}: slices {a0}:{a1} and {b0}:{b1} leave a gap or overlap'
    c448 = [(launch.tag, launch.reads['x'][1:]) for launch in plan if launch.reads.get('x', ('',))[0] == 'cat448']
    assert c448 == [('tri.first_conv', (256, 448)), ('tri.first_conv_after_cat', (0, 352))]
    writers = {launch.tag: launch.writes['y'][1:] for launch in plan for b in launch.writes.values() if b[0] == 'cat448'}
    assert writers == {'low.final_conv': (256, 352), 'high.final': (352, 448), 'tri.shuffle': (0, 256)}


@pytest.mark.parametrize('H', SIZES + [1024])
def test_tensor_core_route(H):
    """r3dp_sr_tc_conv exactly where the module's rule takes it: a stride-1 3x3 conv with 128 or 256 outputs, a dense input of a multiple
    of 64 channels, h % 128 == 0, its own output, no residual, an fp16 store."""
    plan = ref.launch_plan(H, 1)
    tc = [launch.tag for launch in plan if launch.fn == 'r3dp_sr_tc_conv']
    at_h2 = ['low.conv_after_upsample2', 'tri.second_conv', 'tri.second_conv_after_cat', 'tri.third_conv_after_cat']
    want = (['low.conv_after_upsample1'] if H % 512 == 0 else []) + (at_h2 if H % 256 == 0 else [])
    if H % 1024 == 0:                                           # layer2's convs without a residual and the decoder conv, at H/8
        want = [f'layer2.{b}.conv1' for b in (1, 2, 3)] + ['decoder'] + want
    assert tc == want
    for launch in plan:
        if launch.fn == 'r3dp_sr_tc_conv':
            N, Nw, I, O, h, w, k, act = launch.args
            assert O in (128, 256) and I % 64 == 0 and h % 128 == 0 and k == 3 and act in (0, 2, 3)
        elif launch.fn == 'r3dp_mf_conv3d' and launch.args[8] == 3:
            xs, _, cin, N, D, h, w, kd, kh, kw, _, O, cop, relu, ys, yc0, _, f32, _ = launch.args
            own = ys == O and yc0 == 0
            assert not (O in (128, 256) and cin % 64 == 0 and xs == cin and h % 128 == 0 and own and 'res' not in launch.reads and not f32), \
                f'{launch.tag} qualifies for r3dp_sr_tc_conv'


def test_leaky_slopes_and_in_place_layernorms():
    plan = ref.launch_plan(512, 1)
    slopes = {launch.args[1] for launch in plan if launch.fn == 'r3dp_sp_leaky'}
    assert slopes == {0.0, 0.01}
    relu = [launch.tag for launch in plan if launch.fn == 'r3dp_sp_leaky' and launch.args[1] == 0.0]
    assert len(relu) == sum(ref.LAYERS)                         # one per BasicBlock, after its residual add
    inplace = [launch.tag for launch in plan if launch.fn == 'r3dp_sp_layernorm' and 'xo' in launch.writes]
    assert all(launch.writes['xo'][0] == launch.reads['x'][0] for launch in plan if 'xo' in launch.writes)
    assert len(inplace) == 2 * 5 - 1 + 2 * 1 - 1
    assert {launch.args[3] for launch in plan if launch.fn == 'r3dp_sp_dwconv_gelu'} == {ref.MLP}


def test_conv_class_tables_are_plan_launches():
    """The hand-written classes of tests/test_gpu_img2plane_conv_classes.py (kernel, K, cout, epilogue, slices; reduced sizes) each name a
    class the forward launches at one of SIZES, and every class of the 512^2 forward has one."""
    import test_gpu_img2plane_conv_classes as cc

    def classes(H):
        mf, tc = {}, {}
        for launch in ref.launch_plan(H, 1):
            if launch.fn == 'r3dp_mf_conv3d':
                xs, _, cin, N, D, h, w, kd, kh, kw, _, O, cop, relu, ys, yc0, _, f32, _ = launch.args
                mf.setdefault(('box' if kh == 3 else 'gemm', cin, O, bool(relu), 'res' in launch.reads, bool(f32), xs, launch.reads['x'][1], ys,
                               yc0), launch.tag)
            elif launch.fn == 'r3dp_sr_tc_conv':
                tc.setdefault((launch.args[2], launch.args[3], launch.args[7]), launch.tag)
        return mf, tc

    every = {}
    for H in SIZES:
        every.update(classes(H)[0])
    rows = {tuple(r[1:11]): r[0] for r in cc.ROWS}
    stale = [r for k, r in rows.items() if k not in every]
    assert not stale, f'conv-class rows no forward launches: {stale}'
    mf512, tc512 = classes(512)
    missing = [f'{t}: {k}' for k, t in mf512.items() if k not in rows]
    assert not missing, '512^2 launch classes without a row in ROWS:\n' + '\n'.join(missing)
    assert {(r[1], r[2], r[3]) for r in cc.TC_ROWS} == set(tc512)


# ---- why the end-to-end bar stays -----------------------------------------------------------------------------------------------------
def _emulated(sd, x, mode):
    """ref.forward with every conv2d / linear on fp16-rounded operands (the input and the weight; bias as given), accumulated in
    float64 ('f64') or float32 ('f32'); 'exact' leaves the operands alone and accumulates in float32."""
    conv2d, linear = F.conv2d, F.linear

    def wrap(fn):
        def call(inp, w, b=None, *a, **k):
            if mode == 'exact':
                return fn(inp.float(), w.float(), None if b is None else b.float(), *a, **k).double()
            inp, w = inp.half().double(), w.half().double()
            if mode == 'f32':
                return fn(inp.float(), w.float(), None if b is None else b.float(), *a, **k).double()
            return fn(inp, w, b, *a, **k)
        return call
    F.conv2d, F.linear = wrap(conv2d), wrap(linear)
    try:
        return ref.forward(sd, x)
    finally:
        F.conv2d, F.linear = conv2d, linear


@torch.no_grad()
def test_fp16_rounding_boundaries_swamp_accumulation_order():
    """At 64^2 (standard, B = 1): fp16 operand rounding moves the planes by ~1.25e-3 max|ref| (what the H100 measures end to end), and the
    same rounded operands accumulated in fp32 instead of float64 land ~1e-3 away again, although fp32 against float64 accumulation without
    the rounding differs by ~1e-6: each rounding boundary turns a 1e-6 difference into a full fp16 step.  A faithful fp16 emulation agrees
    with the kernels no better than float64 does, so no end-to-end bar can sit much below 3e-3; faults smaller than that are the per-launch
    tests' to catch (tests/test_gpu_img2plane_launches.py)."""
    m = Img2PlaneModel()
    sd = {k: v.double() if v.is_floating_point() else v for k, v in ref.make_params({k: v.shape for k, v in m.state_dict().items()}, 5).items()}
    x = ref.make_inputs(1, 64, 11).double()
    exact = ref.forward(sd, x)
    scale = float(exact.abs().max())
    r64 = _emulated(sd, x, 'f64')
    r32 = _emulated(sd, x, 'f32')
    e32 = _emulated(sd, x, 'exact')
    rounding = float((r64 - exact).abs().max()) / scale
    order = float((r32 - r64).abs().max()) / scale
    fp32 = float((e32 - exact).abs().max()) / scale
    print(f'64^2: fp16 operands vs exact {rounding:.2e}; fp32 vs float64 accumulation of them {order:.2e}; fp32 vs float64, no rounding '
          f'{fp32:.2e}')
    assert fp32 < 1e-5
    assert 5e-4 < rounding < 3e-3
    assert order > 3e-4
