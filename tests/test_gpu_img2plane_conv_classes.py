"""Every distinct r3dp_mf_conv3d class (kernel, K, cout, epilogue, operand slicing) that Img2PlaneModel.forward launches at 512^2, once
each, against float64 of the operands the kernel reads, with tests/sr_conv_reference.py's bound:

    |got - ref| <= alpha |ref| + beta S,   S = the same operation on |x|, |w|, |bias| (and |res|),

alpha = 2^-11 for fp16 stores and 2^-24 for fp32 stores (the residual is added before the one fp16 rounding).  beta is each kernel's own
accumulation term: r3dp_mf_conv3d's 2^-18 (BETA_MF, the bar tests/test_gpu_torso_motion.py set for it), r3dp_sr_tc_conv's BETA['tc'].
Worst ratio measured here on an H100 80GB HBM3 (700 W power limit): r3dp_mf_conv3d 7.06e-7, the fp32-out `sr` GEMM (K = 4096; the fp32
stores expose the whole accumulation term, the fp16 rows hide part of it under alpha).  The weights
are packed by the module's own packers (img2plane._Conv, secc2plane._pack_gemm) and read back.  Spatial sizes are reduced (the class is
the kernel, K and cout; the kernel tiles 128 output voxels whatever the image size); slices and strides are the forward's.  Outputs sit in
NaN-filled buffers: every element of the slice must be written and no other channel."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import sr_conv_reference as scr
from real3dportrait_b200 import _capi as capi
from real3dportrait_b200 import img2plane as ip

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
F16, F64 = torch.float16, torch.float64
P = capi.ptr
BETA_MF = 2.0 ** -18                         # r3dp_mf_conv3d, fp16 operands (tests/test_gpu_torso_motion.py BETA3[False])

# (name, kind, cin, cout, relu, res, out_f32, xs, xc0, ys, yc0, bias): kind 'box' = 3x3 (1,3,3) taps, 'gemm' = one tap over K = cin (token
# linears, 1x1 convs, and the patch rows of the strided / dilated convs, K = k*k*C padded to a multiple of 32)
ROWS = [
    # ResNet-34 encoder (BatchNorm folded into a bias)
    ('stem 7x7/2 patch rows', 'gemm', 416, 64, True, False, False, 416, 0, 64, 0, True),
    ('high.first 7x7/2 patch rows', 'gemm', 416, 64, False, False, False, 416, 0, 64, 0, True),
    ('layer1 conv1', 'box', 64, 64, True, False, False, 64, 0, 64, 0, True),
    ('layer1 conv2 + identity', 'box', 64, 64, False, True, False, 64, 0, 64, 0, True),
    ('layer2.0 conv1 3x3/2 patch rows', 'gemm', 576, 128, True, False, False, 576, 0, 128, 0, True),
    ('layer2.0 downsample 1x1/2 patch rows', 'gemm', 64, 128, False, False, False, 64, 0, 128, 0, True),
    ('layer2 conv1', 'box', 128, 128, True, False, False, 128, 0, 128, 0, True),
    ('layer2 conv2 + identity', 'box', 128, 128, False, True, False, 128, 0, 128, 0, True),
    ('layer3.0 conv1 dilated patch rows', 'gemm', 1152, 256, True, False, False, 1152, 0, 256, 0, True),
    ('layer3.0 downsample 1x1', 'gemm', 128, 256, False, False, False, 128, 0, 256, 0, True),
    ('layer3 conv1 dilated patch rows', 'gemm', 2304, 256, True, False, False, 2304, 0, 256, 0, True),
    ('layer3 conv2 dilated patch rows + identity', 'gemm', 2304, 256, False, True, False, 2304, 0, 256, 0, True),
    ('layer4.0 conv1 dilated patch rows', 'gemm', 2304, 512, True, False, False, 2304, 0, 512, 0, True),
    ('layer4.0 downsample 1x1', 'gemm', 256, 512, False, False, False, 256, 0, 512, 0, True),
    ('layer4 conv1 dilated patch rows', 'gemm', 4608, 512, True, False, False, 4608, 0, 512, 0, True),
    ('layer4 conv2 dilated patch rows + identity', 'gemm', 4608, 512, False, True, False, 4608, 0, 512, 0, True),
    # ASPP and the decoder conv (bias-free convs)
    ('aspp 1x1 into slice 0 of 1280', 'gemm', 512, 256, True, False, False, 512, 0, 1280, 0, False),
    ('aspp rate-12 patch rows into slice 256 of 1280', 'gemm', 4608, 256, True, False, False, 4608, 0, 1280, 256, False),
    ('aspp rate-24 patch rows into slice 512 of 1280', 'gemm', 4608, 256, True, False, False, 4608, 0, 1280, 512, False),
    ('aspp rate-36 patch rows into slice 768 of 1280', 'gemm', 4608, 256, True, False, False, 4608, 0, 1280, 768, False),
    ('aspp pooled rows', 'gemm', 512, 256, True, False, False, 512, 0, 256, 0, False),
    ('aspp project', 'gemm', 1280, 256, True, False, False, 1280, 0, 256, 0, False),
    ('decoder conv', 'box', 256, 256, False, False, False, 256, 0, 256, 0, False),
    # the ViTs
    ('low patch embed rows', 'gemm', 2304, 1024, False, False, True, 2304, 0, 1024, 0, True),
    ('tri patch embed rows', 'gemm', 1152, 1024, False, False, True, 1152, 0, 1024, 0, True),
    ('tri sr 2x2/2 rows', 'gemm', 4096, 1024, False, False, True, 4096, 0, 1024, 0, True),
    ('q', 'gemm', 1024, 1024, False, False, False, 1024, 0, 1024, 0, True),
    ('kv', 'gemm', 1024, 2048, False, False, False, 1024, 0, 2048, 0, True),
    ('proj', 'gemm', 1024, 1024, False, False, True, 1024, 0, 1024, 0, True),
    ('fc1', 'gemm', 1024, 2048, False, False, False, 1024, 0, 2048, 0, True),
    ('fc2', 'gemm', 2048, 1024, False, False, True, 2048, 0, 1024, 0, True),
    # conv tails
    ('low conv_after_upsample1', 'box', 256, 128, True, False, False, 256, 0, 128, 0, True),
    ('low conv_after_upsample2', 'box', 128, 128, True, False, False, 128, 0, 128, 0, True),
    ('low final into slice 256 of 448', 'box', 128, 96, False, False, False, 128, 0, 448, 256, True),
    ('high conv_layers.0', 'box', 64, 96, False, False, False, 64, 0, 96, 0, True),
    ('high conv_layers.2', 'box', 96, 96, False, False, False, 96, 0, 96, 0, True),
    ('high final into slice 352 of 448', 'box', 96, 96, False, False, False, 96, 0, 448, 352, True),
    ('tri first_conv from slice 256 of 448', 'box', 192, 256, False, False, False, 448, 256, 256, 0, True),
    ('tri second_conv (W % 128 != 0)', 'box', 256, 128, False, False, False, 256, 0, 128, 0, True),
    ('tri first_conv_after_cat from slice 0 of 448', 'box', 352, 256, False, False, False, 448, 0, 256, 0, True),
    ('tri third_conv_after_cat (W % 128 != 0)', 'box', 128, 128, False, False, False, 128, 0, 128, 0, True),
    ('tri final fp32', 'box', 128, 96, False, False, True, 128, 0, 96, 0, True),
]


def ctypes_ptr(t, elems):
    return ctypes.c_void_p(t.data_ptr() + t.element_size() * elems)


def _g(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


@pytest.mark.parametrize('row', ROWS, ids=[r[0] for r in ROWS])
@torch.no_grad()
def test_conv_class(row):
    name, kind, cin, cout, relu, res, out_f32, xs, xc0, ys, yc0, with_bias = row
    Bn, h = 2, 24                                                     # box: 2 x 24 x 24 = 1152 voxels (9 tiles of 128, one partial)
    rows = Bn * h * h if kind == 'box' else (2 if name == 'aspp pooled rows' else 1000)
    w = torch.randn(cout, cin, *((3, 3) if kind == 'box' else (1, 1)), generator=_g(1), device=DEV, dtype=F64) / cin ** 0.5
    b = 0.1 * torch.randn(cout, generator=_g(2), device=DEV, dtype=F64) if with_bias else None
    cv = ip._Conv(w, b, 3 if kind == 'box' else 1, 1, 1 if kind == 'box' else 0, 1, DEV)
    wp, bias, O, cop = cv.pk
    x = torch.randn(rows, xs, generator=_g(3), device=DEV).to(F16)
    r = torch.randn(rows, cout, generator=_g(4), device=DEV).to(F16) if res else None
    ydt = torch.float32 if out_f32 else F16
    y = torch.full((rows, ys), float('nan'), device=DEV, dtype=ydt)
    xp = ctypes_ptr(x, xc0)
    geo = (Bn, 1, h, h, 1, 3, 3) if kind == 'box' else (1, 1, rows, 1, 1, 1, 1)
    capi.check(capi.lib().r3dp_mf_conv3d(xp, xs, 0, cin, P(wp, F16), P(bias), None if r is None else P(r, F16), *geo, 0, O, cop, int(relu),
                                         ctypes_ptr(y, 0), ys, yc0, 0, int(out_f32), 0, capi.stream()))
    torch.cuda.synchronize()
    # float64 of the operands read: the fp16 slice of x, the packed weights read back, the fp32 bias
    xv = x[:, xc0:xc0 + cin].to(F64)
    bv = bias[:cout].to(F64)
    if kind == 'box':
        wv = wp[:, :cout].to(F64).reshape(3, 3, cout, cin).permute(2, 3, 0, 1)
        xi = xv.view(Bn, h, h, cin).permute(0, 3, 1, 2)
        ref = F.conv2d(xi, wv, bv, 1, 1).permute(0, 2, 3, 1).reshape(rows, cout)
        S = F.conv2d(xi.abs(), wv.abs(), bv.abs(), 1, 1).permute(0, 2, 3, 1).reshape(rows, cout)
    else:
        wv = wp[:cout].to(F64)
        ref = xv @ wv.T + bv
        S = xv.abs() @ wv.abs().T + bv.abs()
    if relu:
        ref = ref.clamp_min(0)
    if res:
        ref = ref + r.to(F64)
        S = S + r.to(F64).abs()
    got = y[:, yc0:yc0 + cout]
    scr.check_bound(got, ref, S, scr.ALPHA_F32 if out_f32 else scr.ALPHA_F16, BETA_MF, extra=None if out_f32 else scr.FLOOR_F16, tag=name)
    assert torch.isnan(y[:, :yc0]).all() and torch.isnan(y[:, yc0 + cout:]).all(), 'write outside the output slice'


# r3dp_sr_tc_conv classes of the forward (dense inputs, W % 128 == 0): LowResolutionViT's conv_after_upsample1/2 (ReLU, act 3) and
# TriplanePredictorViT's second_conv, second/third_conv_after_cat (LeakyReLU(0.01), act 2), with the module's packing
TC_ROWS = [('low conv_after_upsample1', 256, 128, 3), ('low conv_after_upsample2', 128, 128, 3), ('tri second_conv', 256, 128, 2),
           ('tri third_conv_after_cat', 128, 128, 2)]


@pytest.mark.parametrize('name,cin,cout,act', TC_ROWS, ids=[r[0] for r in TC_ROWS])
@torch.no_grad()
def test_tc_conv_class(name, cin, cout, act):
    Bn, h = 1, 128
    w = torch.randn(cout, cin, 3, 3, generator=_g(5), device=DEV, dtype=F64) / (9 * cin) ** 0.5
    b = 0.1 * torch.randn(cout, generator=_g(6), device=DEV, dtype=F64)
    cv = ip._Conv(w, b, 3, 1, 1, 1, DEV)
    assert cv.tc is not None
    bias = cv.pk[1]
    x = torch.randn(Bn, h, h, cin, generator=_g(7), device=DEV).to(F16)
    y = torch.full((Bn, h, h, cout), float('nan'), device=DEV, dtype=F16)
    capi.check(capi.lib().r3dp_sr_tc_conv(P(x, F16), P(cv.tc, F16), P(bias), Bn, 1, cin, cout, h, h, 3, act, P(y, F16), capi.stream()))
    torch.cuda.synchronize()
    wv = scr.taps3x3(scr.packed_weights(cv.tc.view(1, 9, cout, cin), cin, False))
    xv = scr.activations(x, cin, False)
    bv = bias[:cout].to(F64)
    ref = scr.bias_act(scr.conv_same(xv, wv), bv, act)
    S = scr.act_gain(act) * (scr.conv_same(xv.abs(), wv.abs()) + bv.abs().view(1, -1, 1, 1))
    scr.check_bound(scr.nhwc(y, False), ref, S, scr.ALPHA_F16, scr.BETA['tc'], extra=scr.FLOOR_F16, tag=name)
