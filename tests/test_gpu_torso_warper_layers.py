"""Every stage-2 entry point of the torso warper (r3dp_tw_*) layer by layer against float64 references built from the operands the kernel reads,
with the element-wise bound of tests/sr_conv_reference.py (|got - ref| <= alpha |ref| + extra + beta S), in 'tc' and 'tc_exact' (split).  Every
output lives inside a NaN-filled allocation: nothing before or after it is written and every element of it is.  The persistent conv launches
also show that the last image of an N > 1 launch is the N = 1 launch of that image, bit for bit.  The run_* helpers take a launch's
arguments; tests/test_gpu_torso_warper_launches.py calls them at every launch of the warper (N = 4 and 1)."""
import pytest
import torch
import torch.nn.functional as F

from real3dportrait_b200 import _capi as capi, sr_tc
import sr_conv_reference as scr
import torso_warper_ref as twr

pytestmark = pytest.mark.gpu
DEV = 'cuda'
F16 = torch.float16
PAD = 4096
U32 = 2.0 ** -24                         # fp32 unit roundoff


def _canary(shape, dtype):
    """(buffer, output view): the output sits between two PAD-element NaN guards."""
    n = 1
    for s in shape:
        n *= s
    buf = torch.full((n + 2 * PAD,), float('nan'), device=DEV, dtype=dtype)
    return buf, buf[PAD:PAD + n].view(*shape)


def _check_canary(buf, out, tag):
    torch.cuda.synchronize()
    assert bool(torch.isnan(buf[:PAD]).all()) and bool(torch.isnan(buf[-PAD:]).all()), f'{tag}: written outside the output'
    assert bool(torch.isfinite(out).all()), f'{tag}: an output element was not written'


def _nhwc(x: torch.Tensor, split: bool) -> torch.Tensor:
    """fp32 NCHW [N,C,H,W] (any H, W) -> NHWC fp16 with channels padded to 64 ([hi | lo] halves when split)."""
    N, C, H, W = x.shape
    Cp = (C + 63) // 64 * 64
    xp = torch.zeros(N, H, W, Cp, device=x.device)
    xp[..., :C] = x.permute(0, 2, 3, 1)
    hi = xp.half()
    return torch.cat([hi, (xp - hi.float()).half()], dim=-1) if split else hi


def _pack(w: torch.Tensor, split: bool) -> torch.Tensor:
    """fp32 [nw,O,I,3,3] -> packed [nw,9,O,Ip(*2)] by the library's packer."""
    nw, O, I = w.shape[:3]
    out = torch.empty(nw, 9, O, (I + 63) // 64 * 64 * (2 if split else 1), device=DEV, dtype=F16)
    capi.check(sr_tc._fn('pack_weights', split)(capi.ptr(w.contiguous()), nw, O, I, capi.ptr(out, F16), capi.stream()))
    return out


def _act(v, slope):
    return torch.maximum(v, v * slope)


# N, H, W, I, O, ksize, slope, residual: the stage's own layers (in_conv, mid_conv, res conv1 / conv2) and the other widths the entry point takes
CONV_CASES = [
    (3, 64, 64, 512, 256, 3, 0.2, False),
    (3, 64, 64, 256, 256, 1, 1.0, False),
    (3, 64, 64, 256, 256, 3, 0.0, False),
    (3, 64, 64, 256, 256, 3, 1.0, True),
    (3, 32, 128, 128, 128, 3, 0.0, True),
    (3, 16, 256, 64, 128, 3, 0.2, False),
    (3, 64, 64, 32, 128, 3, 0.2, False),          # I <= 32: the 32-channel K chunks at W = 64 (one tile per row, its right half TMA zero fill)
]


@pytest.mark.parametrize('case', CONV_CASES, ids=lambda c: f'N{c[0]}_{c[1]}x{c[2]}_{c[3]}to{c[4]}_k{c[5]}_s{c[6]}_res{int(c[7])}')
@pytest.mark.parametrize('split', [False, True], ids=['tc', 'tcx'])
def test_tw_conv(case, split):
    run_tw_conv(case, split)


def run_tw_conv(case, split):
    """One r3dp_tw_conv launch (N, H, W, I, O, ksize, slope, residual) against float64, one image at a time; the last image of an N > 1
    launch equals its N = 1 launch bit for bit."""
    N, H, W, I, O, k, slope, res = case
    g = torch.Generator().manual_seed(H * 7 + W + I + O + k + int(res))
    x16 = _nhwc(torch.randn(N, I, H, W, generator=g).to(DEV), split)
    wf = (torch.randn(1, O, I, 3, 3, generator=g) / (I * 3)).to(DEV)
    if k == 1:
        wf[..., :, :] *= torch.tensor([[0., 0., 0.], [0., 1., 0.], [0., 0., 0.]], device=DEV)
    b = (0.1 * torch.randn(O, generator=g)).to(DEV)
    wp = _pack(wf, split)
    wide = 2 if split else 1
    r16 = _nhwc(torch.randn(N, O, H, W, generator=g).to(DEV), split) if res else None
    buf, y = _canary((N, H, W, O * wide), F16)

    def run(xx, rr, yy, n):
        capi.check(capi.lib().r3dp_tw_conv(capi.ptr(xx, F16), capi.ptr(wp, F16), capi.ptr(b), n, I, O, H, W, k, slope, capi.ptr(rr, F16),
                                           capi.ptr(yy, F16), int(split), capi.stream()))
    run(x16, r16, y, N)
    _check_canary(buf, y, 'tw_conv')
    w = scr.taps3x3(scr.packed_weights(wp, I, split))
    for n in range(N):
        x = scr.activations(x16[n:n + 1], I, split)
        v = scr.conv_same(x, w, k) + b.double().view(1, -1, 1, 1)
        S = scr.conv_same(x.abs(), w.abs(), k) + b.double().abs().view(1, -1, 1, 1)
        ref, extra = _act(v, slope), scr.FLOOR_F16
        if res:
            r = scr.activations(r16[n:n + 1], O, split)
            if not split:                              # tc rounds the activated value to fp16 before adding the residual
                extra = extra + scr.ALPHA_F16 * ref.abs() + scr.FLOOR_F16
            ref, S = ref + r, S + r.abs()
        scr.check_bound(scr.nhwc(y[n:n + 1], split), ref, S, scr.alpha_store(split), scr.BETA['tcx' if split else 'tc'], extra,
                        tag=f'tw_conv {case} image {n}')
    if N > 1:
        y1 = torch.empty(1, H, W, O * wide, device=DEV, dtype=F16)
        run(x16[N - 1:].contiguous(), None if r16 is None else r16[N - 1:].contiguous(), y1, 1)
        assert torch.equal(y1[0].view(torch.int16), y[N - 1].view(torch.int16)), f'the last image of the N={N} launch differs from its N=1 launch'


# N, H, W, I, O, slope: up.0 and up.1 of the Generator (the 64 couts of up.1 padded with zero filters to 128) and a linear case
UP_CASES = [(3, 64, 64, 256, 128, 0.0), (1, 128, 128, 128, 128, 0.0), (3, 32, 64, 64, 256, 1.0)]


@pytest.mark.parametrize('case', UP_CASES, ids=lambda c: f'N{c[0]}_{c[1]}x{c[2]}_{c[3]}to{c[4]}_s{c[5]}')
@pytest.mark.parametrize('split', [False, True], ids=['tc', 'tcx'])
def test_tw_conv_up_nearest(case, split):
    """nearest x2 + 3x3 as four parity phases of 2x2 composed taps, against the same taps in float64 (and those taps against
    upsample-then-conv of the unpacked composition in tests/test_cpu_torso_warper.py)."""
    run_up_nearest(case, split)


def run_up_nearest(case, split):
    """One r3dp_tw_conv_up_nearest launch (N, H, W, I, O, slope) against float64, one image at a time; the last image of an N > 1 launch
    equals its N = 1 launch bit for bit."""
    N, H, W, I, O, slope = case
    g = torch.Generator().manual_seed(H + W + I + O)
    x16 = _nhwc(torch.randn(N, I, H, W, generator=g).to(DEV), split)
    w3 = (torch.randn(O, I, 3, 3, generator=g) / (I * 3)).double()
    from real3dportrait_b200 import torso_warp as tw
    wp = _pack(tw.compose_nearest_up(w3).float().to(DEV), split)
    b = (0.1 * torch.randn(O, generator=g)).to(DEV)
    wide = 2 if split else 1
    buf, y = _canary((N, 2 * H, 2 * W, O * wide), F16)

    def run(xx, yy, n):
        capi.check(capi.lib().r3dp_tw_conv_up_nearest(capi.ptr(xx, F16), capi.ptr(wp, F16), capi.ptr(b), n, I, O, H, W, slope, capi.ptr(yy, F16),
                                                       int(split), capi.stream()))
    run(x16, y, N)
    _check_canary(buf, y, 'tw_conv_up_nearest')
    w4 = scr.taps3x3(scr.packed_weights(wp, I, split))                  # [4,O,I,3,3]
    for n in range(N):
        x = scr.activations(x16[n:n + 1], I, split)
        ref = _act(twr.conv_up_nearest_phases(x, w4, b.double()), slope)
        S = twr.conv_up_nearest_phases(x.abs(), w4.abs(), b.double().abs())
        scr.check_bound(scr.nhwc(y[n:n + 1], split), ref, S, scr.alpha_store(split), scr.BETA['tcx' if split else 'tc'], scr.FLOOR_F16,
                        tag=f'up_nearest {case} image {n}')
    if N > 1:
        y1 = torch.empty(1, 2 * H, 2 * W, O * wide, device=DEV, dtype=F16)
        run(x16[N - 1:].contiguous(), y1, 1)
        assert torch.equal(y1[0].view(torch.int16), y[N - 1].view(torch.int16)), f'the last image of the N={N} launch differs from its N=1 launch'


@pytest.mark.parametrize('split', [False, True], ids=['tc', 'tcx'])
def test_tw_affine_relu(split):
    N, H, W, C = 3, 64, 64, 256
    g = torch.Generator().manual_seed(4)
    x16 = sr_tc.to_nhwc_f16(3 * torch.randn(N, C, H, W, generator=g).to(DEV), W, split)
    s, t = (0.5 + torch.rand(C, generator=g)).to(DEV), (0.3 * torch.randn(C, generator=g)).to(DEV)
    buf, y = _canary(tuple(x16.shape), F16)
    capi.check(capi.lib().r3dp_tw_affine_relu(capi.ptr(x16, F16), capi.ptr(s), capi.ptr(t), N, H, W, C, int(split), capi.ptr(y, F16), capi.stream()))
    _check_canary(buf, y, 'affine_relu')
    x = scr.activations(x16, C, split)
    ref = torch.relu(x * s.double().view(1, -1, 1, 1) + t.double().view(1, -1, 1, 1))
    S = x.abs() * s.double().view(1, -1, 1, 1) + t.double().abs().view(1, -1, 1, 1)
    # fp32: hi + lo summed (split), one fma: a few roundings of S
    scr.check_bound(scr.nhwc(y, split), ref, S, scr.alpha_store(split), 4 * U32, scr.FLOOR_F16, tag='affine_relu')


# K, CO, act, input: 'f16' (64 of 128 channels, optionally split), 'f32' (32 dense channels); ex: the occlusion map resized on the fly
NARROW_CASES = [
    (7, 3, 0, 'f16', False, True),       # out_conv -> rgb_torso NCHW
    (3, 32, 1, 'f16', True, False),      # predictor 0: hid + bilinear_up(occlusion_2) -> 32, ReLU, NHWC
    (3, 32, 1, 'f32', False, False),     # predictor 1
    (3, 1, 2, 'f32', False, True),       # predictor 2: sigmoid, NCHW
]


@pytest.mark.parametrize('case', NARROW_CASES, ids=lambda c: f'k{c[0]}_co{c[1]}_act{c[2]}_{c[3]}_ex{int(c[4])}')
@pytest.mark.parametrize('split', [False, True], ids=['tc', 'tcx'])
def test_tw_narrow_conv(case, split):
    run_narrow_conv(case, split, 3)


def run_narrow_conv(case, split, N):
    """One r3dp_tw_narrow_conv launch (K, CO, act, input kind, resized extra channel, NCHW output) on N images of 256^2 against float64,
    one image at a time."""
    K, CO, act, kind, with_ex, nchw = case
    H, W = 256, 256
    g = torch.Generator().manual_seed(K + CO + act)
    L = capi.lib()
    if kind == 'f16':
        xa = sr_tc.to_nhwc_f16(torch.randn(N, 128, H, W, generator=g).to(DEV), W, split)   # hid layout: 128 channels, 64 used
        ca, sa, lo = 64, xa.shape[-1], (128 if split else 0)
        x = scr.activations(xa, 64, split)
        xf = None
    else:
        xf = torch.randn(N, H, W, 32, generator=g).to(DEV)
        x = xf.double().permute(0, 3, 1, 2)
        xa = None
    ex = torch.sigmoid(torch.randn(N, 1, 64, 64, generator=g)).to(DEV) if with_ex else None
    cin = x.shape[1] + (1 if with_ex else 0)
    w = (torch.randn(CO, cin, K, K, generator=g) / (cin * K)).to(DEV)
    b = (0.1 * torch.randn(CO, generator=g)).to(DEV)
    wk = w.permute(2, 3, 1, 0).contiguous()
    buf, y = _canary((N, CO, H, W) if nchw else (N, H, W, CO), torch.float32)
    if kind == 'f16':
        capi.check(L.r3dp_tw_narrow_conv(capi.ptr(xa, F16), sa, ca, lo, None, 0, 0, capi.ptr(ex), 64 if with_ex else 0, 64 if with_ex else 0,
                                         capi.ptr(wk), capi.ptr(b), N, H, W, K, CO, act, int(nchw), capi.ptr(y), capi.stream()))
    else:
        capi.check(L.r3dp_tw_narrow_conv(None, 0, 0, 0, capi.ptr(xf), 32, 32, capi.ptr(ex), 64 if with_ex else 0, 64 if with_ex else 0,
                                         capi.ptr(wk), capi.ptr(b), N, H, W, K, CO, act, int(nchw), capi.ptr(y), capi.stream()))
    _check_canary(buf, y, 'narrow_conv')
    # fp32 accumulation of K*K*cin products in order: |err| <= K*K*cin * 2^-24 S (gamma_n); the resized channel adds its fp32 interpolation
    beta = K * K * cin * U32 + (8 * U32 if with_ex else 0)
    for n in range(N):
        xn = x[n:n + 1]
        if with_ex:
            xn = torch.cat([xn, F.interpolate(ex[n:n + 1].double(), size=(H, W), mode='bilinear', align_corners=False)], dim=1)
        v = F.conv2d(xn, w.double(), b.double(), padding=K // 2)
        S = F.conv2d(xn.abs(), w.double().abs(), b.double().abs(), padding=K // 2)
        if act == 2:                                # sigmoid is 1/4-Lipschitz; expf / the division add a few ulp of the result
            ref, S, alpha = torch.sigmoid(v), 0.25 * S, 8 * U32
        else:
            ref, alpha = (torch.relu(v) if act == 1 else v), U32
        got = y[n:n + 1].double() if nchw else y[n:n + 1].double().permute(0, 3, 1, 2)
        scr.check_bound(got, ref, S, alpha, beta, tag=f'narrow_conv {case} N{N} image {n}')


@pytest.mark.parametrize('split', [False, True], ids=['tc', 'tcx'])
def test_tw_hid_to_nchw(split):
    """hi (+ lo) summed in fp32 and transposed: bit for bit."""
    run_hid_to_nchw(split, 3)


def run_hid_to_nchw(split, N):
    H, W = 256, 256
    hid = sr_tc.to_nhwc_f16(torch.randn(N, 128, H, W, generator=torch.Generator().manual_seed(1)).to(DEV), W, split)
    buf, y = _canary((N, 64, H, W), torch.float32)
    capi.check(capi.lib().r3dp_tw_hid_to_nchw(capi.ptr(hid, F16), N, 64, H, W, hid.shape[-1], 128 if split else 0, capi.ptr(y), capi.stream()))
    _check_canary(buf, y, 'hid_to_nchw')
    ref = hid[..., :64].float() + (hid[..., 128:192].float() if split else 0)
    assert torch.equal(y, ref.permute(0, 3, 1, 2))


@pytest.mark.parametrize('split', [False, True], ids=['tc', 'tcx'])
def test_tw_gather3d_canary_and_shared_volume(split):
    """The gather inside NaN guards, N = 3; fs_shared reads one volume for every image and equals the launch on its broadcast copy bit for bit."""
    run_gather3d(split, 3, True)


def run_gather3d(split, N, shared):
    """r3dp_tw_gather3d on N images at 64^2 inside NaN guards against float64, one image at a time.  shared (N > 1): one volume read by every
    image, bit for bit the launch on its broadcast copy; otherwise each image reads its own volume."""
    fs, deformation, _ = twr.make_stage2_inputs(N, 64, seed=12)
    vol = fs[:1] if shared else fs                                     # [1 or N, 32, 16, 64, 64]
    fsn = vol.permute(0, 2, 3, 4, 1).contiguous().to(DEV)
    deformation = deformation.to(DEV)
    wide = 2 if split else 1
    buf, y = _canary((N, 64, 64, 512 * wide), F16)
    L = capi.lib()
    capi.check(L.r3dp_tw_gather3d(capi.ptr(fsn), int(shared), capi.ptr(deformation), N, 32, 16, 64, 64, capi.ptr(y, F16), int(split), capi.stream()))
    _check_canary(buf, y, 'gather3d')
    if shared:
        y_b = torch.empty_like(y)
        capi.check(L.r3dp_tw_gather3d(capi.ptr(fsn.expand(N, -1, -1, -1, -1).contiguous()), 0, capi.ptr(deformation), N, 32, 16, 64, 64,
                                      capi.ptr(y_b, F16), int(split), capi.stream()))
        assert torch.equal(y.view(torch.int16), y_b.view(torch.int16))
    # The kernel unnormalises the coordinates in fp32 (as torch's fp32 grid_sample does): each of the three source coordinates is off by at
    # most delta = 4 ulp of (size - 1) <= 4 * 63 * 2^-24 voxels, which moves the trilinear weights of each axis by delta and the value by at most
    # 2 * delta * max|fs| per axis.  The weighted sum of 8 corners in fp32 adds <= 12 * 2^-24 S; the store rounds as the convs' do.
    delta = 4 * 63 * U32
    for n in range(N):
        v = vol[0 if shared else n][None].double().to(DEV)
        ref = F.grid_sample(v, deformation[n:n + 1].double(), align_corners=True, padding_mode='border').reshape(1, 512, 64, 64)
        S = F.grid_sample(v.abs(), deformation[n:n + 1].double(), align_corners=True, padding_mode='border').reshape(1, 512, 64, 64)
        extra = 3 * 2 * delta * float(v.abs().max()) + scr.FLOOR_F16
        scr.check_bound(scr.nhwc(y[n:n + 1], split), ref, S, scr.alpha_store(split), 16 * U32, extra, tag=f'gather3d N{N} shared{int(shared)} image {n}')
