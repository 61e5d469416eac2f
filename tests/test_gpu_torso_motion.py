"""torso_motion='cuda' on the GPU: the 3-D wgmma convolution (csrc/conv3d_tc.cu r3dp_mf_conv3d) against float64 for every shape the motion-field
estimator uses plus ragged ones, the kernels around it against torch float64, the whole estimator against the reference's own
MotionFieldEstimator('standard', 34, 4) (TF32 off), the torso head end to end, and a FrameEngine clip (graph = eager, bit for bit)."""
import pytest
import torch
import torch.nn.functional as F

import real3dportrait_b200 as r3
from real3dportrait_b200 import _capi as capi, synthetic as syn, torso_warp as tw
import sr_conv_reference as scr
import torso_motion_reference as tmr
import torso_warper_ref as twr

pytestmark = pytest.mark.gpu
DEV = 'cuda'
F16 = torch.float16
# Measured on an H100 80GB HBM3, 700 W power limit (max-abs / range against the reference modules in fp32, TF32 off):
#   estimator   K = 4  tc: deformation 7.1e-5, occlusion 4.3e-4, occlusion_2 3.7e-4    tc_exact: 1.6e-5, 5.0e-5, 4.5e-5
#               K = 9  tc: 1.0e-4, 3.8e-4, 3.9e-4                                     tc_exact: 3.0e-5, 7.9e-5, 9.8e-5
#   whole head  tc: image 2.8e-4, occlusion_2 2.5e-3                            tc_exact: 2.2e-5, 2.5e-4
EXACT_REL = 1e-3                  # the project's tc_exact bar: max-abs < 1e-3 * range
EST_TC_REL = 1e-3                 # the estimator alone in tc: 2.3x over its largest measured value (occlusion, 4.3e-4)
TC_REL = 5e-3                     # the whole head in tc (the estimator's 15 convs, then stage 2's 16): 2x over its largest value (occlusion_2)


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max()) / max(float(b.max() - b.min()), 1e-12)


def _store(v: torch.Tensor, split: bool) -> torch.Tensor:
    """float tensor [..., C] -> fp16 [..., C] or split [..., 2C] = [hi | lo]."""
    hi = v.half()
    return torch.cat([hi, (v.double() - hi.double()).half()], -1) if split else hi


def _unpack(wp: torch.Tensor, cin: int, split: bool) -> torch.Tensor:
    """packed [nph,taps,cop,cin(x2)] -> float64 [nph,taps,cop,cin] as the kernel reads it."""
    return (wp[..., :cin].double() + wp[..., cin:].double()) / 1024.0 if split else wp.double()


def _run_conv(N, D, H, W, cin_real, cout, taps, up, split, relu=1, res=False, slice_=False, seed=0, out_f32=False):
    g = torch.Generator().manual_seed(seed)
    cin = (cin_real + 31) // 32 * 32
    wide = 2 if split else 1
    nph = 4 if up else 1
    x = torch.randn(N, D, H, W, cin_real, generator=g)
    w = torch.randn(nph, cout, cin_real, *taps, generator=g) / (cin_real * taps[0] * taps[1] * taps[2]) ** 0.5
    b = 0.1 * torch.randn(cout, generator=g)
    xs_pad = cin + 8                                                        # a wider voxel than the channels read
    xfull = torch.zeros(N, D, H, W, xs_pad)
    xfull[..., :cin_real] = x
    x16 = _store(xfull.to(DEV), split).contiguous()
    wp, bias, O, cop = tw.pack_conv3d(w.double().to(DEV), b.double().to(DEV), cin, split)
    Ho, Wo = (2 * H, 2 * W) if up else (H, W)
    yc0 = 6 if slice_ else 0
    cs = yc0 + cout + (4 if slice_ else 0)
    cs += cs % 2
    if out_f32:
        buf = torch.full((N * D * Ho * Wo * cs + 4096,), -7.0, device=DEV)
        y = buf[:N * D * Ho * Wo * cs].view(N, D, Ho, Wo, cs)
        ys, ylo = cs, 0
    else:
        buf = torch.full((N * D * Ho * Wo * cs * wide + 4096,), -7.0, device=DEV, dtype=F16)
        y = buf[:N * D * Ho * Wo * cs * wide].view(N, D, Ho, Wo, cs * wide)
        ys, ylo = cs * wide, cs
    r16 = None
    if res:
        r = torch.randn(N, D, Ho, Wo, cs, generator=g).to(DEV)
        r16 = _store(r, split).contiguous()
    capi.check(capi.lib().r3dp_mf_conv3d(capi.ptr(x16, F16), xs_pad * wide, xs_pad, cin, capi.ptr(wp, F16), capi.ptr(bias), capi.ptr(r16, F16), N, D, H, W,
                                         *taps, int(up), O, cop, relu, capi.ptr(y, torch.float32 if out_f32 else F16), ys, yc0, ylo, int(out_f32),
                                         int(split), capi.stream()))
    torch.cuda.synchronize()
    assert bool((buf[-4096:] == -7.0).all()), 'written past the output'
    xin = (scr.join(x16) if split else x16.double())[..., :cin].permute(0, 4, 1, 2, 3)
    wd = _unpack(wp, cin, split)[:, :, :O]
    pre = tmr.ref_conv(xin, wd, taps, up, bias[:O])
    S = tmr.ref_conv(xin.abs(), wd.abs(), taps, up, bias[:O].abs())
    ref = torch.relu(pre) if relu else pre
    if res:
        rv = (scr.join(r16) if split else r16.double())[..., yc0:yc0 + cout].permute(0, 4, 1, 2, 3)
        ref, S = ref + rv, S + rv.abs()
    got_all = y.double() if out_f32 else (scr.join(y) if split else y.double())
    got = got_all[..., yc0:yc0 + cout].permute(0, 4, 1, 2, 3)
    raw = y[..., :cs] if not (split and not out_f32) else torch.cat([y[..., :cs], y[..., cs:]], -1)
    inside = torch.zeros(cs, dtype=torch.bool)
    inside[yc0:yc0 + cout] = True
    ins = inside.repeat(1 if out_f32 else wide).to(DEV)
    assert not bool((raw[..., ins] == -7.0).any()), 'an output element was not written'
    assert bool((raw[..., ~ins] == -7.0).all()), 'written outside the channel slice'
    alpha = scr.ALPHA_F32 if out_f32 else scr.alpha_store(split)
    extra = 0.0 if out_f32 else (2 * scr.FLOOR_F16 + (scr.ALPHA_F16 * pre.abs() if (res and not split) else 0.0))
    return scr.check_bound(got, ref, S, alpha, tmr.BETA3[split], extra, tag=f'conv3d N{N} D{D} {H}x{W} {cin_real}->{cout} {taps} up{up} split{split}'), \
        (x16, wp, bias, y)


# every conv shape of the estimator at batch 2 (the down / up layers at their own resolutions), then the ragged cases
EST_CASES = [
    dict(N=2, D=16, H=64, W=64, cin_real=25, cout=64, taps=(3, 3, 3), up=0),          # down.0 (input 25 -> 32 channels)
    dict(N=2, D=16, H=32, W=32, cin_real=64, cout=128, taps=(3, 3, 3), up=0),         # down.1
    dict(N=2, D=16, H=16, W=16, cin_real=128, cout=256, taps=(3, 3, 3), up=0),        # down.2
    dict(N=2, D=16, H=8, W=8, cin_real=256, cout=512, taps=(3, 3, 3), up=0),          # down.3
    dict(N=2, D=16, H=4, W=4, cin_real=512, cout=1024, taps=(3, 3, 3), up=0),         # down.4
    dict(N=2, D=16, H=2, W=2, cin_real=1024, cout=512, taps=(3, 2, 2), up=1),         # up.0 (W = 2: tiles span rows, slices, images)
    dict(N=2, D=16, H=4, W=4, cin_real=512, cout=256, taps=(3, 2, 2), up=1),          # up.1
    dict(N=2, D=16, H=8, W=8, cin_real=256, cout=128, taps=(3, 2, 2), up=1),          # up.2
    dict(N=2, D=16, H=16, W=16, cin_real=128, cout=64, taps=(3, 2, 2), up=1),         # up.3
    dict(N=2, D=16, H=32, W=32, cin_real=64, cout=32, taps=(3, 2, 2), up=1, slice_=True),  # up.4 (into a slice of the fuser input)
    dict(N=2, D=1, H=128, W=128, cin_real=4, cout=32, taps=(1, 7, 7), up=0),          # tgt-head encoder 7x7 (D = 1)
    dict(N=2, D=1, H=128, W=128, cin_real=32, cout=32, taps=(1, 3, 3), up=0),         # encoder res conv1 (BN2 folded, ReLU)
    dict(N=2, D=1, H=128, W=128, cin_real=32, cout=32, taps=(1, 3, 3), up=0, relu=0, res=True),  # encoder res conv2 + residual
    dict(N=2, D=16, H=64, W=64, cin_real=89, cout=32, taps=(7, 7, 7), up=0, relu=0),  # fuser, K = 4
    dict(N=2, D=16, H=64, W=64, cin_real=114, cout=32, taps=(7, 7, 7), up=0, relu=0),  # fuser, K = 9 (114 -> 128 channels)
    dict(N=2, D=16, H=64, W=64, cin_real=32, cout=5, taps=(7, 7, 7), up=0, relu=0, out_f32=True),   # mask logits, K = 4
    dict(N=2, D=16, H=64, W=64, cin_real=32, cout=10, taps=(7, 7, 7), up=0, relu=0, out_f32=True),  # mask logits, K = 9
]
RAGGED = [
    dict(N=3, D=3, H=5, W=2, cin_real=25, cout=5, taps=(3, 3, 3), up=0),              # M = 90: one partial tile, Cout = 5
    dict(N=3, D=2, H=3, W=2, cin_real=64, cout=40, taps=(3, 2, 2), up=1, slice_=True),
    dict(N=1, D=1, H=9, W=7, cin_real=96, cout=130, taps=(1, 3, 3), up=0, res=True),  # two cout tiles, the second ragged
    dict(N=3, D=4, H=6, W=6, cin_real=89, cout=32, taps=(7, 7, 7), up=0, relu=0, slice_=True),
]


@pytest.mark.parametrize('split', [False, True])
@pytest.mark.parametrize('case', range(len(EST_CASES) + len(RAGGED)))
def test_conv3d_conformance(case, split):
    kw = dict((EST_CASES + RAGGED)[case])
    _run_conv(split=split, seed=case, **kw)


@pytest.mark.parametrize('split', [False, True])
def test_conv3d_batch_and_repeat_bits(split):
    """Image k of an N = 3 launch equals the N = 1 launch on that image, and a repeated launch gives the same bits."""
    _, (x16, wp, bias, y) = _run_conv(3, 4, 6, 6, 89, 32, (7, 7, 7), 0, split, relu=0, seed=11)
    wide = 2 if split else 1
    cin, cs = 96, y.shape[-1] // wide

    def launch(xx, n):
        out = torch.empty(n, *y.shape[1:], device=DEV, dtype=F16)
        capi.check(capi.lib().r3dp_mf_conv3d(capi.ptr(xx, F16), x16.shape[-1], x16.shape[-1] // wide, cin, capi.ptr(wp, F16), capi.ptr(bias), None,
                                             n, 4, 6, 6, 7, 7, 7, 0, 32, 32, 0, capi.ptr(out, F16), cs * wide, 0, cs, 0, int(split), capi.stream()))
        return out
    a, b = launch(x16, 3), launch(x16, 3)
    one = launch(x16[1:2].contiguous(), 1)
    assert torch.equal(a, b) and torch.equal(a[1:2], one)


# ---- the kernels around the convolutions --------------------------------------------------------------------------------------------------
def _grid(D, H, W, dev):
    lin = lambda n: 2 * (torch.arange(n, device=dev, dtype=torch.float64) / (n - 1)) - 1        # noqa: E731
    z, y, x = torch.meshgrid(lin(D), lin(H), lin(W), indexing='ij')
    return torch.stack([x, y, z], -1)                                         # components (W, H, D)


def _input_f64(fc, kp_s, kp_d):
    """float64 restatement of the estimator's input: [N,(K+1)*5,D,H,W]."""
    N, D, H, W, _ = fc.shape
    K = kp_s.shape[1]
    grid = _grid(D, H, W, fc.device)
    src = fc.double().permute(0, 4, 1, 2, 3)
    chans = []
    for k in range(K + 1):
        if k == 0:
            hm, sm = torch.zeros(N, D, H, W, dtype=torch.float64, device=fc.device), grid.expand(N, -1, -1, -1, -1)
        else:
            gd = lambda kp: torch.exp(-0.5 * ((grid[None] - kp.double()[:, k - 1, None, None, None]) ** 2).sum(-1) / 0.01)   # noqa: E731
            hm = gd(kp_d) - gd(kp_s)
            sm = grid[None] - kp_d.double()[:, k - 1, None, None, None] + kp_s.double()[:, k - 1, None, None, None]
        chans.append(hm[:, None])
        chans.append(F.grid_sample(src, sm, mode='bilinear', padding_mode='zeros', align_corners=True))
    return torch.cat(chans, 1)


@pytest.mark.parametrize('split', [False, True])
def test_input_kernel(split):
    g = torch.Generator().manual_seed(3)
    N, K, D, S = 2, 4, 16, 64
    fc = torch.randn(1, D, S, S, 4, generator=g).to(DEV)
    kp_s, kp_d = [(0.9 * (2 * torch.rand(N, K, 3, generator=g) - 1)).to(DEV) for _ in range(2)]
    P0, CF = 32, 96
    y = torch.full((N, D, S, S, CF * (2 if split else 1)), -7.0, device=DEV, dtype=F16)
    capi.check(capi.lib().r3dp_mf_input(capi.ptr(fc), 1, capi.ptr(kp_s), capi.ptr(kp_d), N, K, D, S, S, P0, capi.ptr(y, F16), y.shape[-1], CF, int(split),
                                        capi.stream()))
    got = (y[..., :CF].double() + (y[..., CF:].double() if split else 0))[..., :P0]
    ref = _input_f64(fc.expand(N, -1, -1, -1, -1), kp_s, kp_d).permute(0, 2, 3, 4, 1)
    err = float((got[..., :25] - ref).abs().max())
    print(f'input kernel split={split}: max abs err {err:.2e}')
    # split: the kernel's fp32 arithmetic (coordinates, expf of arguments down to -600, trilinear weights), measured 2.0e-5 on an H100
    assert err < (1e-4 if split else 2e-3 * float(ref.abs().max())), err
    assert bool((got[..., 25:] == 0).all())


@pytest.mark.parametrize('K', [4, 9])
def test_input_and_deform_against_reference_func_utils(K):
    """r3dp_mf_input and r3dp_mf_deform against the reference's own create_heatmap_representations, create_sparse_motions and
    create_deformed_source_image (func_utils.py:130-191, Rs = Rd = I), run in fp32 on the same device.  Split outputs: the comparison sees the
    kernels' fp32 arithmetic, not the fp16 storage."""
    if not twr.ref_classes():
        pytest.skip('the reference warper modules are not staged under oracle/_ref')
    from modules.real3d.facev2v_warp import func_utils as fu
    g = torch.Generator().manual_seed(21 + K)
    N, D, S = 2, 16, 64
    c0, P0 = (K + 1) * 5, ((K + 1) * 5 + 31) // 32 * 32
    fc = torch.randn(1, D, S, S, 4, generator=g).to(DEV)
    kp_s, kp_d = [(0.9 * (2 * torch.rand(N, K, 3, generator=g) - 1)).to(DEV) for _ in range(2)]
    fs = fc.permute(0, 4, 1, 2, 3).expand(N, -1, -1, -1, -1).contiguous()
    eye = torch.eye(3, device=DEV)[None].repeat(N, 1, 1)
    with torch.no_grad():
        sparse = fu.create_sparse_motions(fs, kp_s, kp_d, eye, eye)
        ref_in = torch.cat([fu.create_heatmap_representations(fs, kp_s, kp_d), fu.create_deformed_source_image(fs, sparse)], dim=2)
        ref_in = ref_in.reshape(N, -1, D, S, S).permute(0, 2, 3, 4, 1)
    y = torch.empty(N, D, S, S, 2 * P0, device=DEV, dtype=F16)
    L, st = capi.lib(), capi.stream()
    capi.check(L.r3dp_mf_input(capi.ptr(fc), 1, capi.ptr(kp_s), capi.ptr(kp_d), N, K, D, S, S, P0, capi.ptr(y, F16), 2 * P0, P0, 1, st))
    e_in = float((scr.join(y)[..., :c0] - ref_in.double()).abs().max())
    ls = (K + 2) // 2 * 2
    logits = torch.randn(N, D, S, S, ls, generator=g).to(DEV)
    de = torch.empty(N, D, S, S, 3, device=DEV)
    capi.check(L.r3dp_mf_deform(capi.ptr(logits), ls, capi.ptr(kp_s), capi.ptr(kp_d), N, K, D, S, S, capi.ptr(de), st))
    mask = F.softmax(logits[..., :K + 1].permute(0, 4, 1, 2, 3), dim=1).unsqueeze(-1)
    e_de = float((de - (sparse * mask).sum(dim=1)).abs().max())
    print(f'K={K}: input max abs err {e_in:.2e}, deformation {e_de:.2e}')
    # both sides compute in fp32; the input's worst differences sit on the steep flanks of the 0.01-variance Gaussians.  Measured on an
    # H100: input 3.9e-5 (K = 4 and 9), deformation 4.8e-7
    assert e_in < 1e-4 and e_de < 1e-5, (e_in, e_de)


def test_small_kernels():
    """pool, tgt-head input, head broadcast, softmax / deformation and the occlusion pair against torch float64 (split operands)."""
    g = torch.Generator().manual_seed(4)
    L, st = capi.lib(), capi.stream()
    N, D = 2, 16
    # AvgPool3d (1,2,2)
    x = torch.randn(N, D, 8, 8, 64, generator=g).to(DEV)
    x16 = _store(x, True)
    y = torch.empty(N, D, 4, 4, 128, device=DEV, dtype=F16)
    capi.check(L.r3dp_mf_pool(capi.ptr(x16, F16), N, D, 4, 4, 64, 128, 64, capi.ptr(y, F16), 128, 64, 1, st))
    ref = F.avg_pool3d(scr.join(x16).permute(0, 4, 1, 2, 3), (1, 2, 2)).permute(0, 2, 3, 4, 1)
    assert float((scr.join(y) - ref).abs().max()) < 1e-6
    # tgt-head input = interpolate(cat[rgb, w], 1/2, bilinear)
    rgb, wt = torch.randn(N, 3, 256, 256, generator=g).to(DEV), torch.rand(N, 1, 256, 256, generator=g).to(DEV)
    e = torch.empty(N, 128, 128, 64, device=DEV, dtype=F16)
    capi.check(L.r3dp_mf_head_input(capi.ptr(rgb), capi.ptr(wt), N, 128, 128, 32, capi.ptr(e, F16), 64, 32, 1, st))
    ref = F.interpolate(torch.cat([rgb, wt], 1).double(), size=(128, 128), mode='bilinear').permute(0, 2, 3, 1)
    assert float((scr.join(e)[..., :4] - ref).abs().max()) < 1e-6 and bool((scr.join(e)[..., 4:] == 0).all())
    # 128 -> 64 mean broadcast over depth into a channel slice
    xf = torch.zeros(N, D, 64, 64, 192, device=DEV, dtype=F16)
    capi.check(L.r3dp_mf_head_bcast(capi.ptr(e, F16), N, D, 64, 64, 32, 64, 32, capi.ptr(xf, F16), 192, 64, 96, 1, st))
    ref = F.interpolate(scr.join(e).permute(0, 3, 1, 2), size=(64, 64), mode='bilinear').permute(0, 2, 3, 1)
    got = scr.join(xf)[..., 64:96]
    assert float((got - ref[:, None]).abs().max()) < 1e-6 and bool((scr.join(xf)[..., :64] == 0).all())
    # softmax + deformation
    K = 4
    logits = torch.randn(N, D, 64, 64, 8, generator=g).to(DEV)
    kp_s, kp_d = [(2 * torch.rand(N, K, 3, generator=g) - 1).to(DEV) for _ in range(2)]
    de = torch.empty(N, D, 64, 64, 3, device=DEV)
    capi.check(L.r3dp_mf_deform(capi.ptr(logits), 8, capi.ptr(kp_s), capi.ptr(kp_d), N, K, D, 64, 64, capi.ptr(de), st))
    grid = _grid(D, 64, 64, DEV)
    sm = torch.stack([grid.expand(N, -1, -1, -1, -1)] + [grid[None] - kp_d.double()[:, k, None, None, None] + kp_s.double()[:, k, None, None, None]
                                                        for k in range(K)], 1)
    mask = torch.softmax(logits[..., :K + 1].double(), -1).permute(0, 4, 1, 2, 3)[..., None]
    assert float((de.double() - (sm * mask).sum(1)).abs().max()) < 2e-6
    # occlusion pair over the c*16 + d view
    fx = torch.randn(N, D, 64, 64, 32, generator=g).to(DEV)
    f16 = _store(fx, True)
    c1, c2 = torch.nn.Conv2d(512, 1, 7, 1, 3).to(DEV).double(), torch.nn.Conv2d(512, 1, 7, 1, 3).to(DEV).double()
    wk = torch.stack([c.weight[0].reshape(32, D, 7, 7).permute(1, 2, 3, 0) for c in (c1, c2)], -1).reshape(D, 49, 32, 2).float().contiguous()
    bk = torch.cat([c1.bias, c2.bias]).float().contiguous()
    o1, o2 = torch.empty(N, 1, 64, 64, device=DEV), torch.empty(N, 1, 64, 64, device=DEV)
    capi.check(L.r3dp_mf_occlusion(capi.ptr(f16, F16), N, D, 64, 64, 32, 64, 32, 1, capi.ptr(wk), capi.ptr(bk), capi.ptr(o1), capi.ptr(o2), st))
    xv = scr.join(f16).permute(0, 4, 1, 2, 3).reshape(N, 512, 64, 64)
    with torch.no_grad():
        for o, c in ((o1, c1), (o2, c2)):
            assert float((o.double() - torch.sigmoid(c(xv))).abs().max()) < 1e-5


# ---- the whole estimator against the reference module -------------------------------------------------------------------------------------
def _ref_mfe(K=4):
    if not twr.ref_classes():
        pytest.skip('the reference warper modules are not staged under oracle/_ref (build() stages them where the reference exists)')
    from modules.real3d.facev2v_warp.network2 import MotionFieldEstimator
    torch.manual_seed(0)
    return twr.randomize(MotionFieldEstimator('standard', input_channels=34, num_keypoints=K), seed=51).to(DEV)


def _mfe_inputs(N, seed, K=4):
    g = torch.Generator().manual_seed(seed)
    motion_inp = torch.randn(1, 34, 16, 64, 64, generator=g).to(DEV).expand(N, -1, -1, -1, -1)
    kp_s, kp_d = [(0.8 * (2 * torch.rand(N, K, 3, generator=g) - 1)).to(DEV) for _ in range(2)]
    rgb = (2 * torch.rand(N, 3, 256, 256, generator=g) - 1).to(DEV)
    wt = torch.rand(N, 1, 256, 256, generator=g).to(DEV)
    return motion_inp, kp_s, kp_d, rgb, wt


@pytest.mark.parametrize('K', [4, 9])
@pytest.mark.parametrize('mode', ['tc', 'tc_exact'])
def test_estimator_against_reference(mode, K):
    """MotionFieldEstimator('standard', 34, K) of the reference against motion() for torso_kp_num 4 and 9 (K = 9: 50 input channels padded to
    64, a 128-channel fuser input, 10 mask logits).  Image k of an N = 2 launch equals the N = 1 launch, and a repeat gives the same bits."""
    mfe = _ref_mfe(K)
    N = 2
    motion_inp, kp_s, kp_d, rgb, wt = _mfe_inputs(N, 52, K)
    eye = torch.eye(3, device=DEV)[None].repeat(N, 1, 1)
    with torch.no_grad():
        ref = mfe(motion_inp.contiguous(), kp_s, kp_d, eye, eye, rgb, wt)
    wts = tw.MotionWeights(mfe, split=mode == 'tc_exact')
    fc = tw.compress_volume(wts, motion_inp[:1])
    out = tw.motion(wts, fc, kp_s, kp_d, rgb, wt)
    errs = [_rel(o, r) for o, r in zip(out, ref)]
    print(f'{mode} K={K}: max-abs / range of deformation, occlusion, occlusion_2: ' + ', '.join(f'{e:.2e}' for e in errs))
    assert max(errs) < (EXACT_REL if mode == 'tc_exact' else EST_TC_REL), errs
    again = tw.motion(wts, fc, kp_s, kp_d, rgb, wt)
    one = tw.motion(wts, fc, kp_s[1:], kp_d[1:], rgb[1:], wt[1:])
    for a, b, c in zip(out, again, one):
        assert torch.equal(a, b) and torch.equal(a[1:], c)


# ---- the torso head and the engine ---------------------------------------------------------------------------------------------------------
def _warper(seed=41):
    if not twr.ref_classes():
        pytest.skip('the reference warper modules are not staged under oracle/_ref')
    torch.manual_seed(seed)
    return twr.randomize(twr.ref_classes()[1]('standard'), seed=seed).to(DEV)


@pytest.mark.parametrize('mode', ['tc', 'tc_exact'])
def test_head_torso_motion_cuda_vs_torch(mode):
    warper = _warper()
    srp = syn.make_sr_warp_params(seed=6)
    srp.update({'torso_model.' + k: v for k, v in warper.state_dict().items()})
    heads = {}
    for mo in ('torch', 'cuda'):
        m = r3.SuperresolutionHybrid8XDC_Warp(channels=32, img_resolution=512, sr_num_fp16_res=0, sr_antialias=True, sr_mode=mode, hp=syn.WARP_HPARAMS,
                                              torso_model=_warper(), torso_stage2='cuda', torso_motion=mo)
        m.load_state_dict(srp, strict=True)
        heads[mo] = m.to(DEV).eval()
    N = 2
    g = torch.Generator().manual_seed(3)
    rgb, x = torch.randn(N, 3, 128, 128, generator=g).to(DEV), torch.randn(N, 32, 128, 128, generator=g).to(DEV)
    ws = torch.randn(N, 14, 512, generator=g).to(DEV)
    wimg = torch.rand(N, 1, 128, 128, generator=g).to(DEV)
    inp = {k: v.to(DEV) for k, v in syn.make_warp_inputs(1, seed=8).items()}
    args = (inp['ref_torso_rgb'].expand(N, -1, -1, -1), inp['ref_bg_rgb'].expand(N, -1, -1, -1), wimg, inp['segmap'].expand(N, -1, -1, -1),
            inp['kp_s'].expand(N, -1, -1), torch.rand(N, 68, 3, generator=g).to(DEV) * 2 - 1)
    with torch.no_grad():
        ref, ref_ret = heads['torch'](rgb, x, ws, *args)
        out, ret = heads['cuda'](rgb, x, ws, *args)
        e_img, e_occ = _rel(out, ref), _rel(ret['occlusion_2'], ref_ret['occlusion_2'])
        print(f'{mode}: head image max-abs / range {e_img:.2e}, occlusion_2 {e_occ:.2e}')
        bar = EXACT_REL if mode == 'tc_exact' else TC_REL
        assert e_img < bar and e_occ < bar, (e_img, e_occ)
        m = heads['cuda']
        m.begin_clip(inp['ref_torso_rgb'], inp['ref_bg_rgb'], segmap=inp['segmap'])
        assert 'fc' in m._clip_cache['torso_app']
        cached, _ = m(rgb, x, ws, *args)
        m.end_clip()
        e_c = _rel(cached, out)
        print(f'{mode}: cached vs uncached image max-abs / range {e_c:.2e}')
        assert e_c < EXACT_REL, e_c
        # a clip begun before torso_motion='cuda' was set: the compressed volume is added to its cache once, from the cached motion input
        m.set_torso_motion('torch')
        m.begin_clip(inp['ref_torso_rgb'], inp['ref_bg_rgb'], segmap=inp['segmap'])
        assert 'fc' not in m._clip_cache['torso_app']
        m.set_torso_motion('cuda')
        late, _ = m(rgb, x, ws, *args)
        assert 'fc' in m._clip_cache['torso_app'] and torch.equal(late, cached)
        m.end_clip()


def test_frame_engine_torso_motion_cuda():
    """A FrameEngine torso clip with torso_motion='cuda': graph and eager steps agree bit for bit, and an in-place clip refill (the
    compressed source volume included) changes what the graph renders."""
    from real3dportrait_b200 import engine
    warper = _warper()
    srp = syn.make_sr_warp_params(seed=6)
    srp.update({'torso_model.' + k: v for k, v in warper.state_dict().items()})
    mlp = syn.make_decoder_params(seed=4)
    inp, inp2 = syn.make_warp_inputs(1, seed=8), syn.make_warp_inputs(1, seed=9)
    outs = []
    for use_graph in (False, True):
        eng = engine.FrameEngine(batch=2, sr_mode='tc', hp=dict(syn.WARP_HPARAMS, num_samples_fine=0), torso_model=_warper(), use_graph=use_graph,
                                 torso_stage2='cuda', torso_motion='cuda')
        eng.load_params(mlp, srp)
        assert eng.head.superresolution.torso_motion == 'cuda'
        planes, cam = syn.make_planes(2, seed=0).to(DEV), syn.make_cameras(2, seed=1).to(DEV)
        kp_d = (torch.rand(2, 68, 3, generator=torch.Generator().manual_seed(2)) * 2 - 1).to(DEV)
        u_c, _ = syn.make_jitter(2, 4096, 48, 0, seed=3)
        frames = []
        for clip in (inp, inp2):
            eng.begin_clip(clip['ref_torso_rgb'].to(DEV), clip['ref_bg_rgb'].to(DEV), clip['segmap'].to(DEV), clip['kp_s'].to(DEV))
            assert 'fc' in eng.head.superresolution._clip_cache['torso_app']
            frames += [eng.step(planes, cam, u_c.to(DEV), kp_d=kp_d).clone() for _ in range(2)]
        assert torch.equal(frames[0], frames[1]) and torch.equal(frames[2], frames[3]) and not torch.equal(frames[0], frames[2])
        outs.append(frames)
        eng.end_clip()
    for a, b in zip(*outs):
        assert torch.equal(a, b)
