"""torso_stage2='cuda' on the GPU: the 3-D deformation gather, the 64-wide tensor-core conv with an output canary, the whole stage 2 (Generator +
occlusion_2_predictor) in 'tc' and 'tc_exact' against the reference's own modules run by PyTorch on the same device with TF32 off, batch and
repeat determinism, and the torso head end to end with the reference warper in both torso_stage2 modes, cached and uncached."""
import pytest
import torch
import torch.nn.functional as F

import real3dportrait_b200 as r3
from real3dportrait_b200 import _capi as capi, synthetic as syn, torso_warp as tw
import torso_warper_ref as twr

pytestmark = pytest.mark.gpu
DEV = 'cuda'
# Measured on an H100 80GB HBM3 (max-abs / range against the reference modules in fp32, TF32 off):
#   stage 2     tc: rgb_torso 7.6e-4, hid 1.1e-3, occlusion_2 8.4e-4    tc_exact: 3.2e-5, 4.6e-5, 3.5e-5
#   whole head  tc: image 1.9e-4, occlusion_2 1.6e-3                    tc_exact: 6.3e-6, 3.7e-5
EXACT_REL = 1e-3                  # the project's tc_exact bar: max-abs < 1e-3 * range
TC_REL = 5e-3                     # tc (fp16 operands, 16 conv layers deep): about 3x headroom over the largest measured value


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _ref_or_skip():
    cls = twr.ref_classes()
    if cls is None:
        pytest.skip('the reference warper modules are not staged under oracle/_ref (build() stages them where the reference exists)')
    return cls


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max()) / max(float(b.max() - b.min()), 1e-12)


@pytest.mark.parametrize('split', [0, 1])
def test_gather3d_matches_grid_sample(split):
    """r3dp_tw_gather3d = F.grid_sample(trilinear, border, align_corners=True).view(N, C*D, H, W), coordinates past [-1, 1] included."""
    fs, deformation, _ = twr.make_stage2_inputs(3, 64, seed=5)
    fs, deformation = fs.to(DEV), deformation.to(DEV)
    ref = F.grid_sample(fs, deformation, align_corners=True, padding_mode='border').reshape(3, 512, 64, 64).permute(0, 2, 3, 1)
    y = torch.empty(3, 64, 64, 512 * (2 if split else 1), device=DEV, dtype=torch.float16)
    capi.check(capi.lib().r3dp_tw_gather3d(capi.ptr(fs.permute(0, 2, 3, 4, 1).contiguous()), 0, capi.ptr(deformation), 3, 32, 16, 64, 64,
                                           capi.ptr(y, torch.float16), split, capi.stream()))
    got = y[..., :512].float() + (y[..., 512:].float() if split else 0)
    err = float((got - ref).abs().max())
    assert err < (1e-5 if split else 2e-3 * float(ref.abs().max())), err


@pytest.mark.parametrize('split', [0, 1])
def test_conv_64_wide_canary(split):
    """r3dp_tw_conv on a 64-wide map (half of each 128-pixel tile is TMA zero fill) against float64, inside a sentinel-filled allocation:
    every output element is written and nothing after it."""
    g = torch.Generator().manual_seed(9)
    N, H, W, I, O = 2, 64, 64, 256, 128
    x = torch.randn(N, I, H, W, generator=g).to(DEV)
    w = (torch.randn(O, I, 3, 3, generator=g) / 48).to(DEV)
    b = (0.1 * torch.randn(O, generator=g)).to(DEV)
    from real3dportrait_b200 import sr_tc
    wide = 2 if split else 1
    x16 = sr_tc.to_nhwc_f16(x, W, bool(split))
    wp = torch.empty(1, 9, O, I * wide, device=DEV, dtype=torch.float16)
    capi.check(sr_tc._fn('pack_weights', bool(split))(capi.ptr(w.contiguous()), 1, O, I, capi.ptr(wp, torch.float16), capi.stream()))
    n_out = N * H * W * O * wide
    buf = torch.full((n_out + 4096,), -7.0, device=DEV, dtype=torch.float16)
    y = buf[:n_out].view(N, H, W, O * wide)
    capi.check(capi.lib().r3dp_tw_conv(capi.ptr(x16, torch.float16), capi.ptr(wp, torch.float16), capi.ptr(b), N, I, O, H, W, 3, 0.2, None,
                                       capi.ptr(y, torch.float16), split, capi.stream()))
    torch.cuda.synchronize()
    assert bool((buf[n_out:] == -7.0).all()), 'written past the output'
    xin = x16[..., :I].double() + (x16[..., I:].double() if split else 0)
    ref = F.leaky_relu(F.conv2d(xin.permute(0, 3, 1, 2), w.double(), b.double(), padding=1), 0.2).permute(0, 2, 3, 1)
    got = y[..., :O].double() + (y[..., O:].double() if split else 0)
    assert bool(torch.isfinite(got).all()) and not bool((y == -7.0).any()), 'an output element was not written'
    assert _rel(got, ref) < (3e-5 if split else 2e-3)                # measured 1.2e-5 with split operands on an H100 80GB HBM3


def _stage2_modules(seed=31):
    gen = twr.randomize(_ref_or_skip()[0](), seed=seed).to(DEV)
    pred = twr.randomize(twr.make_predictor(), seed=seed + 1).to(DEV)
    return gen, pred


@pytest.mark.parametrize('mode', ['tc', 'tc_exact'])
def test_stage2_against_reference(mode):
    """Generator + occlusion_2_predictor on the kernels against the reference modules in fp32 (TF32 off): rgb_torso, deformed_torso_hid and
    occlusion_2.  Image k of an N=3 launch equals the N=1 launch, and a repeated launch gives the same bits."""
    gen, pred = _stage2_modules()
    wts = tw.Stage2Weights(gen, pred, split=mode == 'tc_exact')
    fs, deformation, occ = [t.to(DEV) for t in twr.make_stage2_inputs(3, 64, seed=32)]
    with torch.no_grad():
        ref = twr.reference_stage2(gen, pred, fs, deformation, occ)
    fsn = fs.permute(0, 2, 3, 4, 1).contiguous()
    rgb, hid16, occ2 = tw.stage2(wts, fsn, deformation, occ)
    hid = tw.hid_to_nchw(hid16, 64, wts.split)
    errs = [_rel(o, r) for o, r in zip((rgb, hid, occ2), ref)]
    print(f'{mode}: max-abs / range of rgb_torso, hid, occlusion_2: ' + ', '.join(f'{e:.2e}' for e in errs))
    bar = EXACT_REL if mode == 'tc_exact' else TC_REL
    assert max(errs) < bar, errs
    rgb_b, hid_b, occ_b = tw.stage2(wts, fsn, deformation, occ)
    assert torch.equal(rgb, rgb_b) and torch.equal(hid16, hid_b) and torch.equal(occ2, occ_b)
    rgb1, hid1, occ1 = tw.stage2(wts, fsn[1:2], deformation[1:2], occ[1:2])
    assert torch.equal(rgb1, rgb[1:2]) and torch.equal(hid1, hid16[1:2]) and torch.equal(occ1, occ2[1:2])


def _warper(seed=41):
    WarpModel = _ref_or_skip()[1]
    torch.manual_seed(seed)
    return twr.randomize(WarpModel('standard'), seed=seed).to(DEV)


@pytest.mark.parametrize('mode', ['tc', 'tc_exact'])
def test_head_torso_stage2_cuda_vs_torch(mode):
    """The torso head with the reference warper: torso_stage2='cuda' against the caller's PyTorch warper (TF32 off), and the per-clip appearance
    cache (begin_clip with the segmap) against the uncached path."""
    warper = _warper()
    srp = syn.make_sr_warp_params(seed=6)
    srp.update({'torso_model.' + k: v for k, v in warper.state_dict().items()})
    heads = {}
    for st2 in ('torch', 'cuda'):
        m = r3.SuperresolutionHybrid8XDC_Warp(channels=32, img_resolution=512, sr_num_fp16_res=0, sr_antialias=True, sr_mode=mode, hp=syn.WARP_HPARAMS,
                                              torso_model=_warper(), torso_stage2=st2)
        m.load_state_dict(srp, strict=True)
        heads[st2] = m.to(DEV).eval()
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
        assert set(ret) >= {'kp_src', 'kp_drv', 'occlusion', 'occlusion_2', 'deformed_torso_hid'}
        m = heads['cuda']
        m.begin_clip(inp['ref_torso_rgb'], inp['ref_bg_rgb'], segmap=inp['segmap'])
        cached, cret = m(rgb, x, ws, *args)
        m.end_clip()
        # the cache runs appearance_extractor on one image instead of the batch (PyTorch may pick other conv algorithms): equal to rounding
        e_c = _rel(cached, out)
        print(f'{mode}: cached vs uncached image max-abs / range {e_c:.2e}')
        assert e_c < EXACT_REL, e_c


def test_frame_engine_torso_stage2_cuda():
    """A FrameEngine torso clip with torso_stage2='cuda': graph and eager steps agree bit for bit and both run the new stage 2."""
    from real3dportrait_b200 import engine
    warper = _warper()
    srp = syn.make_sr_warp_params(seed=6)
    srp.update({'torso_model.' + k: v for k, v in warper.state_dict().items()})
    mlp = syn.make_decoder_params(seed=4)
    inp = syn.make_warp_inputs(1, seed=8)
    outs = []
    for use_graph in (False, True):
        eng = engine.FrameEngine(batch=2, sr_mode='tc', hp=dict(syn.WARP_HPARAMS, num_samples_fine=0), torso_model=_warper(), use_graph=use_graph,
                                 torso_stage2='cuda')
        eng.load_params(mlp, srp)
        assert eng.head.superresolution.torso_stage2 == 'cuda'
        eng.begin_clip(inp['ref_torso_rgb'].to(DEV), inp['ref_bg_rgb'].to(DEV), inp['segmap'].to(DEV), inp['kp_s'].to(DEV))
        assert eng.head.superresolution._clip_cache['torso_app'] is not None
        planes, cam = syn.make_planes(2, seed=0).to(DEV), syn.make_cameras(2, seed=1).to(DEV)
        kp_d = (torch.rand(2, 68, 3, generator=torch.Generator().manual_seed(2)) * 2 - 1).to(DEV)
        u_c, _ = syn.make_jitter(2, 4096, 48, 0, seed=3)
        frames = [eng.step(planes, cam, u_c.to(DEV), kp_d=kp_d).clone() for _ in range(2)]
        assert torch.equal(frames[0], frames[1])
        outs.append(frames[0])
        eng.end_clip()
    assert torch.equal(outs[0], outs[1])


def _cuda_head(mode='tc'):
    warper = _warper()
    srp = syn.make_sr_warp_params(seed=6)
    srp.update({'torso_model.' + k: v for k, v in warper.state_dict().items()})
    m = r3.SuperresolutionHybrid8XDC_Warp(channels=32, img_resolution=512, sr_num_fp16_res=0, sr_antialias=True, sr_mode=mode, hp=syn.WARP_HPARAMS,
                                          torso_model=_warper(), torso_stage2='cuda')
    m.load_state_dict(srp, strict=True)
    return m.to(DEV).eval()


def _head_args(N, seed):
    g = torch.Generator().manual_seed(seed)
    inp = {k: v.to(DEV) for k, v in syn.make_warp_inputs(1, seed=seed + 1).items()}
    base = (torch.randn(N, 3, 128, 128, generator=g).to(DEV), torch.randn(N, 32, 128, 128, generator=g).to(DEV), torch.randn(N, 14, 512, generator=g).to(DEV))
    rest = (inp['ref_torso_rgb'].expand(N, -1, -1, -1), inp['ref_bg_rgb'].expand(N, -1, -1, -1), torch.rand(N, 1, 128, 128, generator=g).to(DEV),
            inp['segmap'].expand(N, -1, -1, -1), inp['kp_s'].expand(N, -1, -1), torch.rand(N, 68, 3, generator=g).to(DEV) * 2 - 1)
    return inp, base + rest


@pytest.mark.parametrize('mode', ['tc', 'tc_exact'])
def test_cached_equals_uncached_bitwise(mode):
    """With one image the cached appearance features are computed exactly as the uncached call computes them: the two paths agree bit for bit."""
    m = _cuda_head(mode)
    inp, args = _head_args(1, 30)
    with torch.no_grad():
        out, ret = m(*args)
        m.begin_clip(inp['ref_torso_rgb'], inp['ref_bg_rgb'], segmap=inp['segmap'])
        cached, cret = m(*args)
        m.end_clip()
    assert torch.equal(cached, out) and torch.equal(cret['occlusion_2'], ret['occlusion_2'])


def test_begin_clip_in_place_refills_the_appearance_cache():
    """A second in-place begin_clip writes the new clip's appearance features into the SAME tensors (graphs that captured the warper read them
    by address), and those equal a fresh begin_clip of the second clip."""
    m = _cuda_head()
    c1, _ = _head_args(1, 40)
    c2, _ = _head_args(1, 50)
    with torch.no_grad():
        assert not m.begin_clip(c1['ref_torso_rgb'], c1['ref_bg_rgb'], batch=2, in_place=True, segmap=c1['segmap'])
        app = m._clip_cache['torso_app']
        ptrs = {k: v.data_ptr() for k, v in app.items()}
        assert m.begin_clip(c2['ref_torso_rgb'], c2['ref_bg_rgb'], batch=2, in_place=True, segmap=c2['segmap'])
        assert m._clip_cache['torso_app'] is app and {k: v.data_ptr() for k, v in app.items()} == ptrs
        refilled = {k: v.clone() for k, v in app.items()}
        m.end_clip()
        m.begin_clip(c2['ref_torso_rgb'], c2['ref_bg_rgb'], batch=2, segmap=c2['segmap'])
        fresh = m._clip_cache['torso_app']
    for k in refilled:
        assert torch.equal(refilled[k], fresh[k]), k


def test_stage2_weights_follow_parameter_changes():
    """The folded weights are rebuilt after the warper's parameters change in place (a load_state_dict of torso_model alone)."""
    m = _cuda_head()
    w0 = m._stage2_weights()
    assert m._stage2_weights() is w0
    with torch.no_grad():
        m.torso_model.deform_based_generator.out_conv.bias.add_(1.0)
    w1 = m._stage2_weights()
    assert w1 is not w0 and torch.equal(w1.out_conv[1], w0.out_conv[1] + 1.0)
