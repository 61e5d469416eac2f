"""sr_mode='tc_exact' (split fp16 operands, fp32-grade results) in the torso head (SuperresolutionHybrid8XDC_Warp) and in large_sr.

Whole-head tests compare against the reference fixtures / the CPU oracle and print the 'tc' error on the same inputs beside the 'tc_exact' one.
Bars: max-abs < 1e-3 * range (the project's tc_exact bar) and < 2e-4 absolute (the regression guard of the plain head's tc_exact test).
Unit tests run each split entry point at small shapes against fp64 torch computed from the reconstructed hi + lo operands."""
import pytest
import torch
import torch.nn.functional as F

import real3dportrait_b200 as r3
from real3dportrait_b200 import _capi as capi, sr_tc, synthetic as syn
from launch_harness import check_split_layout, split_cat
from oracle import real3d_oracle as orc

pytestmark = pytest.mark.gpu
DEV = 'cuda'
EXACT_REL, EXACT_ABS = 1e-3, 2e-4


def _maxdiff(a, b):
    return float((a.detach().float().cpu() - b.detach().float().cpu()).abs().max())


def _join(t: torch.Tensor) -> torch.Tensor:
    """[hi | lo] fp16 [..., 2C] -> fp64 [..., C]."""
    C_ = t.shape[-1] // 2
    return t[..., :C_].double() + t[..., C_:].double()


def _exact_bars(tag, err, rng, err_tc, guard=EXACT_ABS):
    print(f'{tag}: tc_exact max-abs {err:.3e} (tc {err_tc:.3e}) on range {rng:.2f}')
    assert err < EXACT_REL * rng, (err, rng)
    assert err < guard, err


# ---- whole heads -------------------------------------------------------------------------------------------------------------------
def _warp_fixture_run(golden, fuse, mode):
    g = golden('render_full48')
    fx = golden({'v2': 'sr_warp_full', 'v1': 'sr_warp_v1', 'v3': 'sr_warp_v3'}[fuse])
    fimg = orc.feature_image(g['rgb'], 64).to(DEV)
    wimg = fx['weights_img'].to(DEV) if 'weights_img' in fx else orc.feature_image(g['wsum'], 64).to(DEV)
    inp = {k: v.to(DEV) for k, v in syn.make_warp_inputs(1, seed=7).items()}
    m = r3.SuperresolutionHybrid8XDC_Warp(channels=32, img_resolution=512, sr_num_fp16_res=0, sr_antialias=True, sr_mode=mode,
                                          hp=dict(syn.WARP_HPARAMS, htbsr_head_weight_fuse_mode=fuse), torso_model=syn.StubTorsoModel())
    m.load_state_dict(syn.make_sr_warp_params(seed=6, fuse_mode=fuse), strict=True)
    m = m.to(DEV).eval()
    with torch.no_grad():
        img, _ = m(fimg[:, :3].contiguous(), fimg, torch.ones(1, 14, 512, device=DEV), inp['ref_torso_rgb'], inp['ref_bg_rgb'], wimg, inp['segmap'],
                   inp['kp_s'], inp['kp_d'], noise_mode='none')
    return img[..., ::2, ::2], fx['image_s2']


@pytest.mark.parametrize('fuse', ['v2', 'v1', 'v3'])
def test_torso_head_tc_exact_vs_reference(golden, fuse):
    """Torso head in tc_exact against the reference class's fp32 image (fixtures sr_warp_full / sr_warp_v1 / sr_warp_v3, stub torso child)."""
    img, ref = _warp_fixture_run(golden, fuse, 'tc_exact')
    img_tc, _ = _warp_fixture_run(golden, fuse, 'tc')
    _exact_bars(f'torso head fuse mode {fuse}', _maxdiff(img, ref), float(ref.max() - ref.min()), _maxdiff(img_tc, ref))


def test_torso_head_tc_exact_two_frames_per_sample_styles_and_clip_cache():
    """N=2 with different styles per frame against the oracle; the per-clip cached path (x_bg stored split) equals the uncached one, bit for bit."""
    N = 2
    g = torch.Generator().manual_seed(70)
    fimg = (torch.rand(N, 32, 64, 64, generator=g) * 2 - 1)
    wimg = torch.rand(N, 1, 64, 64, generator=g)
    ws = 1 + 0.2 * torch.randn(N, 14, 512, generator=g)
    inp = syn.make_warp_inputs(1, seed=71)
    inp = {k: v.expand(N, *v.shape[1:]).contiguous() for k, v in inp.items()}
    inp['kp_d'] = torch.rand(N, 68, 3, generator=g) * 2 - 1
    srp = syn.make_sr_warp_params(seed=6)
    ref, _ = orc.superres_warp(fimg[:, :3], fimg, ws, inp['ref_torso_rgb'], inp['ref_bg_rgb'], wimg, inp['segmap'], inp['kp_s'], inp['kp_d'], srp,
                               syn.StubTorsoModel())
    dv = {k: v.to(DEV) for k, v in inp.items()}
    args = (fimg[:, :3].contiguous().to(DEV), fimg.to(DEV), ws.to(DEV), dv['ref_torso_rgb'], dv['ref_bg_rgb'], wimg.to(DEV), dv['segmap'], dv['kp_s'], dv['kp_d'])
    outs = {}
    for mode in ('tc', 'tc_exact'):
        m = r3.SuperresolutionHybrid8XDC_Warp(channels=32, img_resolution=512, sr_num_fp16_res=0, sr_antialias=True, hp=syn.WARP_HPARAMS, sr_mode=mode,
                                              torso_model=syn.StubTorsoModel())
        m.load_state_dict(srp, strict=True)
        m = m.to(DEV).eval()
        with torch.no_grad():
            outs[mode], _ = m(*args, noise_mode='none')
    _exact_bars('torso head N=2, per-sample styles', _maxdiff(outs['tc_exact'], ref), float(ref.max() - ref.min()), _maxdiff(outs['tc'], ref))
    with torch.no_grad():
        m.begin_clip(dv['ref_torso_rgb'][:1], dv['ref_bg_rgb'][:1])
        assert m._clip_cache['x_bg'].shape == (1, 256, 256, 512)
        img_c, _ = m(*args, noise_mode='none')
        img_c2, _ = m(*args, noise_mode='none')
        m.end_clip()
    assert torch.equal(img_c, outs['tc_exact']) and torch.equal(img_c2, outs['tc_exact'])


def test_large_sr_tc_exact_vs_reference(golden):
    """large_sr=True in tc_exact (split residual epilogue, split ToRGB) against the reference class's fp32 image."""
    fimg = orc.feature_image(golden('render_full48')['rgb'], 64).to(DEV)
    ref = golden('sr_large')['image_s2']
    imgs = {}
    for mode in ('tc', 'tc_exact'):
        sr = r3.SuperresolutionHybrid8XDC(channels=32, img_resolution=512, sr_num_fp16_res=0, sr_antialias=True, large_sr=True, sr_mode=mode,
                                          resblocks_in_large_sr=2)
        sr.load_state_dict(syn.make_sr_large_params(seed=8, n_res=2), strict=True)
        imgs[mode] = sr.to(DEV)(fimg[:, :3], fimg, torch.ones(1, 14, 512, device=DEV), noise_mode='none')[..., ::2, ::2]
    # Guard 6e-4 instead of 2e-4: the image spans 15.6 (1.4 for the torso head), and the four ResBlock2d convolutions of each block carry it.  Against
    # an fp64 oracle their outputs measure 2.4e-5 (block0.resblocks.0.conv1) to 4.9e-5 (block1.resblocks.1.conv2 + x) of their largest value, which grows
    # to 9.5; the image error, 3.8e-4, is 2.4e-5 of its range, the same relative size as the torso head's.  No single layer stands out.
    _exact_bars('large_sr', _maxdiff(imgs['tc_exact'], ref), float(ref.max() - ref.min()), _maxdiff(imgs['tc'], ref), guard=6e-4)
    with pytest.raises(NotImplementedError):
        sr(fimg[:, :3], fimg, torch.ones(1, 14, 512, device=DEV), noise_mode='none', out_uint8=True)


def test_torso_render_head_config5_tc_exact_vs_oracle():
    """Config 5 for one frame (48 + 48 samples -> torso SR head) with RenderHead(sr_mode='tc_exact') against the oracle."""
    N = 1
    planes, cam = syn.make_planes(N, seed=40), syn.make_cameras(N, seed=41)
    u_c, u_f = syn.make_jitter(N, 4096, 48, 48, seed=42)
    mlp, srp = syn.make_decoder_params(seed=4), syn.make_sr_warp_params(seed=6)
    inp = syn.make_warp_inputs(N, seed=43)
    c2w, K = syn.split_camera(cam)
    o, d = orc.gen_rays(c2w, K, 64)
    feat, depth, wsum, _ = orc.render(planes, mlp, o, d, S=48, S_imp=48, u_coarse=u_c, u_fine=u_f, lib=True)
    fimg, wimg = orc.feature_image(feat, 64), orc.feature_image(wsum, 64)
    ref, _ = orc.superres_warp(fimg[:, :3], fimg, torch.ones(N, 14, 512), inp['ref_torso_rgb'], inp['ref_bg_rgb'], wimg, inp['segmap'], inp['kp_s'],
                               inp['kp_d'], srp, syn.StubTorsoModel())
    ref = ref.clamp(-1, 1)
    cond = {'ref_torso_img': inp['ref_torso_rgb'].to(DEV), 'bg_img': inp['ref_bg_rgb'].to(DEV), 'segmap': inp['segmap'].to(DEV),
            'kp_s': inp['kp_s'].to(DEV), 'kp_d': inp['kp_d'].to(DEV)}
    errs = {}
    for mode in ('tc', 'tc_exact'):
        head = r3.RenderHead(hp=dict(syn.WARP_HPARAMS, num_samples_fine=48), torso_model=syn.StubTorsoModel(), sr_mode=mode)
        assert head.superresolution.sr_mode == mode
        sd = {'decoder.' + k: v for k, v in mlp.items()}
        sd.update({'superresolution.' + k: v for k, v in srp.items()})
        head.load_state_dict(sd, strict=True)
        head = head.to(DEV).eval()
        out = head.synthesis(planes.to(DEV), cam.to(DEV), cond=cond, u_coarse=u_c.to(DEV), u_fine=u_f.to(DEV))
        errs[mode] = _maxdiff(out['image'], ref)
    _exact_bars('config-5 render head', errs['tc_exact'], float(ref.max() - ref.min()), errs['tc'])


# ---- the split entry points at small shapes ---------------------------------------------------------------------------------------------
def _rand(*shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def _unpack_plain(wp, O, I):
    """packed split weights [1,9,O,2*Ip] (x 2^10) -> fp64 [O,I,3,3] of the reconstructed hi + lo values."""
    w = _join(wp.cpu())[0, :, :, :I] / 1024.0                    # [9,O,I]
    return w.permute(1, 2, 0).reshape(O, I, 3, 3)


def test_tcx_conv_res_relu_residual():
    N, H, W, I, O = 2, 5, 128, 64, 128
    conv = torch.nn.Conv2d(I, O, 3, padding=1)
    torch.nn.init.uniform_(conv.bias, -0.5, 0.5)
    conv = conv.to(DEV)
    packed = sr_tc.pack_plain(conv, I, split=True)
    xs = split_cat(_rand(N, H, W, I, seed=1)).to(DEV)
    res = split_cat(_rand(N, H, W, O, seed=2)).to(DEV)
    y = sr_tc.conv_plain(xs, packed, 3, residual=res, split=True)
    torch.cuda.synchronize()
    assert y.shape == (N, H, W, 2 * O)
    w = _unpack_plain(packed[0], O, I)
    ref = torch.relu(F.conv2d(_join(xs.cpu()).permute(0, 3, 1, 2), w, packed[1].cpu().double()[:O], padding=1)).permute(0, 2, 3, 1) + _join(res.cpu())
    err = _maxdiff(_join(y.cpu()), ref)
    print(f'tcx_conv_res: max-abs {err:.3e} on max |ref| {float(ref.abs().max()):.2f}')
    assert err < 2e-5 * float(ref.abs().max()), err
    check_split_layout(y.cpu())


@pytest.mark.parametrize('shared', [False, True])
def test_tcx_alpha_cat_ex(shared):
    N, H, W, Ca, Cb = 2, 3, 5, 64, 128
    xa = split_cat(_rand(N, H, W, Ca, seed=3)).to(DEV)
    xb = split_cat(_rand(1 if shared else N, H, W, Cb, seed=4)).to(DEV)
    al = torch.rand(N, H, W, generator=torch.Generator().manual_seed(5)).to(DEV)
    out = torch.empty(N, H, W, 2 * (Ca + Cb), device=DEV, dtype=torch.float16)
    capi.check(capi.lib().r3dp_sr_tcx_alpha_cat_ex(capi.ptr(xa, torch.float16), Ca, 2 * Ca, capi.ptr(xb, torch.float16), Cb, 2 * Cb, int(shared),
                                                    capi.ptr(al), N, H, W, capi.ptr(out, torch.float16), capi.stream()))
    torch.cuda.synchronize()
    a = al.cpu().double()[..., None]
    ref = torch.cat([_join(xa.cpu()) * a, _join(xb.cpu()).expand(N, -1, -1, -1) * (1 - a)], dim=-1)
    err = _maxdiff(_join(out.cpu()), ref)
    assert err < 1e-6 * float(ref.abs().max()), err
    check_split_layout(out.cpu())


def test_tcx_alpha_mix():
    N, H, W, Cc = 2, 3, 5, 64
    xa, xb = split_cat(_rand(N, H, W, Cc, seed=6)).to(DEV), split_cat(_rand(N, H, W, Cc, seed=7)).to(DEV)
    al = torch.rand(N, H, W, generator=torch.Generator().manual_seed(8)).to(DEV)
    out = torch.empty(N, H, W, 2 * Cc, device=DEV, dtype=torch.float16)
    capi.check(capi.lib().r3dp_sr_tcx_alpha_mix(capi.ptr(xa, torch.float16), 2 * Cc, capi.ptr(xb, torch.float16), 2 * Cc, capi.ptr(al), Cc, N, H, W,
                                                 capi.ptr(out, torch.float16), capi.stream()))
    torch.cuda.synchronize()
    a = al.cpu().double()[..., None]
    ref = _join(xa.cpu()) * a + _join(xb.cpu()) * (1 - a)
    err = _maxdiff(_join(out.cpu()), ref)
    assert err < 1e-6 * float(ref.abs().max()), err
    check_split_layout(out.cpu())


@pytest.mark.parametrize('same_res', [0, 1])
def test_tcx_torgb_ex(same_res):
    N, H, W, Cc = 2, 8, 12, 64
    xs = split_cat(_rand(N, H, W, Cc, seed=9)).to(DEV)
    wrgb, brgb = (0.1 * _rand(N, 3, Cc, seed=10)).to(DEV), _rand(3, seed=11).to(DEV)
    img_prev = _rand(N, 3, H, W, seed=12) if same_res else _rand(N, 3, H // 2, W // 2, seed=12)
    out = torch.empty(N, 3, H, W, device=DEV)
    capi.check(capi.lib().r3dp_sr_tcx_torgb_ex(capi.ptr(xs, torch.float16), capi.ptr(wrgb), capi.ptr(brgb), capi.ptr(img_prev.to(DEV)), same_res, N, N,
                                                Cc, H, W, capi.ptr(out), capi.stream()))
    torch.cuda.synchronize()
    skip = img_prev.double() if same_res else orc.upsample2x(img_prev.double())
    ref = torch.einsum('nhwc,nkc->nkhw', _join(xs.cpu()), wrgb.cpu().double()) + brgb.cpu().double().view(1, 3, 1, 1) + skip
    err = _maxdiff(out, ref)
    assert err < 1e-5 * float(ref.abs().max()), err


def test_tcx_layer_torgb_noup():
    N, H, W, I, O = 2, 4, 128, 64, 128
    xs = split_cat(_rand(N, H, W, I, seed=13)).to(DEV)
    wf = (_rand(1, O, I, 3, 3, seed=14) / 24.0).to(DEV)
    wp = torch.empty(1, 9, O, 2 * I, device=DEV, dtype=torch.float16)
    L = capi.lib()
    capi.check(L.r3dp_sr_tcx_pack_weights(capi.ptr(wf), 1, O, I, capi.ptr(wp, torch.float16), capi.stream()))
    bias, wrgb, brgb = (0.1 * _rand(O, seed=15)).to(DEV), (0.1 * _rand(1, 3, O, seed=16)).to(DEV), _rand(3, seed=17).to(DEV)
    img_prev = _rand(N, 3, H, W, seed=18).to(DEV)
    y = torch.empty(N, H, W, 2 * O, device=DEV, dtype=torch.float16)
    img = torch.empty(N, 3, H, W, device=DEV)
    capi.check(L.r3dp_sr_tcx_layer_torgb_noup(capi.ptr(xs, torch.float16), capi.ptr(wp, torch.float16), capi.ptr(bias), capi.ptr(wrgb), capi.ptr(brgb),
                                               capi.ptr(img_prev), N, 1, I, O, H, W, capi.ptr(y, torch.float16), capi.ptr(img), capi.stream()))
    torch.cuda.synchronize()
    w = _unpack_plain(wp, O, I)
    v = F.conv2d(_join(xs.cpu()).permute(0, 3, 1, 2), w, bias.cpu().double(), padding=1)
    v = F.leaky_relu(v, 0.2) * 2 ** 0.5                                    # [N,O,H,W]
    ref_img = img_prev.cpu().double() + torch.einsum('nohw,ko->nkhw', v, wrgb.cpu().double()[0]) + brgb.cpu().double().view(1, 3, 1, 1)
    err_y, err_img = _maxdiff(_join(y.cpu()), v.permute(0, 2, 3, 1)), _maxdiff(img, ref_img)
    print(f'tcx_layer_torgb_noup: y max-abs {err_y:.3e}, image max-abs {err_img:.3e}')
    assert err_y < 2e-5 * float(v.abs().max()) and err_img < 2e-5 * float(ref_img.abs().max()), (err_y, err_img)
    check_split_layout(y.cpu())
