"""The torso head's other reference configurations on the GPU: weight_fuse=False (cat[x, x_torso, x_bg] -> fuse_fg_bg_convs(768 -> 64) -> block1
without a skip image, sr_with_ref.py:158-161) and torso_model_version 'v1' (the warper takes no head weights image, sr_with_ref.py:84-85).
The three-way concat and the skip-less last layer as units, the head against the reference fixture and the oracle in 'tc' and 'tc_exact', the
per-clip cache, and FrameEngine's eager / split-graph / whole-graph / prepared steps."""
import pytest
import torch

import real3dportrait_b200 as r3
from real3dportrait_b200 import _capi as capi, engine, synthetic as syn
import torso_config_oracle as tco
from oracle import real3d_oracle as orc

pytestmark = pytest.mark.gpu
DEV = 'cuda'
TC_MAXABS, TC_PSNR = 5e-3, 70.0          # the tensor-core SR's stated tolerance against fp32 (tests/test_gpu_parity.py)
EXACT_REL = 1e-3                         # the project's tc_exact bar: max-abs < 1e-3 * range
NOFUSE_EXACT_GUARD = 1e-4                # regression guard of tc_exact against sr_warp_nofuse (measured 3.8e-5 on an H100 80GB HBM3)
NOFUSE = dict(syn.WARP_HPARAMS, weight_fuse=False)
V1 = dict(syn.WARP_HPARAMS, torso_model_version='v1')


def _maxdiff(a, b):
    return float((a.detach().float().cpu() - b.detach().float().cpu()).abs().max())


def _psnr(img, ref):
    mse = float(((img.detach().float().cpu() - ref) ** 2).mean())
    return 10 * torch.log10(torch.tensor(float(ref.max() - ref.min()) ** 2 / max(mse, 1e-30))).item()


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.float16 else t


class _V1AsV2(torch.nn.Module):
    """A v2 warper whose outputs are those of a v1 warper: it drops the head weights image."""

    def __init__(self, v1):
        super().__init__()
        self.v1 = v1

    def forward(self, torso_src_img, segmap, kp_s, kp_d, tgt_head_img, tgt_head_weights, cal_loss=False, target_torso_mask=None):
        return self.v1(torso_src_img, segmap, kp_s, kp_d, tgt_head_img, cal_loss=cal_loss, target_torso_mask=target_torso_mask)


def _head(hp, mode, warper, params):
    m = r3.SuperresolutionHybrid8XDC_Warp(channels=32, img_resolution=512, sr_num_fp16_res=0, sr_antialias=True, sr_mode=mode, hp=hp, torso_model=warper)
    m.load_state_dict(params, strict=True)
    return m.to(DEV).eval()


# ---- 1. the kernels --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('shared', [False, True])
@pytest.mark.parametrize('split', [0, 1])
def test_cat3_is_torch_cat(shared, split):
    """cat[xa, xb, xc] equals torch.cat of the fp16 tensors bit for bit; split: the [hi | lo] layout of the result (each operand's halves
    copied unchanged); shared: xc is one frame read by every frame of the batch.  xa has a pixel stride wider than its channels (each half padded)."""
    N, H, W, C, P = 3, 7, 9, 256, 64
    wide = 2 if split else 1
    g = torch.Generator().manual_seed(11 + split + 2 * shared)
    xa_pad = torch.randn(N, H, W, (C + P) * wide, generator=g).half().to(DEV)
    xa_halves = [xa_pad[..., h * (C + P):h * (C + P) + C] for h in range(wide)]
    xb = torch.randn(N, H, W, C * wide, generator=g).half().to(DEV)
    xc = torch.randn(1 if shared else N, H, W, C * wide, generator=g).half().to(DEV)
    out = torch.full((N, H, W, 3 * C * wide), 7.0, device=DEV, dtype=torch.float16)
    fn = capi.lib().r3dp_sr_tcx_cat3 if split else capi.lib().r3dp_sr_cat3
    capi.check(fn(capi.ptr(xa_pad, torch.float16), C, xa_pad.shape[-1], capi.ptr(xb, torch.float16), C, C * wide, capi.ptr(xc, torch.float16), C, C * wide,
                  int(shared), N, H, W, capi.ptr(out, torch.float16), capi.stream()))
    torch.cuda.synchronize()
    xc_n = xc.expand(N, -1, -1, -1)
    want = torch.cat([t for h in range(wide) for t in (xa_halves[h], xb[..., h * C:(h + 1) * C], xc_n[..., h * C:(h + 1) * C])], dim=-1)
    assert torch.equal(_bits(out), _bits(want))


@pytest.mark.parametrize('split', [0, 1])
def test_last_layer_without_skip_equals_zero_skip(split):
    """img_prev == NULL: the image is ToRGB + bias alone; it equals the image with an all-zero img_prev (compared with ==: adding +0.0 turns a
    -0.0 into +0.0), in fp32 and as uint8 frames."""
    N, H, W, I = 2, 4, 128, 64
    wide = 2 if split else 1
    g = torch.Generator().manual_seed(20 + split)
    L = capi.lib()
    x = torch.randn(N, H, W, I, generator=g)
    x16 = (torch.cat([x.half(), (x - x.half().float()).half()], -1) if split else x.half()).contiguous().to(DEV)
    wf = (torch.randn(1, 128, I, 3, 3, generator=g) / 24.0).to(DEV)
    wp = torch.empty(1, 9, 128, I * wide, device=DEV, dtype=torch.float16)
    capi.check((L.r3dp_sr_tcx_pack_weights if split else L.r3dp_sr_tc_pack_weights)(capi.ptr(wf), 1, 128, I, capi.ptr(wp, torch.float16), capi.stream()))
    bias, wrgb, brgb = (0.1 * torch.randn(128, generator=g)).to(DEV), (0.1 * torch.randn(1, 3, 128, generator=g)).to(DEV), (0.1 * torch.randn(3, generator=g)).to(DEV)
    zeros = torch.zeros(N, 3, H // 2, W // 2, device=DEV)
    fn = L.r3dp_sr_tcx_last_layer if split else L.r3dp_sr_tc_last_layer_ex
    outs = {}
    for skip in (None, zeros):
        img = torch.full((N, 3, H, W), 7.0, device=DEV)
        u8 = torch.full((N, H, W, 3), 7, device=DEV, dtype=torch.uint8)
        for o, o8, clamp in ((img, None, 0), (None, u8, 1)):
            capi.check(fn(capi.ptr(x16, torch.float16), capi.ptr(wp, torch.float16), capi.ptr(bias), capi.ptr(wrgb), capi.ptr(brgb), capi.ptr(skip), N, 1, I, H, W,
                          capi.ptr(o), capi.ptr(o8, torch.uint8), clamp, capi.stream()))
        outs[skip is None] = (img, u8)
    torch.cuda.synchronize()
    (img_n, u8_n), (img_z, u8_z) = outs[True], outs[False]
    assert bool((img_n == img_z).all()) and torch.equal(u8_n, u8_z)
    assert float(img_n.abs().max()) > 0.1                                  # not trivially zero


# ---- 2. the head against the reference and the oracle ----------------------------------------------------------------------------------
def _fixture_run(golden, mode):
    g = golden('render_full48')
    fimg, wimg = orc.feature_image(g['rgb'], 64).to(DEV), orc.feature_image(g['wsum'], 64).to(DEV)
    inp = {k: v.to(DEV) for k, v in syn.make_warp_inputs(1, seed=7).items()}
    m = _head(NOFUSE, mode, syn.StubTorsoModel(), syn.make_sr_warp_params(seed=6, weight_fuse=False))
    with torch.no_grad():
        img, ret = m(fimg[:, :3].contiguous(), fimg, torch.ones(1, 14, 512, device=DEV), inp['ref_torso_rgb'], inp['ref_bg_rgb'], wimg, inp['segmap'],
                     inp['kp_s'], inp['kp_d'], noise_mode='none')
    assert set(ret) >= {'deformed_torso_hid', 'occlusion_2'}                  # facev2v_ret is still returned
    return img[..., ::2, ::2], golden('sr_warp_nofuse')['image_s2']


def test_weight_fuse_false_vs_reference(golden):
    img_tc, ref = _fixture_run(golden, 'tc')
    img_x, _ = _fixture_run(golden, 'tc_exact')
    rng = float(ref.max() - ref.min())
    err_tc, psnr, err_x = _maxdiff(img_tc, ref), _psnr(img_tc, ref), _maxdiff(img_x, ref)
    print(f'weight_fuse=False vs reference: tc max-abs {err_tc:.3e} (PSNR {psnr:.1f} dB), tc_exact max-abs {err_x:.3e}, range {rng:.2f}')
    assert err_tc < TC_MAXABS and psnr > TC_PSNR, (err_tc, psnr)
    assert err_x < EXACT_REL * rng and err_x < NOFUSE_EXACT_GUARD, (err_x, rng)


@pytest.mark.parametrize('mode', ['tc', 'tc_exact'])
def test_weight_fuse_false_two_frames_per_sample_styles_and_clip_cache(mode):
    """N=2 with a different style per frame against the oracle; the per-clip cached path (x_bg read as one shared frame) equals the uncached one
    bit for bit."""
    N = 2
    g = torch.Generator().manual_seed(70)
    fimg, wimg = torch.rand(N, 32, 64, 64, generator=g) * 2 - 1, torch.rand(N, 1, 64, 64, generator=g)
    ws = 1 + 0.2 * torch.randn(N, 14, 512, generator=g)
    inp = {k: v.expand(N, *v.shape[1:]).contiguous() for k, v in syn.make_warp_inputs(1, seed=71).items()}
    inp['kp_d'] = torch.rand(N, 68, 3, generator=g) * 2 - 1
    srp = syn.make_sr_warp_params(seed=6, weight_fuse=False)
    ref, _ = tco.superres_warp(fimg[:, :3], fimg, ws, inp['ref_torso_rgb'], inp['ref_bg_rgb'], wimg, inp['segmap'], inp['kp_s'], inp['kp_d'], srp,
                               syn.StubTorsoModel(), weight_fuse=False)
    dv = {k: v.to(DEV) for k, v in inp.items()}
    args = (fimg[:, :3].contiguous().to(DEV), fimg.to(DEV), ws.to(DEV), dv['ref_torso_rgb'], dv['ref_bg_rgb'], wimg.to(DEV), dv['segmap'], dv['kp_s'], dv['kp_d'])
    m = _head(NOFUSE, mode, syn.StubTorsoModel(), srp)
    with torch.no_grad():
        img, _ = m(*args, noise_mode='none')
        m.begin_clip(dv['ref_torso_rgb'][:1], dv['ref_bg_rgb'][:1])
        img_c, _ = m(*args, noise_mode='none')
        img_c2, _ = m(*args, noise_mode='none')
        m.end_clip()
    rng = float(ref.max() - ref.min())
    err = _maxdiff(img, ref)
    print(f'weight_fuse=False N=2 per-sample styles, {mode}: max-abs {err:.3e} on range {rng:.2f}')
    if mode == 'tc':
        assert err < TC_MAXABS and _psnr(img, ref) > TC_PSNR, err
    else:
        assert err < EXACT_REL * rng, (err, rng)
    assert torch.equal(img_c, img) and torch.equal(img_c2, img)


@pytest.mark.parametrize('weight_fuse', [True, False])
@pytest.mark.parametrize('mode', ['tc', 'tc_exact'])
def test_torso_v1_equals_v2_on_the_same_warper_outputs(mode, weight_fuse):
    """torso_model_version 'v1' calls the warper with model.py's argument list and changes nothing else: on the same warper outputs its image is
    the v2 head's, bit for bit."""
    g = torch.Generator().manual_seed(80)
    fimg, wimg = torch.rand(1, 32, 64, 64, generator=g) * 2 - 1, torch.rand(1, 1, 64, 64, generator=g)
    inp = {k: v.to(DEV) for k, v in syn.make_warp_inputs(1, seed=7).items()}
    args = (fimg[:, :3].contiguous().to(DEV), fimg.to(DEV), torch.ones(1, 14, 512, device=DEV), inp['ref_torso_rgb'], inp['ref_bg_rgb'], wimg.to(DEV),
            inp['segmap'], inp['kp_s'], inp['kp_d'])
    srp = syn.make_sr_warp_params(seed=6, weight_fuse=weight_fuse)
    v1 = syn.StubTorsoModelV1()
    m1 = _head(dict(V1, weight_fuse=weight_fuse), mode, v1, srp)
    m2 = _head(dict(syn.WARP_HPARAMS, weight_fuse=weight_fuse), mode, _V1AsV2(syn.StubTorsoModelV1()), srp)
    with torch.no_grad():
        a, _ = m1(*args, noise_mode='none')
        b, _ = m2(*args, noise_mode='none')
    assert v1.calls == 1 and torch.equal(a, b)


# ---- 3. FrameEngine ---------------------------------------------------------------------------------------------------------------------
def _engine(hp, mode, warper_cls, **kw):
    eng = engine.FrameEngine(batch=2, sr_mode=mode, hp=dict(hp, num_samples_fine=48), torso_model=warper_cls(), **kw)
    eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_warp_params(seed=6, weight_fuse=hp['weight_fuse']))
    return eng


def _frames(n_steps, B=2, res=64, seed=60):
    out = []
    for s in range(n_steps):
        u_c, u_f = syn.make_jitter(B, res * res, 48, 48, seed=seed + 10 * s + 2)
        kp_d = torch.rand(B, 68, 3, generator=torch.Generator().manual_seed(seed + 10 * s + 4)) * 2 - 1
        out.append((syn.make_planes(B, seed=seed + 10 * s).to(DEV), syn.make_cameras(B, seed=seed + 10 * s + 1).to(DEV), u_c.to(DEV), u_f.to(DEV),
                    kp_d.to(DEV)))
    return out


def _run(eng, frames):
    return torch.cat([eng.step(*f[:4], kp_d=f[4]).clone() for f in frames])


@pytest.mark.parametrize('u8', [False, True])
@pytest.mark.parametrize('config', ['nofuse', 'v1'])
def test_engine_paths_bit_identical(config, u8):
    """Eager, split-graph, whole-graph and prepared steps are bit-identical to each other and to RenderHead.synthesis(lean=True), in fp32 and
    uint8 ('tc'; 'tc_exact' for weight_fuse=False)."""
    hp, warper = (NOFUSE, syn.StubTorsoModel) if config == 'nofuse' else (V1, syn.StubTorsoModelV1)
    inp = syn.make_warp_inputs(1, seed=7)
    consts = tuple(inp[k].to(DEV) for k in ('ref_torso_rgb', 'ref_bg_rgb', 'segmap', 'kp_s'))
    frames = _frames(2)
    for mode in (('tc', 'tc_exact') if config == 'nofuse' else ('tc',)):
        engs = {'eager': _engine(hp, mode, warper, use_graph=False, out_uint8=u8), 'split': _engine(hp, mode, warper, out_uint8=u8),
                'whole': _engine(hp, mode, warper, warper_in_graph=True, out_uint8=u8), 'prepared': _engine(hp, mode, warper, out_uint8=u8)}
        for e in engs.values():
            e.begin_clip(*consts)
        assert engs['split'].eager_reason is None
        ref = _run(engs['eager'], frames)
        assert ref.dtype == (torch.uint8 if u8 else torch.float32)
        assert torch.equal(_run(engs['split'], frames), ref) and torch.equal(_run(engs['whole'], frames), ref)
        assert isinstance(engs['split'].graph, engine._TorsoGraphs) and isinstance(engs['whole'].graph, torch.cuda.CUDAGraph)
        assert engs['prepared'].prepare(frames) == len(frames)
        assert torch.equal(_run(engs['prepared'], frames), ref)
        head, B = engs['eager'].head, 2
        for i, f in enumerate(frames):
            cond = {'ref_torso_img': consts[0], 'bg_img': consts[1], 'segmap': consts[2].expand(B, -1, -1, -1).contiguous(),
                    'kp_s': consts[3].expand(B, -1, -1).contiguous(), 'kp_d': f[4]}
            lean = head.synthesis(f[0], f[1], cond=cond, lean=True, out_uint8=u8, u_coarse=f[2], u_fine=f[3])['image']
            assert torch.equal(lean, ref[i * B:(i + 1) * B]), (config, mode, i)
        if config == 'v1':
            assert engs['eager'].head.superresolution.torso_model.calls > 0
