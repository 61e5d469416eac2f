"""The torso head (SuperresolutionHybrid8XDC_Warp) through FrameEngine: the one-launch input hand-off, eager / split-graph / whole-graph /
zero-copy steps, uint8 frames, per-clip constants over two clips, the other fuse modes, the clip buffer and the host-buffer entry point.
The warper is synthetic.StubTorsoModel everywhere."""
import pytest
import torch

from real3dportrait_b200 import _capi as capi, engine, synthetic as syn
from oracle import real3d_oracle as orc

pytestmark = pytest.mark.gpu
DEV = 'cuda'
TC_MAXABS, TC_PSNR = 5e-3, 70.0        # the tensor-core SR's stated tolerance against fp32 (tests/test_gpu_parity.py)


def _maxdiff(a, b):
    return float((a.detach().float().cpu() - b.detach().float().cpu()).abs().max())


def _psnr(img, ref):
    mse = float(((img.detach().float().cpu() - ref) ** 2).mean())
    return 10 * torch.log10(torch.tensor(float(ref.max() - ref.min()) ** 2 / max(mse, 1e-30))).item()


def _hp(fuse='v2', res=64):
    return dict(syn.WARP_HPARAMS, htbsr_head_weight_fuse_mode=fuse, num_samples_fine=48, neural_rendering_resolution=res)


def _engine(mode='tc', fuse='v2', B=2, res=64, **kw):
    eng = engine.FrameEngine(batch=B, sr_mode=mode, hp=_hp(fuse, res), torso_model=syn.StubTorsoModel(), **kw)
    eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_warp_params(seed=6, fuse_mode=fuse))
    return eng


def _clip_consts(seed):
    inp = syn.make_warp_inputs(1, seed=seed)
    return tuple(inp[k].to(DEV) for k in ('ref_torso_rgb', 'ref_bg_rgb', 'segmap', 'kp_s'))


def _frames(n_steps, B, res=64, seed=60):
    """Per step: (planes [B,3,32,256,256], cameras, u_coarse, u_fine, kp_d) on the device."""
    out = []
    for s in range(n_steps):
        u_c, u_f = syn.make_jitter(B, res * res, 48, 48, seed=seed + 10 * s + 2)
        kp_d = torch.rand(B, 68, 3, generator=torch.Generator().manual_seed(seed + 10 * s + 4)) * 2 - 1
        out.append((syn.make_planes(B, seed=seed + 10 * s).to(DEV), syn.make_cameras(B, seed=seed + 10 * s + 1).to(DEV), u_c.to(DEV), u_f.to(DEV),
                    kp_d.to(DEV)))
    return out


def _run(eng, frames):
    return torch.cat([eng.step(*f[:4], kp_d=f[4]).clone() for f in frames])


def _synthesis(eng, f, consts):
    """RenderHead.synthesis() (the non-lean path, the full ret dict) on the same inputs and constants."""
    B = f[0].shape[0]
    t, bg, seg, kps = consts
    cond = {'ref_torso_img': t.expand(B, -1, -1, -1), 'bg_img': bg.expand(B, -1, -1, -1), 'segmap': seg.expand(B, -1, -1, -1).contiguous(),
            'kp_s': kps.expand(B, -1, -1).contiguous(), 'kp_d': f[4]}
    return eng.head.synthesis(f[0], f[1], cond=cond, u_coarse=f[2], u_fine=f[3])['image']


# ---- 1. the one-launch hand-off ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('res', [64, 128])
@pytest.mark.parametrize('split', [0, 1])
def test_warp_input_equals_three_launch_sequence(res, split):
    N, C, R = 2, 32, 128
    g = torch.Generator().manual_seed(res + split)
    x = (torch.randn(N, res, res, C, generator=g)).to(DEV)
    wsum = torch.rand(N, res * res, 1, generator=g).to(DEV)
    L, wide = capi.lib(), 2 if split else 1
    outs = []
    for fused in (False, True):
        y = torch.full((N, R, R, 64 * wide), 7.0, device=DEV, dtype=torch.float16)
        rgb0 = torch.full((N, 3, R, R), 7.0, device=DEV)
        rgb256, w256 = torch.full((N, 3, 256, 256), 7.0, device=DEV), torch.full((N, 1, 256, 256), 7.0, device=DEV)
        if fused:
            capi.check(L.r3dp_sr_warp_input(capi.ptr(x), capi.ptr(wsum), N, C, res, res, R, capi.ptr(y, torch.float16), capi.ptr(rgb0), capi.ptr(rgb256),
                                            capi.ptr(w256), split, capi.stream()))
        else:
            capi.check(L.r3dp_sr_tc_input_nhwc_rgb(capi.ptr(x), N, C, res, res, R, capi.ptr(y, torch.float16), capi.ptr(rgb0), split, capi.stream()))
            capi.check(L.r3dp_sr_resize_bilinear(capi.ptr(rgb0), N, 3, R, R, 256, capi.ptr(rgb256), capi.stream()))
            capi.check(L.r3dp_sr_resize_bilinear(capi.ptr(wsum), N, 1, res, res, 256, capi.ptr(w256), capi.stream()))
        outs.append((y, rgb0, rgb256, w256))
    torch.cuda.synchronize()
    for name, a, b in zip(('x0', 'rgb0', 'rgb_256', 'weights_256'), *outs):
        assert torch.equal(a.view(torch.int16) if a.dtype == torch.float16 else a.view(torch.int32),
                           b.view(torch.int16) if b.dtype == torch.float16 else b.view(torch.int32)), name


# ---- 2. engine paths against eager and against RenderHead.synthesis() -------------------------------------------------------------------
def test_engine_graph_paths_match_eager_and_synthesis():
    B = 2
    consts = _clip_consts(7)
    frames = _frames(3, B)
    engs = {'eager': _engine(use_graph=False), 'split': _engine(), 'whole': _engine(warper_in_graph=True), 'prepared': _engine()}
    for e in engs.values():
        e.begin_clip(*consts)
    assert engs['split'].head.superresolution.static_prepared_warp is not None
    ref = _run(engs['eager'], frames)
    got_split, got_whole = _run(engs['split'], frames), _run(engs['whole'], frames)
    assert isinstance(engs['split'].graph, engine._TorsoGraphs) and isinstance(engs['whole'].graph, torch.cuda.CUDAGraph)
    assert torch.equal(got_split, ref) and torch.equal(got_whole, ref)
    assert engs['prepared'].prepare(frames) == len(frames)
    assert torch.equal(_run(engs['prepared'], frames), ref)
    # a kp_d buffer refilled in place is read by the prepared graphs
    f0 = frames[0]
    f0[4].copy_(torch.rand(B, 68, 3, generator=torch.Generator().manual_seed(99)).to(DEV) * 2 - 1)
    want = engs['eager'].step(*f0[:4], kp_d=f0[4]).clone()
    assert not torch.equal(want, ref[:B])
    assert torch.equal(engs['prepared'].step(*f0[:4], kp_d=f0[4]), want)
    # the non-lean head call with the same cond (its own weight preparation, NCHW inputs, clamp after the SR)
    for i, f in enumerate(frames):
        full = _synthesis(engs['eager'], f, consts)
        expect = want if i == 0 else ref[i * B:(i + 1) * B]
        err = _maxdiff(full, expect)
        print(f'step {i}: engine vs RenderHead.synthesis() max-abs {err:.2e}')
        assert err <= 1e-6, err


# ---- 3. uint8 frames ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('mode', ['tc', 'tc_exact'])
def test_engine_uint8_frames(mode):
    consts, frames = _clip_consts(7), _frames(2, 2)
    e32, e8 = _engine(mode), _engine(mode, out_uint8=True)
    for e in (e32, e8):
        e.begin_clip(*consts)
    img, img8 = _run(e32, frames), _run(e8, frames)
    want = ((img + 1) / 2 * 255).int().permute(0, 2, 3, 1).to(torch.uint8)
    assert img8.dtype == torch.uint8 and tuple(img8.shape) == (4, 512, 512, 3)
    assert torch.equal(img8, want)


# ---- 4. against the oracle, at both neural rendering resolutions -----------------------------------------------------------------------
@pytest.mark.parametrize('res', [64, 128])
def test_engine_vs_oracle(res):
    N = 1
    planes, cam = syn.make_planes(N, seed=40), syn.make_cameras(N, seed=41)
    u_c, u_f = syn.make_jitter(N, res * res, 48, 48, seed=42)
    mlp, srp = syn.make_decoder_params(seed=4), syn.make_sr_warp_params(seed=6)
    inp = syn.make_warp_inputs(N, seed=43)
    c2w, K = syn.split_camera(cam)
    o, d = orc.gen_rays(c2w, K, res)
    feat, _, wsum, _ = orc.render(planes, mlp, o, d, S=48, S_imp=48, u_coarse=u_c, u_fine=u_f, lib=True)
    fimg, wimg = orc.feature_image(feat, res), orc.feature_image(wsum, res)
    ref, _ = orc.superres_warp(fimg[:, :3], fimg, torch.ones(N, 14, 512), inp['ref_torso_rgb'], inp['ref_bg_rgb'], wimg, inp['segmap'], inp['kp_s'],
                               inp['kp_d'], srp, syn.StubTorsoModel())
    ref = ref.clamp(-1, 1)
    rng = float(ref.max() - ref.min())
    for mode in ('tc', 'tc_exact'):
        eng = _engine(mode, B=N, res=res)
        eng.begin_clip(*(inp[k].to(DEV) for k in ('ref_torso_rgb', 'ref_bg_rgb', 'segmap', 'kp_s')))
        img = eng.step(planes.to(DEV), cam.to(DEV), u_c.to(DEV), u_f.to(DEV), kp_d=inp['kp_d'].to(DEV))
        err, psnr = _maxdiff(img, ref), _psnr(img, ref)
        print(f'res {res} {mode}: max-abs {err:.3e} on range {rng:.2f}, PSNR {psnr:.1f} dB')
        if mode == 'tc':
            assert err < TC_MAXABS and psnr > TC_PSNR, (err, psnr)
        else:
            assert err < 1e-3 * rng, (err, rng)


# ---- 5. two clips in a row ----------------------------------------------------------------------------------------------------------------
def test_second_clip_reuses_the_captured_graphs():
    c1, c2 = _clip_consts(7), _clip_consts(17)
    frames = _frames(2, 2)
    eng, eager = _engine(), _engine(use_graph=False)
    eng.begin_clip(*c1)
    eng.prepare(frames[:1])
    _run(eng, frames)
    graphs = (eng.graph, dict(eng.inplace))
    eng.begin_clip(*c2)                                                        # refilled in place: the same graphs render the new clip
    assert eng.graph is graphs[0] and eng.inplace.keys() == graphs[1].keys()
    eager.begin_clip(*c2)
    want = _run(eager, frames)
    assert torch.equal(_run(eng, frames), want)
    eng.end_clip()
    with pytest.raises(RuntimeError):
        eng.step(*frames[0][:4], kp_d=frames[0][4])
    eng.begin_clip(*c2)                                                        # after end_clip the graphs are captured again
    assert torch.equal(_run(eng, frames), want)


# ---- 6. fuse modes v1 (graphed) and v3 (eager) ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('fuse', ['v1', 'v3'])
@pytest.mark.parametrize('mode', ['tc', 'tc_exact'])
def test_other_fuse_modes(fuse, mode):
    consts, frames = _clip_consts(7), _frames(2, 2)
    eng = _engine(mode, fuse)
    eng.begin_clip(*consts)
    assert (eng.eager_reason is not None) == (fuse == 'v3')
    got = _run(eng, frames)
    assert (eng.graph is None) == (fuse == 'v3')
    for i, f in enumerate(frames):
        err = _maxdiff(_synthesis(eng, f, consts), got[2 * i:2 * i + 2])
        print(f'fuse {fuse} {mode} step {i}: engine vs RenderHead.synthesis() max-abs {err:.2e}')
        assert err <= 1e-6, err


# ---- 7. the clip buffer and the host-buffer entry point ------------------------------------------------------------------------------
def test_open_clip_and_step_host():
    B = 2
    consts, frames = _clip_consts(7), _frames(3, B)
    eng = _engine(out_uint8=True)
    eng.begin_clip(*consts)
    per_step = []
    clip = eng.open_clip(len(frames) * B)
    for s, f in enumerate(frames):
        per_step.append(eng.step(*f[:4], frame_index=s * B, kp_d=f[4]).clone())
    assert torch.equal(eng.close_clip(), torch.cat(per_step)) and clip.shape == (len(frames) * B, 512, 512, 3)
    outs = [torch.empty(B, 512, 512, 3, dtype=torch.uint8).pin_memory() for _ in frames]
    for f, o in zip(frames, outs):
        eng.step_host(*(t.cpu().pin_memory() for t in f[:3]), o, h_u_fine=f[3].cpu().pin_memory(), h_kp_d=f[4].cpu().pin_memory())
    eng.sync_host()
    assert torch.equal(torch.cat(outs), torch.cat(per_step).cpu())
