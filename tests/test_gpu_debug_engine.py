"""FrameEngine(out_mode='concat_debug'): a clip of debug strips equals the restatement of real3d_infer.py:494-521 applied to the same inputs'
fp32 frames from an out_mode='final' engine, image_raw / image_depth from RenderHead.synthesis with the same jitter, and the SECC image the
step used; for the plain head with cond_tgt, the SECC renderer with blink, and the torso head (split graphs, then prepare() graphs).
out_mode='final' keeps the engine's launches and frames."""
import random

import pytest
import torch

import real3dportrait_b200 as r3
import secc2plane_reference as s2p_ref
from debug_frames_reference import concat_debug_reference
from real3dportrait_b200 import engine, synthetic as syn

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
B = 2
TORSO_HP = dict(syn.WARP_HPARAMS, htbsr_head_weight_fuse_mode='v2', num_samples_fine=48, neural_rendering_resolution=64)


def _backbone(seed=7):
    bb = r3.SegFormerSECC2PlaneBackbone()
    bb.load_state_dict(s2p_ref.make_params({k: v.shape for k, v in bb.state_dict().items()}, seed), strict=True)
    return bb.to(DEV).eval()


def _engine(torso=False, **kw):
    kw.setdefault('out_uint8', True)
    if torso:
        eng = engine.FrameEngine(batch=B, sr_mode='tc', hp=TORSO_HP, torso_model=syn.StubTorsoModel(), secc2plane=_backbone(), **kw)
        eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_warp_params(seed=6, fuse_mode='v2'))
        inp = syn.make_warp_inputs(1, seed=3)
        eng.begin_clip(*(inp[k].to(DEV) for k in ('ref_torso_rgb', 'ref_bg_rgb', 'segmap', 'kp_s')))
    else:
        eng = engine.FrameEngine(batch=B, sr_mode='tc', hp={'num_samples_fine': 0}, secc2plane=_backbone(), **kw)
        eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_params(seed=5))
    return eng


def _ref_gt(seed=5):
    b = torch.randint(0, 256, (1, 3, 512, 512), generator=torch.Generator().manual_seed(seed)).float()
    return ((b - 127.5) / 127.5).to(DEV)


def _steps(n, torso, seed=40):
    """Per step: (cond_tgt [B,3,512,512], cameras, u_coarse, u_fine, kp_d)."""
    out = []
    for s in range(n):
        _, _, tgt = s2p_ref.make_inputs(B, 512, seed + s)
        u_c, u_f = syn.make_jitter(B, 4096, 48, 48 if torso else 0, seed=seed + s + 100)
        kp = (torch.rand(B, 68, 3, generator=torch.Generator().manual_seed(seed + s + 300)) * 2 - 1).to(DEV) if torso else None
        out.append((tgt.to(DEV), syn.make_cameras(B, seed=seed + s + 200).to(DEV), u_c.to(DEV), None if u_f is None else u_f.to(DEV), kp))
    return out


def _raw_depth(eng, secc, f):
    """image_raw and image_depth of RenderHead.synthesis (the full ret dict) on the step's planes and jitter."""
    planes = (eng._cano_cl, eng.secc.planes_cl(secc))
    cond = None
    if eng.torso:
        c = eng._cond(f[4])
        cond = dict(c, ref_torso_img=c['ref_torso_img'].expand(B, -1, -1, -1), bg_img=c['bg_img'].expand(B, -1, -1, -1))
    over = {'u_coarse': f[2]} if f[3] is None else {'u_coarse': f[2], 'u_fine': f[3]}
    ret = eng.head.synthesis(planes, f[1], cond=cond, **over)
    return ret['image_raw'].cpu(), ret['image_depth'].cpu()


def _run_clip(dbg, fin, steps, fpr, ref_gt, secc_of, kw_of):
    """Steps through dbg (concat_debug) and fin (final, fp32) -> (dbg's clip, the restatement's clip) on the CPU."""
    dbg.open_clip(fpr, ref_gt_img=ref_gt)
    secc, raw, depth, image = [], [], [], []
    for i, f in enumerate(steps):
        kw = kw_of(f)
        frames = dbg.step(None, *f[1:4], frame_index=i * B, **kw)
        assert frames.shape == (B, 512, 2560, 3) and frames.dtype == torch.uint8
        image.append(fin.step(None, *f[1:4], **kw).clone().cpu())
        s = secc_of(f)
        secc.append(s.cpu())
        r, d = _raw_depth(dbg, s, f)
        raw.append(r)
        depth.append(d)
    clip = dbg.close_clip()
    assert clip.shape == (fpr, 512, 2560, 3)
    want = concat_debug_reference(ref_gt.cpu(), torch.cat(secc)[:fpr], torch.cat(raw)[:fpr], torch.cat(depth)[:fpr], torch.cat(image)[:fpr])
    return clip.cpu(), want


@torch.no_grad()
def test_plain_head_with_cond_tgt():
    dbg, fin = _engine(out_mode='concat_debug'), _engine(out_uint8=False)
    eager = _engine(out_mode='concat_debug', use_graph=False)
    cano, c_cano, c_src = syn.make_planes(1, seed=1).to(DEV), *(t.to(DEV) for t in s2p_ref.make_inputs(1, 512, 1)[:2])
    for e in (dbg, fin, eager):
        e.begin_planes(cano, c_cano, c_src)
    steps = _steps(3, False)
    ref_gt = _ref_gt()
    kw_of = lambda f: {'cond_tgt': f[0]}                                 # noqa: E731
    got, want = _run_clip(dbg, fin, steps, 3 * B - 1, ref_gt, lambda f: f[0], kw_of)   # the last step's second frame falls off the clip
    assert torch.equal(got, want)
    got_e, _ = _run_clip(eager, fin, steps, 3 * B - 1, ref_gt, lambda f: f[0], kw_of)
    assert torch.equal(got_e, want)
    # a second clip through the captured graph, with a new source image
    got2, want2 = _run_clip(dbg, fin, steps[::-1], 3 * B, _ref_gt(6), lambda f: f[0], kw_of)
    assert torch.equal(got2, want2)


@torch.no_grad()
def test_renderer_with_blink(tmp_path):
    r = r3.SECC_Renderer(512, device=DEV, **syn.write_bfm_folder(str(tmp_path), seed=0))
    dbg = _engine(out_mode='concat_debug', secc_renderer=r, blink=True)
    fin = _engine(out_uint8=False, secc_renderer=r, blink=True)
    c = syn.make_coeffs(1, seed=1)
    cano, cs = syn.make_planes(1, seed=1).to(DEV), torch.cat([c['id'], c['exp']], 1).to(DEV)
    for e in (dbg, fin):
        e.begin_planes(cano, coeff_src=cs)
    sched = r3.period_blink_schedule(3 * B, rng=random.Random(3))
    steps, rows = _steps(3, False), []
    for s in range(3):
        cc = syn.make_coeffs(B, seed=50 + s)
        rows.append(torch.cat([cc['id'], cc['exp'], sched[s * B:(s + 1) * B].float()], 1).to(DEV))
    steps = [(rows[i],) + f[1:] for i, f in enumerate(steps)]

    def secc_of(f):
        secc = r.render(f[0][:, :144])[1]
        r.blink(secc, rows=f[0][:, 144:])
        return secc
    got, want = _run_clip(dbg, fin, steps, 3 * B, _ref_gt(), secc_of, lambda f: {'coeff': f[0]})
    assert torch.equal(got, want)


@torch.no_grad()
def test_torso_head_split_graphs_and_prepare():
    dbg, fin = _engine(True, out_mode='concat_debug'), _engine(True, out_uint8=False)
    cano, c_cano, c_src = syn.make_planes(1, seed=1).to(DEV), *(t.to(DEV) for t in s2p_ref.make_inputs(1, 512, 1)[:2])
    for e in (dbg, fin):
        e.begin_planes(cano, c_cano, c_src)
    steps = _steps(3, True)
    kw_of = lambda f: {'cond_tgt': f[0], 'kp_d': f[4]}                    # noqa: E731
    got, want = _run_clip(dbg, fin, steps, 3 * B, _ref_gt(), lambda f: f[0], kw_of)
    assert torch.equal(got, want)
    assert dbg.graph is not None
    assert dbg.prepare([f[:5] for f in steps]) == len(steps)
    got2, want2 = _run_clip(dbg, fin, steps, 3 * B, _ref_gt(), lambda f: f[0], kw_of)
    assert torch.equal(got2, want2) and torch.equal(got2, want)


@torch.no_grad()
def test_final_mode_keeps_launches_and_frames():
    a, b = _engine(), _engine(out_mode='final')
    cano, c_cano, c_src = syn.make_planes(1, seed=1).to(DEV), *(t.to(DEV) for t in s2p_ref.make_inputs(1, 512, 1)[:2])
    for e in (a, b):
        e.begin_planes(cano, c_cano, c_src)
    for f in _steps(2, False):
        assert torch.equal(a.step(None, *f[1:3], cond_tgt=f[0]).clone(), b.step(None, *f[1:3], cond_tgt=f[0]))
    assert a.launches_per_step == b.launches_per_step > 0
    assert b.frame_shape() == (512, 512, 3)
    d, fp = _engine(out_mode='concat_debug'), _engine(out_uint8=False)
    f = _steps(1, False)[0]
    for e in (d, fp):
        e.begin_planes(cano, c_cano, c_src)
    d.open_clip(B, ref_gt_img=_ref_gt())
    d.step(None, *f[1:3], cond_tgt=f[0], frame_index=0)
    fp.step(None, *f[1:3], cond_tgt=f[0])
    assert d.launches_per_step == fp.launches_per_step + 1 and d.frame_shape() == (512, 2560, 3)   # the fp32 step, then the panel kernel


@torch.no_grad()
def test_rejections():
    d = _engine(out_mode='concat_debug')
    cano, c_cano, c_src = syn.make_planes(1, seed=1).to(DEV), *(t.to(DEV) for t in s2p_ref.make_inputs(1, 512, 1)[:2])
    d.begin_planes(cano, c_cano, c_src)
    f = _steps(1, False)[0]
    with pytest.raises(RuntimeError, match='open clip'):
        d.step(None, *f[1:3], cond_tgt=f[0], frame_index=0)
    with pytest.raises(ValueError):
        d.open_clip(B)
    d.open_clip(B, ref_gt_img=_ref_gt())
    with pytest.raises(RuntimeError, match='frame_index'):
        d.step(None, *f[1:3], cond_tgt=f[0])
    with pytest.raises(NotImplementedError):
        d.step_host(*(t.cpu() for t in f[:3]), torch.empty(B, 512, 2560, 3, dtype=torch.uint8))
    with pytest.raises(ValueError):
        _engine().open_clip(B, ref_gt_img=_ref_gt())
