"""SECC blink on the GPU (r3dp_secc_blink, SECC_Renderer.blink, blink_eye_for_secc, FrameEngine(blink=True)):
  - the kernel equals the numpy restatement (tests/blink_reference.py, tie='lowest') bit for bit, on the fixture's inputs and on rendered
    images at S = 512, 224, 250, 97 and B = 1, 4, 13, with untouched, p = 0 and (t, T) images mixed in one call
  - outside tied pixels it equals the reference's own output (tests/golden/blink_secc.npz)
  - untouched images, guards around the batch and the scratch, graph replays, faults, and the engine against render + blink."""
import os
import random

import numpy as np
import pytest
import torch

import blink_reference as bref
import secc2plane_reference as s2p_ref
import real3dportrait_b200 as r3
from real3dportrait_b200 import _capi as capi, engine, synthetic as syn

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'blink_secc.npz')
EB = 4


@pytest.fixture(scope='module')
def bfm_kw(tmp_path_factory):
    return syn.write_bfm_folder(str(tmp_path_factory.mktemp('bfm')), seed=0)


@pytest.fixture(scope='module')
def renderers(bfm_kw):
    return {S: r3.SECC_Renderer(S, device=DEV, **bfm_kw) for S in (512, 224, 250, 97)}


def _want(x, ctl):
    """Restatement of one image x [3,S,S] under control ctl (None = untouched, a float p, or (t, T)) -> (fp32 image, faulted)."""
    if ctl is None:
        return x, False
    p = bref.schedule_p(*ctl) if isinstance(ctl, tuple) else ctl
    try:
        return bref.blink(x, p, tie='lowest')[0], False
    except ValueError:
        return x, True


def _rows(ctls, width=2):
    rows = torch.zeros(len(ctls), width)
    for b, c in enumerate(ctls):
        if isinstance(c, tuple):
            rows[b, -2], rows[b, -1] = c
    return rows.to(DEV)


def _check(r, x, ctls, use_p=False):
    """Run blink on x [B,3,S,S] (numpy fp32) under ctls; every image must equal the restatement bit for bit."""
    secc = torch.from_numpy(x).to(DEV)
    r.blink_faults()
    if use_p:
        r.blink(secc, p=[-1.0 if c is None else (bref.schedule_p(*c) if isinstance(c, tuple) else c) for c in ctls])
    else:
        wide = _rows(ctls, width=7)
        r.blink(secc, rows=wide[:, 5:])                                  # (t, T) read in place from a wider row
    got = secc.cpu().numpy()
    faults = 0
    for b, c in enumerate(ctls):
        want, fault = _want(x[b], c)
        faults += fault
        assert np.array_equal(got[b].view(np.uint32), want.view(np.uint32)), f'image {b} control {c}: {(got[b] != want).sum()} values differ'
    assert r.blink_faults() == faults
    return got


def _gold():
    g = np.load(GOLD)
    return g, [tuple(int(v) for v in c) for c in g['cases']], [g[f'img{k}_q'] for k in range(len(g['images']))]


def test_kernel_on_fixture_inputs_and_against_reference(renderers):
    g, cases, imgs = _gold()
    for k, q in enumerate(imgs):
        S = q.shape[-1]
        r = renderers[S]
        x = bref.encode(q)
        ctls = [None] + cases
        got = _check(r, np.stack([x] * len(ctls)), ctls)
        assert np.array_equal(got[0].view(np.uint32), x.view(np.uint32))        # untouched: byte-identical
        for b, (t, T) in enumerate(cases, 1):
            want_q = q.astype(np.int64).copy().reshape(3, -1)
            idx = g[f'img{k}_t{t}_T{T}_idx']
            want_q[:, idx] = g[f'img{k}_t{t}_T{T}_q']
            _, _, ties, _ = bref.blink(x, bref.schedule_p(t, T), tie='lowest')
            bref.equal_outside_ties(bref.codes(got[b]), q.astype(np.int64), want_q.reshape(q.shape), ties)


@pytest.mark.parametrize('S', [512, 224, 250, 97])
@pytest.mark.parametrize('B', [1, 4, 13])
def test_kernel_on_rendered_images(renderers, S, B):
    r = renderers[S]
    c = syn.make_coeffs(B, seed=100 + S + B)
    secc = r.render(torch.cat([c['id'], c['exp']], 1).to(DEV))[1]
    x = secc.cpu().numpy()
    rng = random.Random(S * 31 + B)
    menu = [None, (0, 8), 0.0, (1, 8), (4, 8), (5, 10), (11, 12), (3, 9), 1.0, 0.44]
    ctls = [menu[(b * 3 + 3) % len(menu)] if B > 1 else (5, 10) for b in range(B)]
    rows_ctls = [c if not isinstance(c, float) else ((0, 8) if c == 0.0 else (rng.randint(1, 7), 8)) for c in ctls]
    _check(r, x, rows_ctls)
    _check(r, x, ctls, use_p=True)


def test_threshold_rows_need_double_p(renderers):
    """Hand-made 128^2 images whose hole columns hold eye rows on which p mean + (1 - p) min lands up to its last rounding (holes over rows
    [32, 51) and [35, 56)), under every (t, T) with 8 <= T <= 12: an fp32 p or a fused multiply-add in the thresholds flips some of them."""
    r = renderers[97]
    imgs, ctls = [], []
    for r0, r1 in ((32, 51), (35, 56)):
        q = np.full((3, 128, 128), 150, dtype=np.int64)
        q[:, r0:r1, 40:50] = 0
        q[:, r0:r1, 72:82] = 0
        for T in range(8, 13):
            for t in range(1, T):
                imgs.append(bref.encode(q))
                ctls.append((t, T))
    x = np.stack(imgs)
    assert any(not np.array_equal(bref.blink(x[b], bref.schedule_p(*c))[1], bref.blink(x[b], bref.schedule_p(*c), p32=True)[1])
               for b, c in enumerate(ctls))
    _check(r, x, ctls)


def test_guards(renderers):
    """Sentinels around the image batch and the scratch buffer stay intact (the C entry point on sliced buffers)."""
    r = renderers[224]
    B, S, G = 3, 224, 4096
    c = syn.make_coeffs(B, seed=5)
    secc = r.render(torch.cat([c['id'], c['exp']], 1).to(DEV))[1]
    x = secc.cpu().numpy()
    big = torch.full((B * 3 * S * S + 2 * G,), float('nan'), device=DEV)
    big[G:-G] = secc.reshape(-1)
    n = int(capi.lib().r3dp_secc_blink_scratch_bytes(B, S))
    sc_big = torch.full((n + 2 * G,), 0xA5, dtype=torch.uint8, device=DEV)
    faults = torch.zeros(1, dtype=torch.int32, device=DEV)
    ctls = [(3, 8), None, (5, 10)]
    rows = _rows(ctls)
    capi.check(capi.lib().r3dp_secc_blink(capi.ptr(big[G:-G]), B, S, capi.ptr(None), capi.ptr(rows), 2,
                                          capi.ptr(sc_big[G:G + n], torch.uint8), capi.ptr(faults, torch.int32), capi.stream()))
    torch.cuda.synchronize()
    assert torch.isnan(big[:G]).all() and torch.isnan(big[-G:]).all()
    assert (sc_big[:G] == 0xA5).all() and (sc_big[G + n:] == 0xA5).all()
    got = big[G:-G].view(B, 3, S, S).cpu().numpy()
    for b, ctl in enumerate(ctls):
        want, _ = _want(x[b], ctl)
        assert np.array_equal(got[b].view(np.uint32), want.view(np.uint32))


def test_graph_replay(renderers):
    r = renderers[512]
    B = 4
    c = syn.make_coeffs(B, seed=9, yaw=0.3)
    src = r.render(torch.cat([c['id'], c['exp']], 1).to(DEV))[1]
    ctl_a, ctl_b = [(2, 8), None, (0, 10), (6, 12)], [None, (5, 10), (4, 8), (1, 9)]
    rows = _rows(ctl_a)
    work = src.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        work.copy_(src)
        r.blink(work, rows=rows)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        work.copy_(src)
        r.blink(work, rows=rows)
    for ctl in (ctl_a, ctl_b, ctl_a):
        rows.copy_(_rows(ctl))
        g.replay()
        eager = src.clone()
        r.blink(eager, rows=_rows(ctl))
        torch.cuda.synchronize()
        assert torch.equal(work.view(torch.int32), eager.view(torch.int32))


def _fault_images(S):
    q = np.full((3, S, S), 150, dtype=np.int64)                        # all face: no coarse pixel
    all_face = bref.encode(q)
    return all_face, bref.encode(np.zeros_like(q))                   # a blank frame: coarse is the whole prior region, er is empty


def test_faults(renderers):
    r = renderers[224]
    S = 224
    c = syn.make_coeffs(1, seed=11)
    good = r.render(torch.cat([c['id'], c['exp']], 1).to(DEV))[1][0].cpu().numpy()
    f1, f2 = _fault_images(S)
    x = np.stack([f1, good, f2])
    got = _check(r, x, [(3, 8), (3, 8), (4, 8)])                       # the faulted images are left as they were, and counted
    assert np.array_equal(got[0].view(np.uint32), f1.view(np.uint32)) and np.array_equal(got[2].view(np.uint32), f2.view(np.uint32))
    for f in (f1, f2):
        with pytest.raises(ValueError):
            r3.blink_eye_for_secc(torch.from_numpy(f).to(DEV), 0.5)
        assert torch.equal(r3.blink_eye_for_secc(torch.from_numpy(f).to(DEV), 0.0).cpu(), torch.from_numpy(bref.dequantise(bref.quantise(f))))
    out = r3.blink_eye_for_secc(torch.from_numpy(good).to(DEV), 0.5)
    assert out.device.type == 'cuda' and out.shape == (3, S, S)
    assert np.array_equal(out.cpu().numpy().view(np.uint32), bref.blink(good, 0.5)[0].view(np.uint32))
    with pytest.raises(ValueError):
        r3.blink_eye_for_secc(torch.from_numpy(good).to(DEV), 1.5)


# ---- engine ----------------------------------------------------------------------------------------------------------------------------

def _backbone(seed=7):
    bb = r3.SegFormerSECC2PlaneBackbone()
    bb.load_state_dict(s2p_ref.make_params({k: v.shape for k, v in bb.state_dict().items()}, seed), strict=True)
    return bb.to(DEV).eval()


def _plain(**kw):
    eng = engine.FrameEngine(batch=EB, sr_mode='tc', hp={'num_samples_fine': 0}, out_uint8=True, **kw)
    eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_params(seed=5))
    return eng


def _src(seed):
    c = syn.make_coeffs(1, seed=seed)
    return syn.make_planes(1, seed=seed).to(DEV), torch.cat([c['id'], c['exp']], 1).to(DEV)


def _clip(n, sched, seed=40):
    """Steps of EB frames: ([id | exp | t | T] rows, cameras, u_coarse)."""
    out = []
    for s in range(n // EB):
        c = syn.make_coeffs(EB, seed=seed + s)
        u_c, _ = syn.make_jitter(EB, 4096, 48, 0, seed=seed + s + 100)
        rows = torch.cat([c['id'], c['exp'], sched[s * EB:(s + 1) * EB].float()], 1)
        out.append((rows.to(DEV), syn.make_cameras(EB, seed=seed + s + 200).to(DEV), u_c.to(DEV)))
    return out


@torch.no_grad()
def test_engine_blink_equals_render_then_blink(renderers):
    r = renderers[512]
    with pytest.raises(ValueError):
        _plain(secc2plane=_backbone(), blink=True)
    sched = r3.period_blink_schedule(16, rng=random.Random(3))
    assert (sched[:, 1] > 0).any() and (sched[:, 1] == 0).any()
    b_eng = _plain(secc2plane=_backbone(), secc_renderer=r, blink=True)
    e_eng = _plain(secc2plane=_backbone(), secc_renderer=r, blink=True, use_graph=False)
    img_eng = _plain(secc2plane=_backbone())
    cano, cs = _src(1)
    for e in (b_eng, e_eng):
        e.begin_planes(cano, coeff_src=cs)
    img_eng.begin_planes(cano, r.render(torch.cat([cs[:, :80], torch.zeros_like(cs[:, 80:])], 1))[1], r.render(cs)[1])
    for rows, cams, u in _clip(16, sched):
        with pytest.raises(ValueError):
            b_eng.step(None, cams, u, coeff=rows[:, :144])
        got = b_eng.step(None, cams, u, coeff=rows).clone()
        secc = r.render(rows[:, :144])[1]
        r.blink(secc, rows=rows[:, 144:])
        want = img_eng.step(None, cams, u, cond_tgt=secc).clone()
        assert torch.equal(got, want) and torch.equal(got, e_eng.step(None, cams, u, coeff=rows))
    assert b_eng.blink_faults() == 0
    # T = 0 everywhere: the same frames as an engine without blink
    plain = _plain(secc2plane=_backbone(), secc_renderer=r)
    plain.begin_planes(cano, coeff_src=cs)
    for rows, cams, u in _clip(8, torch.zeros(8, 2, dtype=torch.int32), seed=60):
        assert torch.equal(b_eng.step(None, cams, u, coeff=rows).clone(), plain.step(None, cams, u, coeff=rows[:, :144]))
    # step_host carries the wider rows in the planes slot
    rows, cams, u = _clip(4, sched)[0]
    h = [t.cpu().pin_memory() for t in (rows, cams, u)]
    h_out = torch.empty(EB, 512, 512, 3, dtype=torch.uint8).pin_memory()
    b_eng.step_host(*h, h_out)
    b_eng.sync_host()
    assert torch.equal(h_out, e_eng.step(None, cams, u, coeff=rows).cpu())


@torch.no_grad()
def test_torso_engine_blink_step(renderers):
    r = renderers[512]
    hp = dict(syn.WARP_HPARAMS, htbsr_head_weight_fuse_mode='v2', num_samples_fine=48, neural_rendering_resolution=64)

    def mk(**kw):
        eng = engine.FrameEngine(batch=EB, sr_mode='tc', hp=hp, torso_model=syn.StubTorsoModel(), out_uint8=True, secc2plane=_backbone(), **kw)
        eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_warp_params(seed=6, fuse_mode='v2'))
        inp = syn.make_warp_inputs(1, seed=3)
        eng.begin_clip(*(inp[k].to(DEV) for k in ('ref_torso_rgb', 'ref_bg_rgb', 'segmap', 'kp_s')))
        return eng
    b_eng, img_eng = mk(secc_renderer=r, blink=True), mk()
    cano, cs = _src(1)
    b_eng.begin_planes(cano, coeff_src=cs)
    img_eng.begin_planes(cano, r.render(torch.cat([cs[:, :80], torch.zeros_like(cs[:, 80:])], 1))[1], r.render(cs)[1])
    sched = torch.tensor([[1, 8], [2, 8], [0, 0], [6, 10]], dtype=torch.int32)
    rows, cams, _ = _clip(4, sched, seed=70)[0]
    u_c, u_f = syn.make_jitter(EB, 64 * 64, 48, 48, seed=71)
    kp_d = (torch.rand(EB, 68, 3, generator=torch.Generator().manual_seed(72)) * 2 - 1).to(DEV)
    got = b_eng.step(None, cams, u_c.to(DEV), u_f.to(DEV), kp_d=kp_d, coeff=rows).clone()
    secc = r.render(rows[:, :144])[1]
    r.blink(secc, rows=rows[:, 144:])
    assert torch.equal(got, img_eng.step(None, cams, u_c.to(DEV), u_f.to(DEV), kp_d=kp_d, cond_tgt=secc))
