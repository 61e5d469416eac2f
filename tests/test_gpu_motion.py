"""ClipMotion on the GPU against the float64 restatement (tests/motion_reference.py) and the reference's fixture.  Bar per output: 2 x the
reference's own float32 deviation from float64 (the fixture's per case; motion_reference.REF_DEV, its bound over the fixture, elsewhere) plus
4 fp32 ulp of the output's largest magnitude.  Also: strided / broadcast inputs, out=, graph capture, the vertex pass's frame split, and the
torso engine fed ClipMotion's outputs."""
import numpy as np
import pytest
import torch

import motion_reference as mref
import secc2plane_reference as s2p_ref
import real3dportrait_b200 as r3
from real3dportrait_b200 import _capi as capi, engine, synthetic as syn

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
NAMES = ('cameras', 'kp_s', 'kp_d')


@pytest.fixture(scope='module')
def bfm(tmp_path_factory):
    kw = syn.write_bfm_folder(str(tmp_path_factory.mktemp('bfm')), seed=0, keypoints=True)
    return kw, mref.load(kw['bfm_folder']), r3.ClipMotion(kw['bfm_folder'], device=DEV)


def _dev(c):
    out = {k: torch.from_numpy(np.ascontiguousarray(c[k])).to(DEV) for k in ('id', 'exp', 'src_euler', 'src_trans', 'src_exp')}
    out['pose'] = None if c['pose'] is None else tuple(torch.from_numpy(x).to(DEV) for x in c['pose'])
    return out


def _run(cm, d, mp=True, **kw):
    return cm.clip(d['id'], d['exp'], d['src_euler'], d['src_trans'], d['src_exp'], pose=d['pose'], map_to_init_pose=mp, **kw)


def _check(got, want, dev, what):
    for g, w, r, name in zip(got, want, dev, NAMES):
        g = g.double().cpu().numpy()
        assert g.shape == w.shape and np.isfinite(g).all()
        bar = 2 * r + 4 * np.spacing(np.float32(np.abs(w).max()))
        err = np.abs(g - w).max()
        print(f'{what} {name}: max |err| {err:.2e}, bar {bar:.2e}')
        assert err <= bar, (what, name, err, bar)


@pytest.mark.parametrize('T,P,mp', [(3, 0, True), (4, 1, True), (7, 20, False), (8, 20, True), (250, 20, True), (250, 300, False),
                                    (15000, 300, True), (15000, 0, True)])
def test_against_float64(bfm, T, P, mp):
    _, m, cm = bfm
    c = mref.make_case(T, P, seed=100 + T + P)
    want = mref.clip(m, c['id'], c['exp'], c['src_euler'], c['src_trans'], c['src_exp'], c['pose'], mp)
    got = _run(cm, _dev(c), mp)
    torch.cuda.synchronize()
    _check(got, want, mref.REF_DEV, f'T={T} P={P}')
    assert (got[1][..., 2] == 0).all() and (got[2][..., 2] == 0).all()


def test_against_the_reference_fixture(bfm, golden):
    _, m, cm = bfm
    z = golden('motion_small')
    k = 0
    while f'c{k}_meta' in z:
        pre = f'c{k}_'
        T, P, mp = (int(v) for v in z[pre + 'meta'])
        c = {n: z[pre + n].numpy() for n in ('id', 'exp', 'src_euler', 'src_trans', 'src_exp')}
        c['pose'] = None if P == 0 else (z[pre + 'pose_euler'].numpy(), z[pre + 'pose_trans'].numpy())
        dev = z[pre + 'dev'].numpy()
        got = _run(cm, _dev(c), bool(mp))
        want = mref.clip(m, c['id'], c['exp'], c['src_euler'], c['src_trans'], c['src_exp'], c['pose'], bool(mp))
        _check(got, want, dev, f'fixture case {k}')
        # and the reference's float32 outputs: both within their bars of float64
        for g, n, r in zip(got, NAMES, dev):
            ref = z[pre + n].double().numpy()
            assert np.abs(g.double().cpu().numpy() - ref).max() <= 3 * r + 4 * np.spacing(np.float32(np.abs(ref).max()))
        k += 1
    assert k >= 10


def test_strided_and_broadcast_inputs_are_read_in_place(bfm):
    _, _, cm = bfm
    T = 57
    d = _dev(mref.make_case(T, 20, seed=5))
    rows = torch.randn(T, 146, device=DEV)
    rows[:, :80] = d['id']
    rows[:, 80:144] = d['exp']
    base = _run(cm, d)
    strided = _run(cm, dict(d, exp=rows[:, 80:144], id=rows[:, :80]))
    per_frame = _run(cm, dict(d, id=d['id'].expand(T, 80).contiguous()))
    torch.cuda.synchronize()
    for a, b, c in zip(base, strided, per_frame):
        assert torch.equal(a, b) and torch.equal(a, c)


@torch.no_grad()
def test_out_and_graph_capture(bfm):
    _, _, cm = bfm
    T = 40
    d = _dev(mref.make_case(T, 30, seed=6))
    out = (torch.full((T, 25), float('nan'), device=DEV), torch.full((1, 68, 3), float('nan'), device=DEV),
           torch.full((T, 68, 3), float('nan'), device=DEV))
    ret = _run(cm, d, out=out)
    assert all(r is o for r, o in zip(ret, out))
    eager = _run(cm, d)
    assert all(torch.equal(a, b) for a, b in zip(out, eager))
    # capture with static inputs, replay after new inputs are copied in
    s = {k: (v.clone() if isinstance(v, torch.Tensor) else tuple(x.clone() for x in v)) for k, v in d.items()}
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _run(cm, s, out=out)                                           # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        _run(cm, s, out=out)
    d2 = _dev(mref.make_case(T, 30, seed=7))
    for k in ('id', 'exp', 'src_euler', 'src_trans', 'src_exp'):
        s[k].copy_(d2[k])
    for a, b in zip(s['pose'], d2['pose']):
        a.copy_(b)
    for o in out:
        o.fill_(float('nan'))
    g.replay()
    want = _run(cm, d2)
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(out, want))


def test_vertex_pass_frame_split_is_exact(bfm):
    """A 15 000-frame call splits its frames over blockIdx.y; one-tile calls do not split: the same bits."""
    _, _, cm = bfm
    T = 15000
    d = _dev(mref.make_case(T, 0, seed=8))
    g = torch.Generator().manual_seed(8)
    e, t = ((torch.rand(T, 3, generator=g) - 0.5).to(DEV), (0.3 * torch.randn(T, 3, generator=g)).to(DEV))
    whole = torch.empty(T, 68, 4, device=DEV)
    cm._vertices(d['id'], 0, d['exp'], 64, e.contiguous(), t.contiguous(), T, whole)
    parts = torch.empty(T, 68, 4, device=DEV)
    for i in range(0, T, 32):
        n = min(32, T - i)
        cm._vertices(d['id'], 0, d['exp'][i:], 64, e[i:i + n].contiguous(), t[i:i + n].contiguous(), n, parts[i:i + n])
    torch.cuda.synchronize()
    assert torch.equal(whole, parts)


def test_reconstruct_lm2d(bfm):
    _, m, cm = bfm
    c = mref.make_case(20, 0, seed=9)
    e = np.repeat(c['src_euler'], 20, 0) + np.linspace(-0.3, 0.3, 20)[:, None].astype(np.float32)
    t = np.repeat(c['src_trans'], 20, 0)
    ident = np.repeat(c['id'], 20, 0)
    got = cm.reconstruct_lm2d(*(torch.from_numpy(np.ascontiguousarray(x)).to(DEV) for x in (ident, c['exp'], e, t)))
    want = mref.lm2d(m, ident, c['exp'], e.astype(np.float64), t.astype(np.float64))
    err = np.abs(got.double().cpu().numpy() - want).max()
    print(f'reconstruct_lm2d: max |err| {err:.2e}')
    assert got.shape == (20, 68, 2) and err <= mref.REF_DEV[1] + 4 * np.spacing(np.float32(np.abs(want).max()))
    got3 = cm.reconstruct_lm2d(*(torch.from_numpy(np.ascontiguousarray(x)).to(DEV).reshape(4, 5, -1) for x in (ident, c['exp'], e, t)))
    assert torch.equal(got3.reshape(20, 68, 2), got)


@torch.no_grad()
def test_torso_engine_driven_by_clip_motion(bfm):
    """begin_clip(kp_s) and prepare() tuples holding slices of ClipMotion's outputs render the frames of the same engine fed clones."""
    kw, _, cm = bfm
    r = r3.SECC_Renderer(512, device=DEV, bfm_folder=kw['bfm_folder'], ncc_path=kw['ncc_path'], eye_faces=kw['eye_faces'])
    B, T = 2, 6
    c = mref.make_case(T, 20, seed=11)
    d = _dev(c)
    rows = torch.cat([d['id'].expand(T, 80), d['exp']], 1).contiguous()
    cams, kp_s, kp_d = cm.clip(rows[:1, :80], rows[:, 80:144], d['src_euler'], d['src_trans'], d['src_exp'], pose=d['pose'])
    hp = dict(syn.WARP_HPARAMS, htbsr_head_weight_fuse_mode='v2', num_samples_fine=48, neural_rendering_resolution=64)
    inp = syn.make_warp_inputs(1, seed=3)
    frames = []
    for clone in (False, True):
        bb = r3.SegFormerSECC2PlaneBackbone()
        bb.load_state_dict(s2p_ref.make_params({k: v.shape for k, v in bb.state_dict().items()}, 7), strict=True)
        eng = engine.FrameEngine(batch=B, sr_mode='tc', hp=hp, torso_model=syn.StubTorsoModel(), out_uint8=True, secc2plane=bb.to(DEV).eval(),
                                 secc_renderer=r)
        eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_warp_params(seed=6, fuse_mode='v2'))
        ks = kp_s.clone() if clone else kp_s
        eng.begin_clip(inp['ref_torso_rgb'].to(DEV), inp['ref_bg_rgb'].to(DEV), inp['segmap'].to(DEV), ks)
        eng.begin_planes(syn.make_planes(1, seed=1).to(DEV), coeff_src=rows[:1].clone())
        items = []
        for s in range(T // B):
            sl = slice(s * B, (s + 1) * B)
            u_c, u_f = syn.make_jitter(B, 64 * 64, 48, 48, seed=70 + s)
            cam, kd, co = cams[sl], kp_d[sl], rows[sl]
            if clone:
                cam, kd, co = cam.clone(), kd.clone(), co.clone()
            items.append((co, cam, u_c.to(DEV), u_f.to(DEV), kd))
        if not clone:
            assert eng.prepare(items) == len(items)
        frames.append(torch.stack([eng.step(None, *it[1:4], kp_d=it[4], coeff=it[0]).clone() for it in items]))
    assert torch.equal(frames[0], frames[1])
    assert frames[0].float().std() > 0
