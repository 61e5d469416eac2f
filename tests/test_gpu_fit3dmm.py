"""Fit3DMM on the GPU against the float64 restatement (tests/fit_reference.py) and the reference's fixture.  Bar per output: 2 x the
reference's own float32 deviation from float64 plus 4 fp32 ulp of the output's largest magnitude (the fixture's deviation per case; for
the long clips, the deviation of the restatement run in float32 on the same landmarks).  Also: one r3dp_fit_grad + r3dp_fit_adam at random
parameters against the float64 autograd gradient, bit-identical reruns, out= with a strided exp, CUDA-graph replay, and the fits feeding
ClipMotion.clip in place."""
import numpy as np
import pytest
import torch

import fit_reference as fref
import real3dportrait_b200 as r3
from real3dportrait_b200 import _capi as capi, synthetic as syn
from real3dportrait_b200.fit3dmm import CHUNKS, MAX_CTAS, N_ID, ROW

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
NAMES = ('id', 'exp', 'euler', 'trans')


@pytest.fixture(scope='module')
def bfm(tmp_path_factory):
    d = syn.write_bfm_folder(str(tmp_path_factory.mktemp('bfm')), seed=0, mp468=True)['bfm_folder']
    return d, fref.load(d), r3.Fit3DMM(d, device=DEV)


def _fit(f, lms, video, **kw):
    x = torch.from_numpy(np.ascontiguousarray(lms)).to(DEV)
    return f.fit_video(x, **kw) if video else f.fit_image(x[0], **kw)


def _check(got, want, dev, what, vs='float64', k=2.0):
    for i, n in enumerate(NAMES):
        g = got[n].double().cpu().numpy()
        w = np.asarray(want[n], np.float64)
        assert g.shape == w.shape and np.isfinite(g).all()
        bar = k * dev[i] + 4 * np.spacing(np.float32(np.abs(w).max()))
        err = np.abs(g - w).max()
        print(f'{what} {n} vs {vs}: max |err| {err:.2e}, bar {bar:.2e}')
        assert err <= bar, (what, n, err, bar)


@pytest.mark.parametrize('k', range(7))
def test_fixture(golden, bfm, k):
    """Every fixture case against float64 (2 x dev + 4 ulp) and against the reference's own outputs (3 x dev + 4 ulp: the two float32
    results each sit within their deviation of float64)."""
    _, m, f = bfm
    z = golden('fit_small')
    pre = f'c{k}_'
    T, video = (int(v) for v in z[pre + 'meta'][:2])
    lms = z[pre + 'lms'].numpy()
    dev = z[pre + 'dev'].numpy()
    got = _fit(f, lms, bool(video))
    _check(got, fref.fit(m, lms, 512, video=bool(video)), dev, f'case {k} T={T} video={video}')
    ref = {n: z[pre + n].numpy() for n in NAMES}
    _check(got, ref, 1.5 * dev, f'case {k} T={T} video={video}', vs='reference', k=2.0)


def test_fixture_cases_are_all_listed(golden):
    assert 'c6_meta' in golden('fit_small') and 'c7_meta' not in golden('fit_small')


@pytest.mark.parametrize('T', [3, 130, 1500, 15000])
def test_long_clips_against_float64(bfm, T):
    _, m, f = bfm
    lms, _ = fref.make_landmarks(m, T, seed=1000 + T)
    got = _fit(f, lms, True)
    want = fref.fit(m, lms, 512, video=True, device=DEV)
    f32 = fref.fit(m, lms, 512, video=True, device=DEV, dtype=torch.float32)
    dev = [np.abs(f32[n].astype(np.float64) - want[n]).max() for n in NAMES]
    _check(got, want, dev, f'T={T}')


def _launch(f, lms, x, video, stage):
    """One r3dp_fit_grad + r3dp_fit_adam at parameters x [80 + 70 T] (fp64) -> the gradient the Adam step used."""
    T, L = lms.shape[0], lms.shape[1]
    p, st = capi.ptr, capi.stream()
    pf = torch.empty(CHUNKS * T * 12, device=DEV, dtype=torch.float64)
    pe = torch.empty(CHUNKS * T * 64, device=DEV)
    pi = torch.empty(CHUNKS * MAX_CTAS * N_ID, device=DEV, dtype=torch.float64)
    xn, m, v, g = (torch.zeros_like(x) for _ in range(4))
    lam = (0.2, 0.6, 1.0) if video else (0.3, 0.05, 0.0)
    w = f.w_video if video else f.w_image
    L_ = capi.lib()
    d = lambda t: p(t, torch.float64)  # noqa: E731
    capi.check(L_.r3dp_fit_grad(p(f.basis), p(f.mean_shape), p(w), p(lms), T, L, 512, d(x), stage, d(pf), p(pe), d(pi), st))
    capi.check(L_.r3dp_fit_adam(d(pf), p(pe), d(pi), T, 5, 0 if stage == 1 else 3, 0.1, *lam, d(x), d(xn), d(m), d(v), d(g), st))
    return g.cpu().double().numpy()


@pytest.mark.parametrize('T,video,stage', [(1, False, 2), (1, True, 2), (70, True, 2), (130, True, 2), (1100, True, 2),
                                           (15000, True, 2), (70, True, 1)])
def test_one_launch_against_autograd(bfm, T, video, stage):
    """A partial frame tile (70 = 64 + 6), more tiles than CTAs (1 100 and 15 000 frames), T = 1, stage 1; the last chunk's 44 padded rows
    always."""
    _, m, f = bfm
    lms, truth = fref.make_landmarks(m, T, seed=7 + T)
    rng = np.random.default_rng(T)
    id_ = truth['id'] + rng.normal(size=(1, 80)) * 0.3
    exp = truth['exp'] + rng.normal(size=(T, 64)) * 0.3
    euler = truth['euler'] + rng.normal(size=(T, 3)) * 0.05
    trans = truth['trans'] + rng.normal(size=(T, 3)) * 0.05
    if stage == 1:
        id_, exp = np.zeros_like(id_), np.zeros_like(exp)
    x32 = [a.astype(np.float32) for a in (id_, exp, euler, trans)]
    x = np.concatenate([x32[0].reshape(-1), np.concatenate(x32[1:], 1).reshape(-1)])
    g = _launch(f, torch.from_numpy(lms).to(DEV), torch.from_numpy(x).to(DEV).double(), video, stage)
    want = fref.gradient(m, lms, *x32, video=video, stage=stage)
    rows = g[N_ID:].reshape(T, ROW)
    got = (g[:N_ID].reshape(1, -1), rows[:, :64], rows[:, 64:67], rows[:, 67:])
    for n, a, b in zip(NAMES, got, want):
        if stage == 1 and n in ('id', 'exp'):
            continue
        err, scale = np.abs(a - b).max(), np.abs(b).max()
        print(f'T={T} video={video} stage={stage} d{n}: max |err| {err:.2e}, max |grad| {scale:.2e}')
        assert err <= 2e-5 * scale + 1e-12, (n, err, scale)


def test_rerun_out_graph_and_clip_motion(bfm, tmp_path):
    d, m, f = bfm
    T = 90
    lms, _ = fref.make_landmarks(m, T, seed=3)
    x = torch.from_numpy(lms).to(DEV)
    a, b = f.fit_video(x), f.fit_video(x)
    for n in NAMES:
        assert torch.equal(a[n], b[n]), n
    # out= with the engine's rows: exp written into the column slice, the other columns untouched
    rows = torch.full((T, 150), 7.0, device=DEV)
    out = {'id': torch.empty(1, 80, device=DEV), 'exp': rows[:, 80:144], 'euler': torch.empty(T, 3, device=DEV),
           'trans': torch.empty(T, 3, device=DEV)}
    r = f.fit_video(x, out=out)
    assert all(r[n] is out[n] for n in NAMES)
    for n in NAMES:
        assert torch.equal(out[n], a[n]), n
    assert (rows[:, :80] == 7).all() and (rows[:, 144:] == 7).all()
    # graph capture, replay after new landmarks are copied in
    static = x.clone()
    gout = {k: torch.empty_like(v, memory_format=torch.contiguous_format) for k, v in a.items()}
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        f.fit_video(static, out=gout)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        f.fit_video(static, out=gout)
    lms2, _ = fref.make_landmarks(m, T, seed=4)
    static.copy_(torch.from_numpy(lms2))
    g.replay()
    want = f.fit_video(torch.from_numpy(lms2).to(DEV))
    for n in NAMES:
        assert torch.equal(gout[n], want[n]), n
    # the source fit and the driving pose feed ClipMotion.clip in place, as clones do
    cm = r3.ClipMotion(d, device=DEV)
    src = f.fit_image(x[0])
    got = cm.clip(src['id'], rows[:, 80:144], src['euler'], src['trans'], src['exp'], pose=(out['euler'], out['trans']))
    ref = cm.clip(src['id'].clone(), rows[:, 80:144].clone(), src['euler'].clone(), src['trans'].clone(), src['exp'].clone(),
                  pose=(out['euler'].clone(), out['trans'].clone()))
    for u, v in zip(got, ref):
        assert torch.equal(u, v)
