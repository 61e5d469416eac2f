"""Every r3dp_mf_* / r3dp_tw_* launch of the torso warper with torso_motion='cuda' and torso_stage2='cuda' (torso_warp.motion, stage2,
hid_to_nchw) at its exact arguments against float64, and a recorded-launch check that keeps these tables equal to what the warper launches.

* The rows come from torso_warper_ref.launch_plan over torso_kp_num K = 4 and 9, `tc` and `tc_exact` (split), and N = 4 frames reading the
  per-clip volume, N = 4 frames with a volume each, and N = 1: one row per distinct launch.
* r3dp_mf_conv3d: the weights come from the module's own packers (pack_conv3d, compose_nearest_up3d, the fuser's channel map), so the padded
  cop rows are the module's.  The bound is sr_conv_reference's |got - ref| <= alpha |ref| + extra + beta S with
  torso_motion_reference.BETA3.  Every output sits between sentinel guards: each element of [yc0, yc0 + cout) of every voxel (and of its lo
  half) is written, nothing else is.  The last image of an N = 4 launch equals its N = 1 launch bit for bit.
* The kernels around the convolutions and r3dp_tw_affine_relu: the bounds derived in tests/torso_motion_reference.py, inside the same
  guards (the fp32 outputs inside NaN guards).  Stage 2's r3dp_tw_conv, _conv_up_nearest, _narrow_conv, _gather3d and _hid_to_nchw: the
  run_* helpers of tests/test_gpu_torso_warper_layers.py at each launch's arguments.
* Every comparison runs one frame at a time, which bounds the float64 memory (the 7^3 fuser at N = 4).
* test_warper_launches_have_rows records one eager step of FrameEngine(batch=4) with the reference's warper (K = 4 and 9, `tc` and
  `tc_exact`), requires the recorded calls to equal launch_plan, fails naming a launch without a row, and fails when a row of the
  recorded plans is no longer launched."""
import pytest
import torch

from real3dportrait_b200 import _capi as capi, torso_warp as tw
import sr_conv_reference as scr
import test_gpu_torso_warper_layers as twl
import torso_motion_reference as tmr
import torso_warper_ref as twr
from launch_harness import (Recorder, assert_plan, assert_rows, assert_written, call_signature, conv3d, guarded, inside, join, split_store)
from torso_motion_reference import BETA3, ref_conv

pytestmark = pytest.mark.gpu
DEV = 'cuda'
F16, F32 = torch.float16, torch.float32
#: (K, N, split, clip) of the plans the tables cover; the N = 4 per-clip ones are what test_warper_launches_have_rows records
PLANS = [(K, N, sp, clip) for K in (4, 9) for sp in (0, 1) for N, clip in ((4, True), (4, False), (1, True))]
RECORDED = [p for p in PLANS if p[1] == 4 and p[3]]
#: the argument positions of the pointers that may be NULL (torso_warper_ref.OPTIONAL_OPERANDS), per entry point
OPTIONAL_POS = {'r3dp_mf_conv3d': (6,), 'r3dp_tw_conv': (10,), 'r3dp_tw_narrow_conv': (0, 4, 7)}


def _prefix(K, N, split, clip):
    """The tag prefix of a plan's rows: 'own' marks frames with a volume each."""
    return f'K{K}-N{N}{"" if clip else "own"}-{"tcx" if split else "tc"}-'


def _rows(fn):
    """{signature: (K, tag)} of one entry point over PLANS, the first (K, tag) of each distinct launch."""
    out = {}
    for K, N, sp, clip in PLANS:
        for tag, f, a in twr.launch_plan(K, N, sp, clip):
            if f == fn:
                out.setdefault(twr.launch_signature(f, a), (K, _prefix(K, N, sp, clip) + tag))
    return out


ROWS = {fn: _rows(fn) for fn in ('r3dp_mf_conv3d', 'r3dp_mf_input', 'r3dp_mf_pool', 'r3dp_mf_head_input', 'r3dp_mf_head_bcast', 'r3dp_mf_deform',
                                 'r3dp_mf_occlusion', 'r3dp_tw_affine_relu', 'r3dp_tw_gather3d', 'r3dp_tw_conv', 'r3dp_tw_conv_up_nearest',
                                 'r3dp_tw_narrow_conv', 'r3dp_tw_hid_to_nchw')}


def _keys(fn):
    return list(ROWS[fn])


def _ids(fn):
    return [ROWS[fn][k][1] for k in ROWS[fn]]


# ---- r3dp_mf_conv3d ----------------------------------------------------------------------------------------------------------------------
def _conv3d_weights(K, tag, cin, O, taps, up, split, g):
    """The module's packing of seeded float64 weights for the layer `tag` (the logical input channels and their map as MotionWeights has
    them).  -> pack_conv3d's (packed fp16, fp32 bias, O, cop)."""
    c0 = (K + 1) * 5
    P0 = (c0 + 31) // 32 * 32
    name = tag.rsplit('-', 1)[-1]
    cin_map = None
    if name == 'mf.down.0':
        I = c0
    elif name == 'mf.fuser':
        I, cin_map = c0 + 64, list(range(c0)) + [P0 + i for i in range(64)]
    elif name == 'mf.enc.0':
        I = 4
    else:
        I = cin
    kd, kh, kw = taps
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV, dtype=torch.float64)      # noqa: E731
    if up:
        w = tw.compose_nearest_up3d(rn(O, I, 3, 3, 3) / (27 * I) ** 0.5)
    else:
        w = (rn(O, I, kd, kh, kw) / (kd * kh * kw * I) ** 0.5)[None]
    return tw.pack_conv3d(w, 0.1 * rn(O), cin, bool(split), cin_map=cin_map)


@torch.no_grad()
@pytest.mark.parametrize('key', _keys('r3dp_mf_conv3d'), ids=_ids('r3dp_mf_conv3d'))
def test_conv3d_launch(key):
    K, tag = ROWS['r3dp_mf_conv3d'][key]
    a = key[1]
    xs, xlo, cin, N, D, H, W, kd, kh, kw, up, O, cop, relu, ys, yc0, ylo, out_f32, split, res = a
    split = bool(split)
    g = torch.Generator(device=DEV).manual_seed(_keys('r3dp_mf_conv3d').index(key) + 700)
    wp, bias, O_mod, cop_mod = _conv3d_weights(K, tag, cin, O, (kd, kh, kw), up, split, g)
    assert (O_mod, cop_mod) == (O, cop), (tag, O_mod, cop_mod)                 # the module's packing pads to the launch's cop
    x = split_store(torch.randn(N, D, H, W, xlo, generator=g, device=DEV), xs, xlo, split)
    Ho, Wo = (2 * H, 2 * W) if up else (H, W)
    M = N * D * Ho * Wo
    r16 = split_store(torch.randn(N, D, Ho, Wo, O, generator=g, device=DEV), ys, ylo, split, yc0) if res else None   # the output's layout
    dt = F32 if out_f32 else F16
    buf, y = guarded(M * ys, dt, device=DEV)
    conv3d(a, x, wp, bias, r16, y)
    mask = inside(ys, yc0, O, ylo, split and not out_f32, device=DEV)
    assert_written(buf, y, ys, mask, tag)
    y = y.view(N, D, Ho, Wo, ys)
    wd = ((wp[..., :cin].double() + wp[..., cin:].double()) / 1024.0 if split else wp.double())[:, :, :O]
    alpha = scr.ALPHA_F32 if out_f32 else scr.alpha_store(split)
    for n in range(N):
        xin = join(x[n:n + 1], 0, cin, xlo, split).permute(0, 4, 1, 2, 3)
        pre = ref_conv(xin, wd, (kd, kh, kw), up, bias[:O])
        S = ref_conv(xin.abs(), wd.abs(), (kd, kh, kw), up, bias[:O].abs())
        ref = torch.relu(pre) if relu else pre
        extra = 0.0 if out_f32 else 2 * scr.FLOOR_F16
        if res:
            rv = join(r16[n:n + 1], yc0, O, ylo, split).permute(0, 4, 1, 2, 3)
            ref, S = ref + rv, S + rv.abs()
            if not split:                                                      # tc rounds the activated value to fp16 before the add
                extra = extra + scr.ALPHA_F16 * pre.abs()
        got = (y[n:n + 1, ..., yc0:yc0 + O].double() if out_f32 else join(y[n:n + 1], yc0, O, ylo, split)).permute(0, 4, 1, 2, 3)
        scr.check_bound(got, ref, S, alpha, BETA3[split], extra, tag=f'{tag} image {n}')
    if N > 1:
        _, one = guarded(D * Ho * Wo * ys, dt, device=DEV)
        conv3d(a, x[N - 1:].contiguous(), wp, bias, None if r16 is None else r16[N - 1:].contiguous(), one, N=1)
        assert torch.equal(one.view(-1, ys)[:, mask], y[N - 1].reshape(-1, ys)[:, mask]), f'{tag}: last image vs its N=1 launch'


# ---- the kernels around the convolutions ------------------------------------------------------------------------------------------------
def _kp(N, K, g):
    return [(0.9 * (2 * torch.rand(N, K, 3, generator=g, device=DEV) - 1)) for _ in range(2)]


@torch.no_grad()
@pytest.mark.parametrize('key', _keys('r3dp_mf_input'), ids=_ids('r3dp_mf_input'))
def test_mf_input_launch(key):
    _, tag = ROWS['r3dp_mf_input'][key]
    shared, N, K, D, H, W, cpad, ys, ylo, split = key[1]
    g = torch.Generator(device=DEV).manual_seed(11 + K + N + shared)
    fc = torch.randn(1 if shared else N, D, H, W, 4, generator=g, device=DEV)
    kp_s, kp_d = _kp(N, K, g)
    buf, y = guarded(N * D * H * W * ys, F16, device=DEV)
    capi.check(capi.lib().r3dp_mf_input(capi.ptr(fc), shared, capi.ptr(kp_s), capi.ptr(kp_d), N, K, D, H, W, cpad, capi.ptr(y, F16), ys, ylo, split,
                                        capi.stream()))
    assert_written(buf, y, ys, inside(ys, 0, cpad, ylo, split, device=DEV), tag)
    y = y.view(N, D, H, W, ys)
    c0 = (K + 1) * 5
    for n in range(N):
        ref, S, extra = tmr.mf_input(fc[0 if shared else n].double(), kp_s[n].double(), kp_d[n].double())
        got = join(y[n], 0, c0, ylo, split)
        scr.check_bound(got, ref, S, scr.alpha_store(split), tmr.BETA_SAMPLE, extra * (1 + 2.0 ** -10) + scr.FLOOR_F16, tag=f'{tag} frame {n}')
        assert bool((y[n, ..., c0:cpad] == 0).all()) and (not split or bool((y[n, ..., ylo + c0:ylo + cpad] == 0).all())), f'{tag}: pad channels'


@torch.no_grad()
@pytest.mark.parametrize('key', _keys('r3dp_mf_pool'), ids=_ids('r3dp_mf_pool'))
def test_mf_pool_launch(key):
    _, tag = ROWS['r3dp_mf_pool'][key]
    N, D, H, W, C, xs, xlo, ys, ylo, split = key[1]
    g = torch.Generator(device=DEV).manual_seed(C + H + N)
    x = split_store(3 * torch.randn(N, D, 2 * H, 2 * W, C, generator=g, device=DEV), xs, xlo, split)
    buf, y = guarded(N * D * H * W * ys, F16, device=DEV)
    capi.check(capi.lib().r3dp_mf_pool(capi.ptr(x, F16), N, D, H, W, C, xs, xlo, capi.ptr(y, F16), ys, ylo, split, capi.stream()))
    assert_written(buf, y, ys, inside(ys, 0, C, ylo, split, device=DEV), tag)
    y = y.view(N, D, H, W, ys)
    for n in range(N):
        ref, S = tmr.pool(join(x[n], 0, C, xlo, split))
        scr.check_bound(join(y[n], 0, C, ylo, split), ref, S, scr.alpha_store(split), tmr.BETA_POOL, scr.FLOOR_F16, tag=f'{tag} frame {n}')


@torch.no_grad()
@pytest.mark.parametrize('key', _keys('r3dp_mf_head_input'), ids=_ids('r3dp_mf_head_input'))
def test_mf_head_input_launch(key):
    _, tag = ROWS['r3dp_mf_head_input'][key]
    N, H, W, cpad, ys, ylo, split = key[1]
    g = torch.Generator(device=DEV).manual_seed(5 + N)
    rgb = 2 * torch.rand(N, 3, 2 * H, 2 * W, generator=g, device=DEV) - 1
    wt = torch.rand(N, 1, 2 * H, 2 * W, generator=g, device=DEV)
    buf, y = guarded(N * H * W * ys, F16, device=DEV)
    capi.check(capi.lib().r3dp_mf_head_input(capi.ptr(rgb), capi.ptr(wt), N, H, W, cpad, capi.ptr(y, F16), ys, ylo, split, capi.stream()))
    assert_written(buf, y, ys, inside(ys, 0, cpad, ylo, split, device=DEV), tag)
    y = y.view(N, H, W, ys)
    for n in range(N):
        ref, S = tmr.head_input(rgb[n:n + 1].double(), wt[n:n + 1].double())
        scr.check_bound(join(y[n:n + 1], 0, 4, ylo, split), ref, S, scr.alpha_store(split), tmr.BETA_HEAD_INPUT, scr.FLOOR_F16, tag=f'{tag} frame {n}')
        assert bool((y[n, ..., 4:cpad] == 0).all()) and (not split or bool((y[n, ..., ylo + 4:ylo + cpad] == 0).all())), f'{tag}: pad channels'


@torch.no_grad()
@pytest.mark.parametrize('key', _keys('r3dp_mf_head_bcast'), ids=_ids('r3dp_mf_head_bcast'))
def test_mf_head_bcast_launch(key):
    _, tag = ROWS['r3dp_mf_head_bcast'][key]
    N, D, H, W, C, xs, xlo, ys, yc0, ylo, split = key[1]
    g = torch.Generator(device=DEV).manual_seed(7 + N + ys)
    x = split_store(torch.randn(N, 2 * H, 2 * W, C, generator=g, device=DEV), xs, xlo, split)
    buf, y = guarded(N * D * H * W * ys, F16, device=DEV)
    capi.check(capi.lib().r3dp_mf_head_bcast(capi.ptr(x, F16), N, D, H, W, C, xs, xlo, capi.ptr(y, F16), ys, yc0, ylo, split, capi.stream()))
    assert_written(buf, y, ys, inside(ys, yc0, C, ylo, split, device=DEV), tag)
    y = y.view(N, D, H, W, ys)
    for n in range(N):
        ref, S = tmr.pool(join(x[n], 0, C, xlo, split))
        got = join(y[n], yc0, C, ylo, split)
        scr.check_bound(got, ref.expand(D, -1, -1, -1), S.expand(D, -1, -1, -1), scr.alpha_store(split), tmr.BETA_POOL, scr.FLOOR_F16,
                        tag=f'{tag} frame {n}')


@torch.no_grad()
@pytest.mark.parametrize('key', _keys('r3dp_mf_deform'), ids=_ids('r3dp_mf_deform'))
def test_mf_deform_launch(key):
    _, tag = ROWS['r3dp_mf_deform'][key]
    ls, N, K, D, H, W = key[1]
    g = torch.Generator(device=DEV).manual_seed(13 + K + N)
    logits = torch.full((N, D, H, W, ls), float('nan'), device=DEV)          # the stride's pad logits are never read
    logits[..., :K + 1] = 3 * torch.randn(N, D, H, W, K + 1, generator=g, device=DEV)
    kp_s, kp_d = _kp(N, K, g)
    buf, y = guarded(N * D * H * W * 3, F32, device=DEV)
    capi.check(capi.lib().r3dp_mf_deform(capi.ptr(logits), ls, capi.ptr(kp_s), capi.ptr(kp_d), N, K, D, H, W, capi.ptr(y), capi.stream()))
    assert_written(buf, y, 3, torch.ones(3, dtype=torch.bool, device=DEV), tag)
    y = y.view(N, D, H, W, 3)
    for n in range(N):
        ref, S, extra = tmr.deform(logits[n, ..., :K + 1].double(), kp_s[n].double(), kp_d[n].double())
        scr.check_bound(y[n], ref, S, 0.0, scr.gamma(K + 2), extra, tag=f'{tag} frame {n}')


@torch.no_grad()
@pytest.mark.parametrize('key', _keys('r3dp_mf_occlusion'), ids=_ids('r3dp_mf_occlusion'))
def test_mf_occlusion_launch(key):
    _, tag = ROWS['r3dp_mf_occlusion'][key]
    N, D, H, W, C, xs, xlo, split = key[1]
    g = torch.Generator(device=DEV).manual_seed(17 + N + split)
    x = split_store(torch.randn(N, D, H, W, C, generator=g, device=DEV), xs, xlo, split)
    wk = (torch.randn(D, 49, C, 2, generator=g, device=DEV) / (D * 49 * C) ** 0.5 * 3).contiguous()
    bk = 0.1 * torch.randn(2, generator=g, device=DEV)
    outs = [guarded(N * H * W, F32, device=DEV) for _ in range(2)]
    capi.check(capi.lib().r3dp_mf_occlusion(capi.ptr(x, F16), N, D, H, W, C, xs, xlo, split, capi.ptr(wk), capi.ptr(bk), capi.ptr(outs[0][1]),
                                            capi.ptr(outs[1][1]), capi.stream()))
    for buf, o in outs:
        assert_written(buf, o, 1, torch.ones(1, dtype=torch.bool, device=DEV), tag)
    for n in range(N):
        bounds = tmr.occlusion(join(x[n], 0, C, xlo, split), wk, bk, split)
        for (_, o), (ref, S, extra) in zip(outs, bounds):
            scr.check_bound(o.view(N, H, W)[n], ref, S, 0.0, tmr.BETA_OCC, extra, tag=f'{tag} frame {n}')


@torch.no_grad()
@pytest.mark.parametrize('key', _keys('r3dp_tw_affine_relu'), ids=_ids('r3dp_tw_affine_relu'))
def test_tw_affine_relu_launch(key):
    _, tag = ROWS['r3dp_tw_affine_relu'][key]
    N, H, W, C, split = key[1]
    g = torch.Generator(device=DEV).manual_seed(19 + C + N)
    cs = C * (2 if split else 1)
    x = split_store(3 * torch.randn(N, H, W, C, generator=g, device=DEV), cs, C, split)
    s, t = 0.5 + torch.rand(C, generator=g, device=DEV), 0.3 * torch.randn(C, generator=g, device=DEV)
    buf, y = guarded(N * H * W * cs, F16, device=DEV)
    capi.check(capi.lib().r3dp_tw_affine_relu(capi.ptr(x, F16), capi.ptr(s), capi.ptr(t), N, H, W, C, split, capi.ptr(y, F16), capi.stream()))
    assert_written(buf, y, cs, inside(cs, 0, C, C, split, device=DEV), tag)
    y = y.view(N, H, W, cs)
    for n in range(N):
        ref, S = tmr.affine_relu(join(x[n], 0, C, C, split), s, t)
        scr.check_bound(join(y[n], 0, C, C, split), ref, S, scr.alpha_store(split), tmr.BETA_AFFINE, scr.FLOOR_F16, tag=f'{tag} frame {n}')


# ---- stage 2 at the warper's launches (the layer helpers of tests/test_gpu_torso_warper_layers.py) ----------------------------------------
@torch.no_grad()
@pytest.mark.parametrize('key', _keys('r3dp_tw_conv'), ids=_ids('r3dp_tw_conv'))
def test_tw_conv_launch(key):
    N, I, O, H, W, k, slope, split, res = key[1]
    twl.run_tw_conv((N, H, W, I, O, k, slope, res), bool(split))


@torch.no_grad()
@pytest.mark.parametrize('key', _keys('r3dp_tw_conv_up_nearest'), ids=_ids('r3dp_tw_conv_up_nearest'))
def test_tw_conv_up_nearest_launch(key):
    N, I, O, H, W, slope, split = key[1]
    twl.run_up_nearest((N, H, W, I, O, slope), bool(split))


def _narrow_case(a):
    """A narrow_conv launch -> (NARROW_CASES row, split, N) of tests/test_gpu_torso_warper_layers.py."""
    sa, ca, lo, sf, cf, eh, ew, N, H, W, K, CO, act, nchw, has_xa, has_xf, has_ex = a
    assert H == W == 256 and (not has_ex or (eh, ew) == (64, 64)) and (not has_xa or (ca, sa) == (64, 128 * (2 if lo else 1)))
    assert not has_xf or (sf, cf) == (32, 32)
    return (K, CO, act, 'f16' if has_xa else 'f32', has_ex, bool(nchw)), bool(lo), N


@torch.no_grad()
@pytest.mark.parametrize('key', _keys('r3dp_tw_narrow_conv'), ids=_ids('r3dp_tw_narrow_conv'))
def test_tw_narrow_conv_launch(key):
    case, split, N = _narrow_case(key[1])
    twl.run_narrow_conv(case, split, N)


@torch.no_grad()
@pytest.mark.parametrize('key', _keys('r3dp_tw_hid_to_nchw'), ids=_ids('r3dp_tw_hid_to_nchw'))
def test_tw_hid_to_nchw_launch(key):
    N, C, H, W, cs, lo = key[1]
    assert (C, H, W, cs) == (64, 256, 256, 256 if lo else 128) and lo in (0, 128)
    twl.run_hid_to_nchw(bool(lo), N)


@torch.no_grad()
@pytest.mark.parametrize('key', _keys('r3dp_tw_gather3d'), ids=_ids('r3dp_tw_gather3d'))
def test_tw_gather3d_launch(key):
    shared, N, C, D, H, W, split = key[1]
    assert (C, D, H, W) == (32, 16, 64, 64)
    twl.run_gather3d(bool(split), N, bool(shared))


# ---- the recorded launches ---------------------------------------------------------------------------------------------------------------
def _reference_warper(K, seed, monkeypatch):
    """The reference's WarpBasedTorsoModelMediaPipe('standard') built for torso_kp_num K: its constructor copies model2.py's global hparams
    (which ref_classes() sets to K = 4, so the class is looked up first)."""
    cls = twr.ref_classes()[1]
    from modules.real3d.facev2v_warp import model2
    with monkeypatch.context() as m:
        m.setitem(model2.hparams, 'torso_kp_num', K)
        torch.manual_seed(seed)
        warper = twr.randomize(cls('standard'), seed=seed).to(DEV)
    assert warper.hparams['torso_kp_num'] == K
    return warper


@torch.no_grad()
def test_warper_launches_have_rows(monkeypatch):
    if not twr.ref_classes():
        pytest.skip('the reference warper modules are not staged under oracle/_ref')
    from real3dportrait_b200 import engine, synthetic as syn
    B = 4
    mlp = syn.make_decoder_params(seed=4)
    inp = {k: v.to(DEV) for k, v in syn.make_warp_inputs(1, seed=8).items()}
    planes, cam = syn.make_planes(B, seed=0).to(DEV), syn.make_cameras(B, seed=1).to(DEV)
    kp_d = (torch.rand(B, 68, 3, generator=torch.Generator().manual_seed(2)) * 2 - 1).to(DEV)
    u_c, _ = syn.make_jitter(B, 4096, 48, 0, seed=3)
    launched, missing = set(), []
    for K, N, sp, clip in RECORDED:
        warper = _reference_warper(K, 41, monkeypatch)
        srp = syn.make_sr_warp_params(seed=6)
        srp.update({'torso_model.' + k: v for k, v in warper.state_dict().items()})
        eng = engine.FrameEngine(batch=B, sr_mode='tc_exact' if sp else 'tc', hp=dict(syn.WARP_HPARAMS, num_samples_fine=0, torso_kp_num=K),
                                 torso_model=warper, use_graph=False, torso_stage2='cuda', torso_motion='cuda')
        eng.load_params(mlp, srp)
        eng.begin_clip(inp['ref_torso_rgb'], inp['ref_bg_rgb'], inp['segmap'], inp['kp_s'])
        with Recorder(capi.lib(), lambda n: n.startswith(('r3dp_mf_', 'r3dp_tw_'))) as rec:
            eng.step(planes, cam, u_c.to(DEV), kp_d=kp_d)
            torch.cuda.synchronize()
        eng.end_clip()
        got = [call_signature(n, a, OPTIONAL_POS.get(n, ())) for n, a in rec.calls]
        plan = twr.launch_plan(K, N, sp, clip)
        where = f'K={K} N={N} {"tc_exact" if sp else "tc"}'
        assert_plan(got, [twr.launch_signature(f, a) for _, f, a in plan], where)
        missing += [f'{where}: {tag} {fn}{a}' for (tag, fn, a), s in zip(plan, got) if s not in ROWS.get(fn, {})]
        launched.update(got)
    stale = [f'{tag}: {key}' for fn, rows in ROWS.items() for key, (_, tag) in rows.items()
             if any(tag.startswith(_prefix(*p)) for p in RECORDED) and key not in launched]
    assert_rows(missing, stale, 'the warper')
