"""The fused render against float64 (tests/render_reference.py) at bars that tell the split-fp16 decoder from plain fp16, on every kernel
r3dp_render_ex can pick:
  path 0  the streaming kernel (render_stream.cu; single-pass renders),
  path 1  the CTA-per-ray-tile kernel with the wgmma decoder (render.cu; two-pass renders whose passes fit its tiles),
  path 2  the CTA-per-ray-tile kernel with the CUDA-core decoder (the other two-pass renders).
Every case asserts the path it is meant to cover (r3dp_render_path), and the module checks that all three were covered.

(a) decoder probe: rays along exactly (0, 0, -1) through a plane set whose planes 1 and 2 are zero give every sample of a ray the same
    features, so rgb = 2 c sum(w) - 1 up to the march's fp32 sums and c = (rgb + 1) / (2 sum w) is the decoded colour of that ray, checked
    element by element against decoder_bound.
(b) whole renders with opaque decoders against float64 at TAU_RGB / TAU_WSUM / TAU_DEPTH.
(c) stand-alone tri-plane / tri-grid sampling, decoder, run_model and ray marcher against float64 with element-wise bounds.
(d) every call: nothing outside the outputs is written and every output element is written (sentinel-filled allocations); frames are
    independent of each other and a repeated render gives the same bits."""
import ctypes as C

import pytest
import torch

from real3dportrait_b200 import _capi as capi
from real3dportrait_b200 import renderer as ren
from real3dportrait_b200 import synthetic as syn
import render_reference as rr

pytestmark = pytest.mark.gpu
DEV = 'cuda'
U = rr.U
SENT32 = 0x7FA5A5A5                       # a NaN payload no kernel produces
PAD = 1024


# ---- calling the renderer ---------------------------------------------------------------------------------------------------------------
def _canary(n, dtype):
    if dtype == torch.uint8:
        buf = torch.full((n + 2 * PAD,), 0xA5, dtype=torch.uint8, device=DEV)
    else:
        buf = torch.full((n + 2 * PAD,), SENT32, dtype=torch.int32, device=DEV).view(torch.float32)
    return buf, buf[PAD:PAD + n]


def _check_canary(buf, tag):
    b = buf.view(torch.int32) if buf.dtype == torch.float32 else buf
    s = SENT32 if buf.dtype == torch.float32 else 0xA5
    outside = torch.cat([b[:PAD], b[-PAD:]])
    assert bool((outside == s).all()), f'{tag}: written outside its output'
    inside = b[PAD:-PAD]
    if buf.dtype == torch.uint8:
        assert bool((inside <= 1).all()), f'{tag}: element not written'
    else:
        assert not bool((inside == s).any()), f'{tag}: element not written'


def render(planes, mlp, S, S_imp=0, *, o=None, d=None, camera=None, res=0, box=1.0, wb=False, u_c, u_f=None, depth=0, planes2=None,
           hwpc=False, path):
    """One r3dp_render_ex call with every output inside a sentinel-filled allocation; asserts the kernel it runs is `path`.
    Returns (rgb [N,M,32], depth [N,M,1], wsum [N,M,1], valid [N,M,1] bool) on the CPU."""
    N = planes.shape[0]
    M = res * res if camera is not None else o.shape[1]
    if depth > 0:
        pcl = ren.grids_to_channels_last(planes.to(DEV), depth)
    elif hwpc:
        pcl = ren.producer_view(planes.to(DEV).reshape(N, -1, *planes.shape[-2:]).contiguous(memory_format=torch.channels_last)
                                .view(planes.shape))
        assert pcl is not None and pcl.layout == 'hwpc'
    else:
        pcl = ren.planes_to_channels_last(planes.to(DEV))
    pcl2 = ren.planes_to_channels_last(planes2.to(DEV)) if planes2 is not None else None
    _, Cc, H, W = pcl.dims
    dec = {k: v.to(DEV).contiguous() for k, v in mlp.items()}
    m = capi.mlp_struct(dec['net.0.weight'], dec['net.0.bias'], dec['net.2.weight'], dec['net.2.bias'])
    bufs = [_canary(N * M * 32, torch.float32), _canary(N * M, torch.float32), _canary(N * M, torch.float32), _canary(N * M, torch.uint8)]
    (_, rgb), (_, dep), (_, wsum), (_, valid) = bufs
    L = capi.lib()
    ws_bytes = L.r3dp_render_workspace_bytes(N, M)
    ws = torch.empty(ws_bytes, device=DEV, dtype=torch.uint8)
    dev = lambda t: None if t is None else capi.f32(t.to(DEV))
    ro, rd, cam, uc, uf = dev(o), dev(d), dev(camera), dev(u_c), dev(u_f)
    g = capi.RenderArgs()
    g.planes, g.layout = capi.ptr(pcl.data).value, pcl.c_layout(N)
    if pcl2 is not None:
        g.planes2, g.layout2 = capi.ptr(pcl2.data).value, pcl2.c_layout(N)
    g.N, g.C, g.H, g.W, g.M, g.res, g.S, g.S_imp = N, Cc, H, W, M, res, S, S_imp
    g.ray_o, g.ray_d, g.camera = capi.ptr(ro).value, capi.ptr(rd).value, capi.ptr(cam).value
    g.box_warp, g.white_back = float(box), int(wb)
    g.u_coarse, g.u_fine, g.mlp = capi.ptr(uc).value, capi.ptr(uf).value, C.pointer(m)
    g.rgb, g.depth, g.weights_sum = capi.ptr(rgb).value, capi.ptr(dep).value, capi.ptr(wsum).value
    g.is_ray_valid, g.workspace, g.workspace_bytes = capi.ptr(valid, torch.uint8).value, capi.ptr(ws, torch.uint8).value, ws_bytes
    got_path = L.r3dp_render_path(C.byref(g))
    assert got_path == path, f'case meant for path {path} runs path {got_path}'
    capi.check(L.r3dp_render_ex(C.byref(g), capi.stream()))
    torch.cuda.synchronize()
    for (buf, _), tag in zip(bufs, ('rgb', 'depth', 'weights_sum', 'is_ray_valid')):
        _check_canary(buf, tag)
    return (rgb.view(N, M, 32).cpu(), dep.view(N, M, 1).cpu(), wsum.view(N, M, 1).cpu(), valid.view(N, M, 1).bool().cpu())


def camera_rays(camera, res):
    """The rays the kernels generate from `camera` (the same make_ray), for the float64 reference."""
    N = camera.shape[0]
    c2w, K = syn.split_camera(camera)
    c2w, K = capi.f32(c2w.to(DEV)), capi.f32(K.to(DEV))            # held: a freed temporary's block is handed to the next allocation
    o = torch.empty(N, res * res, 3, device=DEV)
    d = torch.empty_like(o)
    capi.check(capi.lib().r3dp_gen_rays(capi.ptr(c2w), capi.ptr(K), N, res, capi.ptr(o), capi.ptr(d), capi.stream()))
    return o.cpu(), d.cpu()


# ---- (a) decoder probe --------------------------------------------------------------------------------------------------------------------
PROBE_PATHS = [  # (id, S, S_imp, path)
    ('stream_d8', 13, 0, 0), ('tile_tc_two_pass', 12, 12, 1), ('tile_cuda_core', 33, 15, 2)]
WORST = {}


@pytest.mark.parametrize('scale', [1.0, 8.0, 1e-3])
@pytest.mark.parametrize('pid,S,S_imp,path', PROBE_PATHS, ids=[p[0] for p in PROBE_PATHS])
def test_decoder_probe_element_bound(pid, S, S_imp, path, scale):
    N, M = 1, 4096
    planes = rr.probe_planes(N, 64, 48, scale, seed=3)
    o, d = rr.probe_rays(N, M, seed=5)
    f, q, sg = rr.gather64(planes, o, 1.0)
    eg = rr.gather_bound(q, sg)
    g = torch.Generator().manual_seed(9)
    u_c = torch.rand(N, M, S, 1, generator=g)
    u_f = torch.rand(N * M, S_imp, generator=g) if S_imp else None
    worst = 0.0
    for name, mlp in rr.decoder_set():
        rgb, _, wsum, valid = render(planes, mlp, S, S_imp, o=o, d=d, res=64, u_c=u_c, u_f=u_f, path=path)
        assert bool(valid.all()) and float(wsum.min()) > 0.5
        c_got = ((rgb.double() + 1) / 2) / wsum.double()
        cref, _ = rr.decode64(f, mlp)
        ec, _ = rr.decoder_bound(f, mlp, eg, split=path != 2)
        march = 3 * (S + S_imp + 2) * U * cref.abs() + U / wsum.double()
        ratio = float(((c_got - cref).abs() / (ec + march)).max())
        worst = max(worst, ratio)
        assert ratio <= 1.0, (name, ratio)
    WORST[(pid, scale)] = worst
    print(f'probe {pid} x{scale}: worst error / bound = {worst:.3f}')


# ---- (b) whole renders vs float64 -----------------------------------------------------------------------------------------------------------
def _ragged(N, M, S, S_imp, H, W, seed, miss=True):
    g = torch.Generator().manual_seed(seed)
    planes = torch.randn(N, 3, 32, H, W, generator=g)
    o, d = rr.scatter_rays(N, M, seed + 1, miss=miss)
    u_c = torch.rand(N, M, S, 1, generator=g)
    u_f = torch.rand(N * M, S_imp, generator=g) if S_imp else None
    return planes, o, d, u_c, u_f


def _compare(got, ref, tau_rgb, tag):
    e_rgb, e_w = float((got[0].double() - ref[0]).abs().max()), float((got[2].double() - ref[2]).abs().max())
    e_d = float((got[1].double() - ref[1]).abs().max())
    print(f'{tag}: rgb {e_rgb:.2e} ({e_rgb / tau_rgb:.2f} tau), wsum {e_w:.2e}, depth {e_d:.2e}')
    assert torch.equal(got[3], ref[3]), tag
    assert e_rgb <= tau_rgb and e_w <= rr.TAU_WSUM and e_d <= rr.TAU_DEPTH, tag


# (id, N, M, S, S_imp, H, W, decoder, kwargs, path)
E2E = [
    ('ragged_3x100_s7', 3, 100, 7, 0, 20, 36, 'opaque_s4', {}, 0),
    ('ragged_imp_24_9', 2, 37, 24, 9, 48, 16, 'opaque_s11', {}, 1),
    ('imp_48_48', 2, 64, 48, 48, 32, 32, 'opaque_s4', {}, 1),
    ('s4_m5_2x2_box2', 1, 5, 4, 0, 2, 2, 'opaque_s4', {'box': 2.0}, 0),
    ('s9_odd_h2_w3', 2, 70, 9, 0, 2, 3, 'opaque_s11', {}, 0),
    ('imp_32_16_tiles256', 1, 50, 32, 16, 9, 7, 'opaque_s4', {}, 1),
    ('imp_33_15_fallback', 1, 50, 33, 15, 9, 7, 'opaque_s4', {}, 2),
    ('imp_st384', 1, 20, 192, 192, 16, 16, 'opaque_s11', {}, 1),
    ('single_s384', 1, 9, 384, 0, 16, 16, 'opaque_s4', {'miss': False}, 0),
    ('x4_single', 2, 80, 21, 0, 24, 24, 'opaque_s5_x4', {}, 0),
    ('x005_imp', 1, 64, 16, 16, 24, 24, 'opaque_s23_x0.05', {}, 1),
    ('white_back_imp', 2, 40, 12, 12, 16, 16, 'opaque_s4', {'wb': True}, 1),
]
DECODERS = dict(rr.decoder_set())


@pytest.mark.parametrize('cid,N,M,S,S_imp,H,W,dec,kw,path', E2E, ids=[c[0] for c in E2E])
def test_render_vs_float64(cid, N, M, S, S_imp, H, W, dec, kw, path):
    kw = dict(kw)
    planes, o, d, u_c, u_f = _ragged(N, M, S, S_imp, H, W, seed=len(cid) * 31 + S, miss=kw.pop('miss', True))
    mlp = DECODERS[dec]
    ref = rr.render64(planes, mlp, o, d, S=S, S_imp=S_imp, box_warp=kw.get('box', 1.0), white_back=kw.get('wb', False), u_coarse=u_c, u_fine=u_f)
    got = render(planes, mlp, S, S_imp, o=o, d=d, u_c=u_c, u_f=u_f, path=path, **kw)
    _compare(got, ref, rr.TAU_RGB, f'{cid} path {path}')


@pytest.mark.parametrize('S_imp', [0, 12])
def test_hwpc_view_and_two_plane_sets(S_imp):
    """The producer's channels-last view and `cano + secc` as two sets (the second shared by both frames: frame stride 0)."""
    N, res, S = 2, 16, 12
    g = torch.Generator().manual_seed(5 + S_imp)
    secc, cano = torch.randn(N, 3, 32, 32, 32, generator=g), torch.randn(1, 3, 32, 32, 32, generator=g)
    cam = syn.lookat_camera(torch.tensor([0.1, -0.15]), torch.tensor([-0.3, 0.45]))
    o, d = camera_rays(cam, res)
    u_c, u_f = syn.make_jitter(N, res * res, S, S_imp, seed=13)
    mlp = DECODERS['opaque_s4']
    ref = rr.render64(secc, mlp, o, d, S=S, S_imp=S_imp, u_coarse=u_c, u_fine=u_f, planes2=cano)
    ref1 = rr.render64(secc, mlp, o, d, S=S, S_imp=S_imp, u_coarse=u_c, u_fine=u_f)
    path = 0 if S_imp == 0 else 1
    got = render(secc, mlp, S, S_imp, o=o, d=d, u_c=u_c, u_f=u_f, planes2=cano, path=path)
    hw = render(secc, mlp, S, S_imp, o=o, d=d, u_c=u_c, u_f=u_f, hwpc=True, path=path)
    _compare(got, ref, rr.TAU_RGB, f'two sets S_imp={S_imp} path {path}')
    _compare(hw, ref1, rr.TAU_RGB, f'hwpc S_imp={S_imp} path {path}')


@pytest.mark.parametrize('D,S,S_imp,path', [(2, 11, 0, 0), (4, 9, 6, 1)])
def test_trigrids_vs_float64(D, S, S_imp, path):
    N, M = 2, 90
    g = torch.Generator().manual_seed(D * 7 + S)
    grids = torch.randn(N, 3, 32 * D, 12, 10, generator=g)
    o, d = rr.scatter_rays(N, M, D)
    u_c = torch.rand(N, M, S, 1, generator=g)
    u_f = torch.rand(N * M, S_imp, generator=g) if S_imp else None
    mlp = DECODERS['opaque_s11']
    ref = rr.render64(grids, mlp, o, d, S=S, S_imp=S_imp, u_coarse=u_c, u_fine=u_f, trigrid_depth=D)
    got = render(grids, mlp, S, S_imp, o=o, d=d, u_c=u_c, u_f=u_f, depth=D, path=path)
    _compare(got, ref, rr.TAU_RGB, f'trigrid D={D} S_imp={S_imp} path {path}')


@pytest.mark.parametrize('S_imp,dec', [(0, 'opaque_s4'), (0, 'transparent'), (48, 'transparent'),
                                       pytest.param(48, 'opaque_s4', marks=pytest.mark.xfail(strict=True, reason=(
                                           'importance resampling from fp32 weights: the fp32 oracle is 9.5e-6 from float64 here (the kernel '
                                           '9.4e-6), above TAU_RGB; see render_reference.py')))])
def test_baseline_config1_vs_float64(S_imp, dec):
    """BASELINE config 1: N = 1, 64^2 camera rays generated in-kernel, 48 (+48) samples, 3 x 32 x 256^2 planes."""
    planes, cam = syn.make_planes(1, seed=0), syn.make_cameras(1, seed=1)
    u_c, u_f = syn.make_jitter(1, 4096, 48, S_imp, seed=2)
    o, d = camera_rays(cam, 64)
    mlp = DECODERS[dec] if dec != 'transparent' else rr.transparent_decoder()
    ref = rr.render64(planes, mlp, o, d, S=48, S_imp=S_imp, u_coarse=u_c, u_fine=u_f)
    path = 0 if S_imp == 0 else 1
    got = render(planes, mlp, 48, S_imp, camera=cam, res=64, u_c=u_c, u_f=u_f, path=path)
    _compare(got, ref, rr.TAU_RGB, f'baseline S_imp={S_imp} {dec} path {path}')


@pytest.mark.parametrize('res', [24, 20])
def test_camera_rays_white_back(res):
    """In-kernel camera rays, white_back, some rays missing the box; neither res is a multiple of the streaming kernel's G = 16 (non-image
    ray groups)."""
    N, S = 3, 13
    cam = syn.make_cameras(N, seed=78)
    cam[1, 16] = cam[1, 20] = 1.5                                             # wide FOV: rays miss the box
    g = torch.Generator().manual_seed(res)
    planes = torch.randn(N, 3, 32, 40, 24, generator=g)
    u_c = torch.rand(N, res * res, S, 1, generator=g)
    o, d = camera_rays(cam, res)
    mlp = DECODERS['opaque_s11']
    ref = rr.render64(planes, mlp, o, d, S=S, white_back=True, u_coarse=u_c)
    assert 0 < int(ref[3].sum()) < ref[3].numel()
    got = render(planes, mlp, S, camera=cam, res=res, wb=True, u_c=u_c, path=0)
    _compare(got, ref, rr.TAU_RGB, f'camera res={res}')


def test_every_ray_misses():
    """No valid ray: the limits stay (t0, t1) = (-1, -2) for every ray (the reference does the same) and the samples lie behind the origins."""
    N, M, S = 1, 40, 10
    g = torch.Generator().manual_seed(4)
    planes = torch.randn(N, 3, 32, 8, 8, generator=g)
    o = torch.tensor([2.0, 2.0, 1.6]).expand(N, M, 3).contiguous()                     # beside the box: the lines through it never meet it
    d = torch.nn.functional.normalize(torch.tensor([0.0, 0.0, -1.0]) + 0.1 * torch.randn(N, M, 3, generator=g), dim=-1)
    u_c = torch.rand(N, M, S, 1, generator=g)
    mlp = rr.transparent_decoder()
    ref = rr.render64(planes, mlp, o, d, S=S, u_coarse=u_c)
    assert int(ref[3].sum()) == 0
    got = render(planes, mlp, S, o=o, d=d, u_c=u_c, path=0)
    _compare(got, ref, rr.TAU_RGB, 'all miss')


# ---- (c) stand-alone ops --------------------------------------------------------------------------------------------------------------------
def _edge_points(P, seed, sizes=(16, 8, 4)):
    """Grid coordinates (box_warp = 1) on texel centres, texel edges, the box faces and just outside (taps in the zero padding), for every
    size in `sizes`: all dyadic, so the kernels' pixel coordinates are exact."""
    cand = [-1.0, 1.0, -1.0 - 1 / 64, 1.0 + 1 / 64, -1.0 - 1 / 8, 1.0 + 1 / 8, 0.0]
    for n in sizes:
        cand += [(2 * i + 1) / n - 1 for i in range(n)] + [2 * i / n - 1 for i in range(n + 1)]
    cand = torch.tensor(cand)
    g = torch.Generator().manual_seed(seed)
    pick = cand[torch.randint(len(cand), (1, P, 3), generator=g)]
    jitter = rr.dyadic(torch.rand(1, P, 3, generator=g) * 2 - 1) * (torch.rand(1, P, 3, generator=g) < 0.3)
    return torch.where(jitter != 0, jitter, pick) / 2                         # world x = g / 2


@pytest.mark.parametrize('D', [0, 4])
def test_triplane_trigrid_sample_element_bound(D):
    N, H, W, P = 2, 8, 16, 3000
    g = torch.Generator().manual_seed(40 + D)
    planes = torch.randn(N, 3, 32 * max(D, 1), H, W, generator=g)
    pts = _edge_points(P, D).expand(N, -1, -1).contiguous()
    f, q, sg = rr.gather64(planes, pts, 1.0, D)
    eg = rr.gather_bound(q, sg, D)
    out = torch.empty(N, 3, P, 32, device=DEV)
    coords = capi.f32(pts.to(DEV))
    if D:
        pcl = ren.grids_to_channels_last(planes.to(DEV), D)
        capi.check(capi.lib().r3dp_trigrid_sample(capi.ptr(pcl.data), N, 32, D, H, W, capi.ptr(coords), P, C.c_float(1.0), capi.ptr(out), capi.stream()))
    else:
        pcl = ren.planes_to_channels_last(planes.to(DEV))
        capi.check(capi.lib().r3dp_triplane_sample(capi.ptr(pcl.data), N, 32, H, W, capi.ptr(coords), P, C.c_float(1.0), capi.ptr(out), capi.stream()))
    got = out.cpu().double().mean(1)
    err = (got - f).abs()
    assert bool((err <= eg).all())                                            # eg = 0 where every tap is in the zero padding: exact zeros
    ratio = float((err / eg.clamp_min(1e-300)).max())
    print(f'sample D={D}: worst error / bound = {ratio:.3f}; samples entirely in the zero padding {int((f.abs().amax(-1) == 0).sum())}')


def _mlp_struct(mlp):
    dec = {k: v.to(DEV).contiguous() for k, v in mlp.items()}
    return dec, capi.mlp_struct(dec['net.0.weight'], dec['net.0.bias'], dec['net.2.weight'], dec['net.2.bias'])


@pytest.mark.parametrize('K', [1, 3])
def test_decode_cuda_core_element_bound(K):
    N, P = 2, 3000
    g = torch.Generator().manual_seed(K)
    feat = torch.randn(N, K, P, 32, generator=g) * 0.6
    feat_d = feat.to(DEV)
    for name, mlp in rr.decoder_set():
        dec, m = _mlp_struct(mlp)
        rgb, sig = torch.empty(N, P, 32, device=DEV), torch.empty(N, P, 1, device=DEV)
        capi.check(capi.lib().r3dp_decode(capi.ptr(feat_d), N, K, P, 32, C.byref(m), capi.ptr(rgb), capi.ptr(sig), capi.stream()))
        f = feat.double().mean(1)
        ef = 2 * U * feat.double().abs().mean(1) if K == 3 else 0.0                 # fp32 mean of three: two roundings
        cref, sref = rr.decode64(f, mlp)
        ec, es = rr.decoder_bound(f, mlp, ef, split=False)
        rc = float(((rgb.cpu().double() - cref).abs() / ec).max())
        rs = float(((sig.cpu().double() - sref).abs() / es).max())
        print(f'decode K={K} {name}: colour {rc:.3f}, sigma {rs:.3f} of the bound')
        assert rc <= 1.0 and rs <= 1.0, name


def test_run_model_element_bound():
    """Gather + CUDA-core decoder at the edge coordinates: the gather bound feeds the decoder bound."""
    N, H, W, P = 2, 8, 16, 3000
    g = torch.Generator().manual_seed(50)
    planes = torch.randn(N, 3, 32, H, W, generator=g)
    pts = _edge_points(P, 50).expand(N, -1, -1).contiguous()
    f, q, sg = rr.gather64(planes, pts, 1.0)
    eg = rr.gather_bound(q, sg)
    pcl = ren.planes_to_channels_last(planes.to(DEV))
    coords = capi.f32(pts.to(DEV))
    for name, mlp in rr.decoder_set():
        dec, m = _mlp_struct(mlp)
        rgb, sig = torch.empty(N, P, 32, device=DEV), torch.empty(N, P, 1, device=DEV)
        capi.check(capi.lib().r3dp_run_model(capi.ptr(pcl.data), N, 32, H, W, capi.ptr(coords), P, C.c_float(1.0), C.byref(m), capi.ptr(rgb),
                                             capi.ptr(sig), capi.stream()))
        cref, sref = rr.decode64(f, mlp)
        ec, es = rr.decoder_bound(f, mlp, eg, split=False)
        rc = float(((rgb.cpu().double() - cref).abs() / ec).max())
        rs = float(((sig.cpu().double() - sref).abs() / es).max())
        print(f'run_model {name}: colour {rc:.3f}, sigma {rs:.3f} of the bound')
        assert rc <= 1.0 and rs <= 1.0, name


@pytest.mark.parametrize('opaque', [True, False])
def test_ray_march_element_bound(opaque):
    """Stand-alone marcher vs float64, element by element.  Near-transparent rays: alpha = 1 - __expf(-x) with x ~ 1e-5 cancels, and
    __expf's error ((2 + 1.16 x) ulp of e = exp(-x) ~ 1, 2^-23 absolute) is a relative error of ~1e-2 in alpha.  The bound carries that
    term explicitly; it dominates the depth there (a weighted mean whose weights are each off by ~1e-2 of themselves)."""
    from oracle import real3d_oracle as orc
    N, M, S, Cc = 2, 300, 17, 32
    g = torch.Generator().manual_seed(6)
    col = torch.rand(N, M, S, Cc, generator=g)
    sig = torch.randn(N, M, S, 1, generator=g) * 3 + (30.0 if opaque else -8.0)
    dep = torch.sort(torch.rand(N, M, S, 1, generator=g) + 2.0, dim=2).values
    ref_rgb, ref_depth, ref_w = orc.ray_march(col.double(), sig.double(), dep.double())
    col_d, sig_d, dep_d = col.to(DEV), sig.to(DEV), dep.to(DEV)
    rgb, depth, w = torch.empty(N, M, Cc, device=DEV), torch.empty(N, M, 1, device=DEV), torch.empty(N, M, S - 1, 1, device=DEV)
    ws = torch.empty(64, device=DEV, dtype=torch.uint8)
    capi.check(capi.lib().r3dp_ray_march(capi.ptr(col_d), capi.ptr(sig_d), capi.ptr(dep_d), N, M, S, Cc, 0, capi.ptr(rgb), capi.ptr(depth),
                                         capi.ptr(w), capi.ptr(ws, torch.uint8), capi.stream()))
    torch.cuda.synchronize()
    d64 = dep.double()
    delta = d64[:, :, 1:] - d64[:, :, :-1]
    arg = (sig[:, :, :-1] + sig[:, :, 1:]).double() / 2 - 1
    smid = orc.softplus(arg)
    x = smid * delta
    e = torch.exp(-x)
    alpha = 1 - e
    # smid: softplus_fast + the rounding of its argument; x = smid delta: delta and the product rounded; e: __expf; 1 - e: rounded
    e_smid = rr.SP_ABS + rr.SP_REL * smid + 2 * U * arg.abs()
    e_alpha = e * (e_smid * delta + 2 * U * x + (2 + 1.16 * x) * 2 * U) + U * alpha      # the cancellation term: e (2 + 1.16 x) 2^-23
    e_T = torch.cumsum(e_alpha + 2 * U, 2) - (e_alpha + 2 * U)                            # exclusive: the factors before interval k
    T = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :, :1]), 1 - alpha + 1e-10], 2), 2)[:, :, :-1]
    e_w = e_alpha * T + alpha * e_T + U * ref_w
    err_w = (w.cpu().double() - ref_w).abs()
    c_mid = (col[:, :, :-1] + col[:, :, 1:]).double() / 2
    e_rgb = 2 * ((e_w * (c_mid + U)).sum(2) + (S + 2) * U * (ref_w * c_mid).sum(2)) + U
    err_rgb = (rgb.cpu().double() - ref_rgb).abs()
    wsum = ref_w.sum(2)
    d_mid = (d64[:, :, :-1] + d64[:, :, 1:]) / 2
    slack = (wsum - e_w.sum(2)).clamp_min(0)
    e_depth = (e_w * (d_mid - ref_depth.unsqueeze(2)).abs()).sum(2) / slack + 2 * (S + 2) * U * ref_depth.abs()
    err_depth = (depth.cpu().double() - ref_depth).abs()
    rw, rc, rd = (float((err_w / e_w).max()), float((err_rgb / e_rgb).max()), float((err_depth / e_depth).max()))
    print(f'ray_march opaque={opaque}: worst error / bound: weights {rw:.3f}, rgb {rc:.3f}, depth {rd:.3f}; depth error {float(err_depth.max()):.2e}')
    assert rw <= 1.0 and rc <= 1.0 and rd <= 1.0


# ---- (d) bit-exact properties ---------------------------------------------------------------------------------------------------------------
FRAME_CASES = [(13, 0, 0), (48, 0, 0), (12, 12, 1), (33, 15, 2)]      # (S, S_imp, path)


@pytest.mark.parametrize('S,S_imp,path', FRAME_CASES)
def test_frames_independent_and_repeatable(S, S_imp, path):
    """Frame k of an N = 3 render equals the N = 1 render of frame k, and a repeated render gives the same bits.  Every ray hits the box:
    invalid rays take the call-wide limits (renderer.py:123-126), so with one of them the frames would rightly differ."""
    N, M = 3, 24 * 24
    planes, _, _, u_c, u_f = _ragged(N, M, S, S_imp, 16, 16, seed=S + S_imp)
    o, _ = rr.probe_rays(N, M, seed=S, box=0.7)                               # |x|, |y| <= 0.35: a 0.02 tilt cannot leave through a side
    o[..., 2] = 1.6
    d = torch.nn.functional.normalize(torch.tensor([0.0, 0.0, -1.0]) + 0.02 * torch.randn(N, M, 3, generator=torch.Generator().manual_seed(S)), dim=-1)
    mlp = DECODERS['opaque_s4']
    full = render(planes, mlp, S, S_imp, o=o, d=d, u_c=u_c, u_f=u_f, path=path)
    again = render(planes, mlp, S, S_imp, o=o, d=d, u_c=u_c, u_f=u_f, path=path)
    assert bool(full[3].all())
    for a, b in zip(full, again):
        assert torch.equal(a, b)
    for k in range(N):
        uf = u_f[k * M:(k + 1) * M] if u_f is not None else None
        one = render(planes[k:k + 1], mlp, S, S_imp, o=o[k:k + 1], d=d[k:k + 1], u_c=u_c[k:k + 1], u_f=uf, path=path)
        for a, b in zip(one, full):
            assert torch.equal(a[0], b[k]), k


def test_all_paths_covered():
    """The case tables of this module, each of whose renders asserts its path through r3dp_render_path, span all three paths."""
    paths = {p[-1] for p in PROBE_PATHS} | {c[-1] for c in E2E} | {c[-1] for c in FRAME_CASES}
    assert paths == {0, 1, 2}, paths
