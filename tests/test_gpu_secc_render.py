"""SECC renderer on the GPU against the float64 oracle (tests/secc_render_reference.py), with bars derived from fp32 rounding:

  vertices  |got - ref| <= the propagated bound of the K = 144 fp32 dot product (gamma_{K+1} sum |terms|), the pose and the projection
  raster    decisive pixels (the centre more than delta px inside the winner, every other face within delta px of it farther by more than
            delta_z relative pz) take the oracle's face; every other pixel takes a face the oracle finds within delta px, or none; delta follows
            from the vertex bar and the edge-function rounding
  values    where the faces agree, |secc - ref| <= 2 sum_i |dw_i| spread(ncc) + 12 u, with dw from the same vertex bar over the face's area
Also: every output element written, guards around the outputs untouched, the key buffer left empty; the class end to end; the engine fed
coefficients against the engine fed the class's images, bit for bit."""
import ctypes

import numpy as np
import pytest
import torch

import secc2plane_reference as s2p_ref
import secc_render_reference as ref
import secc_launch_reference as lr
from secc_launch_reference import U, value_bar, vertex_bar
import real3dportrait_b200 as r3
from real3dportrait_b200 import _capi as capi, engine, synthetic as syn

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
@pytest.fixture(scope='module')
def bfm(tmp_path_factory):
    kw = syn.write_bfm_folder(str(tmp_path_factory.mktemp('bfm')), seed=0)
    return kw, ref.load(kw['bfm_folder'], kw['ncc_path'], kw['eye_faces'])


def _coeffs(B, seed, yaw):
    c = syn.make_coeffs(B, seed=seed, yaw=yaw)
    return {k: v.to(DEV) for k, v in c.items()}


def _vertices(r, c, B):
    """r3dp_secc_vertices into a buffer between NaN guards (1024 floats, so the vertices stay 16-byte aligned): every element written, no guard."""
    G = 1024
    big = torch.full((B * r.n_verts * 4 + 2 * G,), float('nan'), device=DEV)
    verts = big[G:-G].view(B, r.n_verts, 4)
    L, p = capi.lib(), capi.ptr
    capi.check(L.r3dp_secc_vertices(p(r.basis), p(r.mean_shape), r.n_verts, r.n_id, r.n_exp, p(c['id']), r.n_id, p(c['exp']), r.n_exp,
                                    p(c['euler']), p(c['trans']), B, 10.0, r.tan_half, p(verts), capi.stream()))
    torch.cuda.synchronize()
    assert torch.isnan(big[:G]).all() and torch.isnan(big[-G:]).all(), 'vertex guard overwritten'
    assert not torch.isnan(verts).any(), 'vertex element not written'
    return verts


@pytest.fixture(scope='module')
def renderers(bfm):
    kw, _ = bfm
    return {S: r3.SECC_Renderer(S, device=DEV, **kw) for S in (512, 224, 97)}


@pytest.mark.parametrize('B,yaw', [(1, 0.0), (4, 0.6), (50, 0.6)])
def test_vertices_against_float64(bfm, renderers, B, yaw):
    _, m = bfm
    r = renderers[512]
    c = _coeffs(B, seed=10 + B, yaw=yaw)
    got = _vertices(r, c, B).cpu().double().numpy()
    v, bar = vertex_bar(m, c)
    err = np.abs(got[..., :3] - v)
    ratio = (err / bar).max()
    print(f'vertices B={B}: max |err| x {err[..., 0:2].max():.2e} z {err[..., 2].max():.2e}; worst err/bar {ratio:.3f}')
    assert ratio <= 1.0
    assert (got[..., 3] == 0).all()


def _raster_case(r, m, c, B, S, drop_face0=True):
    """Run the three launches with the key buffer read back between raster and resolve; returns the kernel's faces, secc, mask and the oracle's."""
    L, p, st = capi.lib(), capi.ptr, capi.stream()
    verts = _vertices(r, c, B)
    G = 1024
    keys = torch.full((B * S * S,), -1, dtype=torch.int64, device=DEV)
    capi.check(L.r3dp_secc_raster(p(verts), r.n_verts, p(r.face_buf, torch.int32), r.n_faces, B, S, p(keys, torch.int64), st))
    kimg = keys.clone()
    secc_big = torch.full((B * 3 * S * S + 2 * G,), float('nan'), device=DEV)
    mask_big = torch.full((B * S * S + 2 * G,), float('nan'), device=DEV)
    capi.check(L.r3dp_secc_resolve(p(verts), r.n_verts, p(r.face_buf, torch.int32), p(r.ncc), B, S, int(drop_face0), p(keys, torch.int64),
                                   ctypes.c_void_p(secc_big.data_ptr() + 4 * G), ctypes.c_void_p(mask_big.data_ptr() + 4 * G), st))
    torch.cuda.synchronize()
    assert (keys == -1).all(), 'resolve leaves the key buffer empty'
    for big in (secc_big, mask_big):
        assert torch.isnan(big[:G]).all() and torch.isnan(big[-G:]).all(), 'guard overwritten'
        assert not torch.isnan(big[G:-G]).any(), 'output element not written'
    k = kimg.cpu().numpy().view(np.uint64)
    face = np.where(k == np.uint64(2 ** 64 - 1), -1, (k & np.uint64(0xffffffff)).astype(np.int64)).reshape(B, S, S)
    secc = secc_big[G:-G].reshape(B, 3, S, S).cpu().double().numpy()
    mask = mask_big[G:-G].reshape(B, 1, S, S).cpu().double().numpy()
    return verts, face, secc, mask


def check_raster(m, c, B, S, face, secc, mask, label, drop_face0=True):
    v, bar = vertex_bar(m, c)
    return lr.check_raster(m, v, lr.raster_err(v, bar), S, face, secc, mask, label, drop_face0)


@pytest.mark.parametrize('S,B,yaw', [(512, 1, 0.0), (512, 4, 0.6), (224, 4, 0.6), (97, 2, 0.6)])
def test_raster_resolve_against_float64(bfm, renderers, S, B, yaw):
    _, m = bfm
    r = renderers[S]
    c = _coeffs(B, seed=20 + S + B, yaw=yaw)
    _, face, secc, mask = _raster_case(r, m, c, B, S)
    check_raster(m, c, B, S, face, secc, mask, f'S={S} B={B}')
    # the kernel path of the class gives the same images
    mk, sk = r(c['id'], c['exp'], c['euler'], c['trans'])
    assert np.array_equal(sk.cpu().double().numpy(), secc) and np.array_equal(mk.cpu().double().numpy(), mask)


def test_class_batch_50_at_512(bfm, renderers):
    _, m = bfm
    r = renderers[512]
    c = _coeffs(50, seed=5, yaw=0.6)
    _, face, secc, mask = _raster_case(r, m, c, 50, 512)
    check_raster(m, c, 50, 512, face, secc, mask, 'S=512 B=50')
    mk, sk = r(c['id'], c['exp'], c['euler'], c['trans'])
    assert np.array_equal(sk.cpu().double().numpy(), secc)


def test_class_end_to_end(bfm, renderers):
    _, m = bfm
    r = renderers[512]
    c = _coeffs(4, seed=31, yaw=0.0)
    _, face, _, _ = _raster_case(r, m, c, 4, 512, drop_face0=False)
    mask, secc = r(c['id'], c['exp'], c['euler'], c['trans'])
    f0 = torch.from_numpy(face == 0).to(DEV)
    assert f0[0].any() and f0[1].any()
    assert (mask[0, 0][f0[0]] == 0).all() and (secc[0][:, f0[0]] == -1).all()        # the packed face 0 is background in image 0 ...
    assert (mask[1, 0][f0[1]] == 1).all()                                              # ... and only there
    # [B,T,C] equals [B*T,C] reshaped
    bt = {k: v.reshape(2, 2, -1) for k, v in c.items()}
    m5, s5 = r(bt['id'], bt['exp'], bt['euler'], bt['trans'])
    assert s5.shape == (2, 3, 2, 512, 512) and m5.shape == (2, 1, 2, 512, 512)
    for n in range(2):
        for t in range(2):
            assert torch.equal(s5[n, :, t], secc[2 * n + t]) and torch.equal(m5[n, :, t], mask[2 * n + t])
    # B = 4 equals four B = 1 calls bit for bit, except where face 0 wins in images 1..3 (image 0 of each single call)
    for i in range(4):
        mi, si = r(*(c[k][i:i + 1] for k in ('id', 'exp', 'euler', 'trans')))
        keep = ~f0[i] if i > 0 else torch.ones_like(f0[i])
        assert torch.equal(si[0][:, keep], secc[i][:, keep]) and torch.equal(mi[0, 0][keep], mask[i, 0][keep])
        if i > 0:
            assert (si[0][:, f0[i]] == -1).all()
    # render(coeff) is forward on [id | exp]
    coeff = torch.cat([c['id'], c['exp']], 1)
    _, sr_ = r.render(coeff, c['euler'], c['trans'])
    assert torch.equal(sr_, secc)


# ---- the engine ---------------------------------------------------------------------------------------------------------------------------
EB = 2


def _backbone(seed=7):
    bb = r3.SegFormerSECC2PlaneBackbone()
    bb.load_state_dict(s2p_ref.make_params({k: v.shape for k, v in bb.state_dict().items()}, seed), strict=True)
    return bb.to(DEV).eval()


def _plain(**kw):
    eng = engine.FrameEngine(batch=EB, sr_mode='tc', hp={'num_samples_fine': 0}, out_uint8=True, **kw)
    eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_params(seed=5))
    return eng


def _coeff_frames(n, seed=40):
    out = []
    for s in range(n):
        c = syn.make_coeffs(EB, seed=seed + s)
        u_c, _ = syn.make_jitter(EB, 4096, 48, 0, seed=seed + s + 100)
        out.append((torch.cat([c['id'], c['exp']], 1).to(DEV), syn.make_cameras(EB, seed=seed + s + 200).to(DEV), u_c.to(DEV)))
    return out


def _src(seed):
    c = syn.make_coeffs(1, seed=seed)
    return syn.make_planes(1, seed=seed).to(DEV), torch.cat([c['id'], c['exp']], 1).to(DEV)


def _images(r, coeff_src):
    cano_c = coeff_src.clone()
    cano_c[:, 80:] = 0
    return r.render(cano_c)[1], r.render(coeff_src)[1]


@torch.no_grad()
def test_engine_rejections(renderers):
    r = renderers[512]
    with pytest.raises(ValueError, match='secc2plane'):
        engine.FrameEngine(batch=EB, secc_renderer=r)
    eng = _plain(secc2plane=_backbone(), secc_renderer=r)
    cano, cs = _src(1)
    with pytest.raises(ValueError):
        eng.begin_planes(cano, *_images(r, cs))
    eng.begin_planes(cano, coeff_src=cs)
    coeff, cams, u = _coeff_frames(1)[0]
    with pytest.raises(ValueError):
        eng.step(None, cams, u, cond_tgt=r.render(coeff)[1])
    with pytest.raises(ValueError):
        _plain(secc2plane=_backbone()).step(None, cams, u, coeff=coeff)


@torch.no_grad()
def test_engine_coeff_step_equals_image_step(renderers):
    r = renderers[512]
    g_eng, e_eng = _plain(secc2plane=_backbone(), secc_renderer=r), _plain(secc2plane=_backbone(), secc_renderer=r, use_graph=False)
    img_eng = _plain(secc2plane=_backbone())
    frames = _coeff_frames(3)
    cano, cs = _src(1)
    for e in (g_eng, e_eng):
        e.begin_planes(cano, coeff_src=cs)
    img_eng.begin_planes(cano, *_images(r, cs))                    # begin_planes(coeff_src=) == begin_planes with the class's two images
    for f in frames:
        got = g_eng.step(None, f[1], f[2], coeff=f[0]).clone()
        eager = e_eng.step(None, f[1], f[2], coeff=f[0]).clone()
        want = img_eng.step(None, f[1], f[2], cond_tgt=r.render(f[0])[1]).clone()
        assert got.shape == (EB, 512, 512, 3)
        assert torch.equal(got, eager) and torch.equal(got, want)
    graph = g_eng.graph
    assert g_eng.launches_per_step > 0
    assert g_eng.prepare(frames) == len(frames)                     # zero-copy graphs over (coeff, cameras, u_coarse) tuples
    for f in frames:
        assert torch.equal(g_eng.step(None, f[1], f[2], coeff=f[0]), e_eng.step(None, f[1], f[2], coeff=f[0]))
    # a second clip through the same graphs
    cano2, cs2 = _src(2)
    g_eng.begin_planes(cano2, coeff_src=cs2)
    e_eng.begin_planes(cano2, coeff_src=cs2)
    img_eng.begin_planes(cano2, *_images(r, cs2))
    assert g_eng.graph is graph and len(g_eng.inplace) == len(frames)
    for f in frames:
        a = g_eng.step(None, f[1], f[2], coeff=f[0]).clone()
        assert torch.equal(a, e_eng.step(None, f[1], f[2], coeff=f[0]))
        assert torch.equal(a, img_eng.step(None, f[1], f[2], cond_tgt=r.render(f[0])[1]))
    # step_host carries the coefficients in the planes slot
    coeff, cams, u = frames[0]
    h = [t.cpu().pin_memory() for t in (coeff, cams, u)]
    h_out = torch.empty(EB, 512, 512, 3, dtype=torch.uint8).pin_memory()
    g_eng.step_host(*h, h_out)
    g_eng.sync_host()
    assert torch.equal(h_out, e_eng.step(None, cams, u, coeff=coeff).cpu())


@torch.no_grad()
def test_graphs_keep_the_renderer_buffers(bfm):
    """Engines share one renderer: a second engine's .to() of it (and an explicit one) frees none of the buffers a first engine's graphs read."""
    kw, _ = bfm
    r = r3.SECC_Renderer(512, device=DEV, **kw)
    g1, e1 = _plain(secc2plane=_backbone(), secc_renderer=r), _plain(secc2plane=_backbone(), secc_renderer=r, use_graph=False)
    cano, cs = _src(1)
    for e in (g1, e1):
        e.begin_planes(cano, coeff_src=cs)
    frames = _coeff_frames(2, seed=50)
    first = [g1.step(None, f[1], f[2], coeff=f[0]).clone() for f in frames]
    assert g1.prepare(frames[:1]) == 1
    keys = r.key_buffer(EB, 512)
    assert g1.graph.keep_alive[0] is r.basis and g1.graph.keep_alive[4] is keys
    g2 = _plain(secc2plane=_backbone(), secc_renderer=r)               # FrameEngine.__init__ calls r.to(device)
    g2.begin_planes(cano, coeff_src=cs)
    r.to(DEV)
    r.float()
    assert r.key_buffer(EB, 512) is keys                               # still the buffer the graphs write
    junk = [torch.full((EB, 512, 512), 7, dtype=torch.int64, device=DEV) for _ in range(8)]    # would land in a freed key buffer
    for f, want in zip(frames, first):
        a = g1.step(None, f[1], f[2], coeff=f[0]).clone()
        assert torch.equal(a, want) and torch.equal(a, e1.step(None, f[1], f[2], coeff=f[0]))
        assert torch.equal(g2.step(None, f[1], f[2], coeff=f[0]), want)
    torch.cuda.synchronize()
    assert (keys == -1).all()
    assert all((j == 7).all() for j in junk)                          # no graph wrote into memory it does not own


@torch.no_grad()
def test_torso_engine_coeff_graphs_match_eager(renderers):
    r = renderers[512]
    hp = dict(syn.WARP_HPARAMS, htbsr_head_weight_fuse_mode='v2', num_samples_fine=48, neural_rendering_resolution=64)

    def mk(**kw):
        eng = engine.FrameEngine(batch=EB, sr_mode='tc', hp=hp, torso_model=syn.StubTorsoModel(), out_uint8=True, secc2plane=_backbone(),
                                 secc_renderer=r, **kw)
        eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_warp_params(seed=6, fuse_mode='v2'))
        inp = syn.make_warp_inputs(1, seed=3)
        eng.begin_clip(*(inp[k].to(DEV) for k in ('ref_torso_rgb', 'ref_bg_rgb', 'segmap', 'kp_s')))
        cano, cs = _src(1)
        eng.begin_planes(cano, coeff_src=cs)
        return eng
    g_eng, e_eng = mk(), mk(use_graph=False)
    frames = []
    for s, (coeff, cams, _) in enumerate(_coeff_frames(2, seed=60)):
        u_c, u_f = syn.make_jitter(EB, 64 * 64, 48, 48, seed=70 + s)
        kp_d = torch.rand(EB, 68, 3, generator=torch.Generator().manual_seed(80 + s)) * 2 - 1
        frames.append((coeff, cams, u_c.to(DEV), u_f.to(DEV), kp_d.to(DEV)))
    for f in frames:
        a = g_eng.step(None, *f[1:4], kp_d=f[4], coeff=f[0]).clone()
        b = e_eng.step(None, *f[1:4], kp_d=f[4], coeff=f[0]).clone()
        assert torch.equal(a, b)
    cano2, cs2 = _src(2)
    g_eng.begin_planes(cano2, coeff_src=cs2)
    e_eng.begin_planes(cano2, coeff_src=cs2)
    for f in frames:
        assert torch.equal(g_eng.step(None, *f[1:4], kp_d=f[4], coeff=f[0]), e_eng.step(None, *f[1:4], kp_d=f[4], coeff=f[0]))


def test_against_pytorch3d(bfm, renderers):
    """The class against the reference's MeshRenderer path on pytorch3d, where pytorch3d is installed."""
    pytorch3d = pytest.importorskip('pytorch3d')  # noqa: F841
    from pytorch3d.renderer import FoVPerspectiveCameras, MeshRasterizer, RasterizationSettings
    from pytorch3d.structures import Meshes
    import pytorch3d.ops
    _, m = bfm
    r = renderers[512]
    c = _coeffs(2, seed=77, yaw=0.0)
    v = torch.from_numpy(ref.vertices(m, *(c[k].cpu().double().numpy() for k in ('id', 'exp', 'euler', 'trans')))).float()
    # back from NDC to the camera-space vertices the reference hands pytorch3d (x already negated)
    z = v[..., 2]
    cam = torch.stack([v[..., 0] * z * ref.TAN_HALF, v[..., 1] * z * ref.TAN_HALF, z], -1).to(DEV)
    tri = r.face_buf.long()
    mesh = Meshes(cam, tri.unsqueeze(0).repeat(2, 1, 1))
    cams = FoVPerspectiveCameras(device=DEV, fov=r.fov, znear=5.0, zfar=15.0)
    frag = MeshRasterizer()(mesh, cameras=cams, raster_settings=RasterizationSettings(image_size=512))
    mask = (frag.pix_to_face.squeeze(-1) > 0).float().unsqueeze(1)
    feat = r.ncc[:, :3].repeat(2, 1)[mesh.faces_packed()]
    img = pytorch3d.ops.interpolate_face_attributes(frag.pix_to_face, frag.bary_coords, feat).squeeze(-2).permute(0, 3, 1, 2)
    want = 2 * mask * img - 1
    mk, sk = r(c['id'], c['exp'], c['euler'], c['trans'])
    agree = (mk == mask).float().mean().item()
    # values where both pick the same face: each side is an fp32 evaluation of the same barycentrics from vertices within the vertex bar of
    # float64, so their difference is within twice the per-pixel bar of tests against float64
    _, face, _, _ = _raster_case(r, m, c, 2, 512)
    p3 = frag.pix_to_face.squeeze(-1).cpu().numpy()
    p3 = np.where(p3 >= 0, p3 - np.arange(2)[:, None, None] * r.n_faces, -1)            # packed -> per-image face index
    v64, bar = vertex_bar(m, c)
    worst, n = 0.0, 0
    for b in range(2):
        same = np.nonzero((face[b].reshape(-1) == p3[b].reshape(-1)) & (face[b].reshape(-1) > 0))[0]
        vbar, _ = value_bar(m, v64[b], face[b].reshape(-1)[same], 2 * bar[b, :, :2].max() + 4 * U)
        err = np.abs(sk[b].reshape(3, -1)[:, same].T.cpu().double().numpy() - want[b].reshape(3, -1)[:, same].T.cpu().double().numpy())
        worst, n = max(worst, float((err / (2 * vbar)).max(initial=0))), n + same.size
    print(f'pytorch3d: mask agreement {agree:.6f}, {n} pixels with the same face, worst secc err / bar {worst:.3f}')
    assert agree > 0.999 and n > 0.3 * 2 * 512 * 512
    assert worst <= 1.0
