"""FrameEngine(secc2plane=..., img2plane=...): a clip started from the source image with begin_planes(img=...) renders the frames of one
started with begin_planes(cano_planes=model(img)), for the plain head, the torso head and the secc_renderer coefficient path; a second
begin_planes(img=...) refills the canonical buffer in place, so the graphs captured for the first clip render the second one as a fresh
engine does; the exclusivity errors."""
import pytest
import torch

import img2plane_reference as iref
import secc2plane_reference as sref
import real3dportrait_b200 as r3
from real3dportrait_b200 import engine, synthetic as syn

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
B = 2
KINDS = ['plain', 'torso', 'renderer']


@pytest.fixture(scope='module')
def img2plane():
    m = r3.Img2PlaneModel()
    m.load_state_dict(iref.make_params({k: v.shape for k, v in m.state_dict().items()}, 5), strict=True)
    return m.to(DEV).eval()


@pytest.fixture(scope='module')
def renderer(tmp_path_factory):
    kw = syn.write_bfm_folder(str(tmp_path_factory.mktemp('bfm')), seed=0)
    return r3.SECC_Renderer(512, device=DEV, **kw)


def _backbone():
    bb = r3.SegFormerSECC2PlaneBackbone()
    bb.load_state_dict(sref.make_params({k: v.shape for k, v in bb.state_dict().items()}, 7), strict=True)
    return bb.to(DEV).eval()


def _engine(kind, r, **kw):
    if kind == 'torso':
        hp = dict(syn.WARP_HPARAMS, htbsr_head_weight_fuse_mode='v2', num_samples_fine=48, neural_rendering_resolution=64)
        eng = engine.FrameEngine(batch=B, sr_mode='tc', hp=hp, torso_model=syn.StubTorsoModel(), out_uint8=True, secc2plane=_backbone(), **kw)
        eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_warp_params(seed=6, fuse_mode='v2'))
        inp = syn.make_warp_inputs(1, seed=3)
        eng.begin_clip(*(inp[k].to(DEV) for k in ('ref_torso_rgb', 'ref_bg_rgb', 'segmap', 'kp_s')))
        return eng
    extra = {'secc_renderer': r} if kind == 'renderer' else {}
    eng = engine.FrameEngine(batch=B, sr_mode='tc', hp={'num_samples_fine': 0}, out_uint8=True, secc2plane=_backbone(), **extra, **kw)
    eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_params(seed=5))
    return eng


def _conds(kind, seed):
    """The per-clip arguments of begin_planes besides the planes: (cond_cano, cond_src) images, or coeff_src for the renderer engine."""
    if kind == 'renderer':
        c = syn.make_coeffs(1, seed=seed)
        return (), {'coeff_src': torch.cat([c['id'], c['exp']], 1).to(DEV)}
    cano, src, _ = sref.make_inputs(1, 512, seed)
    return (cano.to(DEV), src.to(DEV)), {}


def _frames(kind, n, seed=40):
    out = []
    for s in range(n):
        cams = syn.make_cameras(B, seed=seed + s + 200).to(DEV)
        if kind == 'renderer':
            c = syn.make_coeffs(B, seed=seed + s)
            u_c, _ = syn.make_jitter(B, 4096, 48, 0, seed=seed + s + 100)
            out.append(((None, cams, u_c.to(DEV)), {'coeff': torch.cat([c['id'], c['exp']], 1).to(DEV)}))
            continue
        _, _, tgt = sref.make_inputs(B, 512, seed + s)
        if kind == 'torso':
            u_c, u_f = syn.make_jitter(B, 64 * 64, 48, 48, seed=seed + s + 100)
            kp_d = torch.rand(B, 68, 3, generator=torch.Generator().manual_seed(seed + s + 300)) * 2 - 1
            out.append(((None, cams, u_c.to(DEV), u_f.to(DEV)), {'kp_d': kp_d.to(DEV), 'cond_tgt': tgt.to(DEV)}))
        else:
            u_c, _ = syn.make_jitter(B, 4096, 48, 0, seed=seed + s + 100)
            out.append(((None, cams, u_c.to(DEV)), {'cond_tgt': tgt.to(DEV)}))
    return out


def _begin(eng, kind, seed, img=None, planes=None):
    a, kw = _conds(kind, seed)
    eng.begin_planes(planes, *a, **kw, **({'img': img} if img is not None else {}))


@pytest.mark.parametrize('kind', KINDS)
@torch.no_grad()
def test_clip_from_image_matches_clip_from_planes_and_refills_in_place(kind, img2plane, renderer):
    m = img2plane
    from_img, from_planes = _engine(kind, renderer, img2plane=m), _engine(kind, renderer, use_graph=False)
    frames = _frames(kind, 2)
    img = iref.make_inputs(1, 512, 21).to(DEV)
    _begin(from_img, kind, 1, img=img)
    _begin(from_planes, kind, 1, planes=m(img))
    for a, kw in frames:
        assert torch.equal(from_img.step(*a, **kw), from_planes.step(*a, **kw))
    graph, buf = from_img.graph, from_img._cano_cl.data.data_ptr()
    assert graph is not None
    # a second clip: the same canonical buffer, the same graphs, the frames of a fresh engine
    img2 = iref.make_inputs(1, 512, 22).to(DEV)
    _begin(from_img, kind, 2, img=img2)
    assert from_img._cano_cl.data.data_ptr() == buf
    fresh = _engine(kind, renderer, img2plane=m)
    _begin(fresh, kind, 2, img=img2)
    for a, kw in frames:
        assert torch.equal(from_img.step(*a, **kw), fresh.step(*a, **kw))
    assert from_img.graph is graph


def test_exclusivity_errors(img2plane, renderer):
    m = img2plane
    with pytest.raises(ValueError, match='img2plane'):
        engine.FrameEngine(batch=B, img2plane=m)
    eng = _engine('plain', renderer, img2plane=m)
    img = iref.make_inputs(1, 512, 21).to(DEV)
    (c_cano, c_src), _ = _conds('plain', 1)
    with pytest.raises(ValueError, match='exactly one'):
        eng.begin_planes(syn.make_planes(1).to(DEV), c_cano, c_src, img=img)
    with pytest.raises(ValueError, match='exactly one'):
        eng.begin_planes(cond_cano=c_cano, cond_src=c_src)
    with pytest.raises(ValueError, match='img2plane'):
        _engine('plain', renderer).begin_planes(img=img, cond_cano=c_cano, cond_src=c_src)
