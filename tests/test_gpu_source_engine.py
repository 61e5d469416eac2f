"""A torso FrameEngine with img2plane started from prepare_source's outputs (begin_planes(img=ref_head_img), begin_clip(ref_torso_img,
bg_img, ...)) renders the frames of an engine fed the reference's arrays; a second clip refilled through prepare_source(out=) into the same
buffers renders as a fresh engine does, through the graphs captured for the first."""
import numpy as np
import pytest
import torch

import img2plane_reference as iref
import secc2plane_reference as sref
import source_reference as sr
import real3dportrait_b200 as r3
from conftest import GOLDEN
from real3dportrait_b200 import engine, synthetic as syn

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
B = 2


@pytest.fixture(scope='module')
def img2plane():
    m = r3.Img2PlaneModel()
    m.load_state_dict(iref.make_params({k: v.shape for k, v in m.state_dict().items()}, 5), strict=True)
    return m.to(DEV).eval()


def _engine(img2plane, **kw):
    bb = r3.SegFormerSECC2PlaneBackbone()
    bb.load_state_dict(sref.make_params({k: v.shape for k, v in bb.state_dict().items()}, 7), strict=True)
    hp = dict(syn.WARP_HPARAMS, htbsr_head_weight_fuse_mode='v2', num_samples_fine=48, neural_rendering_resolution=64)
    eng = engine.FrameEngine(batch=B, sr_mode='tc', hp=hp, torso_model=syn.StubTorsoModel(), out_uint8=True, secc2plane=bb.to(DEV).eval(),
                             img2plane=img2plane, **kw)
    eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_warp_params(seed=6, fuse_mode='v2'))
    return eng


def _start(eng, head, torso, bg, seg, seed):
    cano, src, _ = sref.make_inputs(1, 512, seed)
    kp_s = torch.rand(1, 68, 3, generator=torch.Generator().manual_seed(seed)) * 2 - 1
    eng.begin_clip(torso, bg, seg, kp_s.to(DEV))
    eng.begin_planes(None, cano.to(DEV), src.to(DEV), img=head)


def _frames(n=2, seed=40):
    out = []
    for s in range(n):
        cams = syn.make_cameras(B, seed=seed + s + 200).to(DEV)
        _, _, tgt = sref.make_inputs(B, 512, seed + s)
        u_c, u_f = syn.make_jitter(B, 64 * 64, 48, 48, seed=seed + s + 100)
        kp_d = torch.rand(B, 68, 3, generator=torch.Generator().manual_seed(seed + s + 300)) * 2 - 1
        out.append(((None, cams, u_c.to(DEV), u_f.to(DEV)), {'kp_d': kp_d.to(DEV), 'cond_tgt': tgt.to(DEV)}))
    return out


@torch.no_grad()
def test_engine_from_prepare_source(img2plane):
    z = np.load(f'{GOLDEN}/source_small.npz')
    name, img, seg = sr.golden_cases(z)[0]
    assert name == 'portrait' and img.shape == (512, 512, 3)
    seg_t = torch.from_numpy(seg).to(DEV)
    src = r3.prepare_source(torch.from_numpy(img).to(DEV), seg_t)
    # the reference's arrays; at pixels where sklearn picked another of several equidistant background pixels, the library's choice
    bg_lib = torch.round(src['bg_img'][0].permute(1, 2, 0) * 127.5 + 127.5).to(torch.uint8).cpu().numpy()
    bg_ref = z['portrait.bg'].copy()
    _, fill, imgs, arg = sr.extract_background(img[None], seg[None])
    assert sr.check_background(bg_lib, bg_ref, fill, sr.source_colours(imgs, arg)) > 0
    bg_ref[(bg_lib != bg_ref).any(-1)] = bg_lib[(bg_lib != bg_ref).any(-1)]
    ref = {'ref_head_img': sr.normalise(z['portrait.head']), 'ref_torso_img': sr.normalise(z['portrait.torso']), 'bg_img': sr.normalise(bg_ref)}
    for k in ref:
        assert torch.equal(src[k].cpu(), ref[k]), k
    frames = _frames()
    lib_eng, ref_eng = _engine(img2plane), _engine(img2plane)
    _start(lib_eng, src['ref_head_img'], src['ref_torso_img'], src['bg_img'], seg_t[None], 1)
    _start(ref_eng, *(ref[k].to(DEV) for k in ('ref_head_img', 'ref_torso_img', 'bg_img')), seg_t[None], 1)
    for a, kw in frames:
        assert torch.equal(lib_eng.step(*a, **kw), ref_eng.step(*a, **kw))
    graph = lib_eng.graph
    assert graph is not None
    # a second clip: prepare_source refills the buffers the engine was fed
    img2, seg2 = syn.make_source_image(512, 512, 11), syn.make_segmap(512, 512, 11, center=0.42, neck_gaps=3)
    seg2_t = torch.from_numpy(seg2).to(DEV)
    ptrs = {k: v.data_ptr() for k, v in src.items()}
    r3.prepare_source(torch.from_numpy(img2).to(DEV), seg2_t, out=src)
    assert all(src[k].data_ptr() == ptrs[k] for k in src)
    assert torch.equal(src['ref_torso_img'].cpu(), sr.normalise(sr.inpaint_torso(img2, seg2)))
    assert torch.equal(src['bg_img'].cpu(), sr.normalise(sr.extract_background(img2[None], seg2[None])[0]))
    _start(lib_eng, src['ref_head_img'], src['ref_torso_img'], src['bg_img'], seg2_t[None], 2)
    fresh = _engine(img2plane)
    _start(fresh, *(src[k].clone() for k in ('ref_head_img', 'ref_torso_img', 'bg_img')), seg2_t[None].clone(), 2)
    for a, kw in frames:
        assert torch.equal(lib_eng.step(*a, **kw), fresh.step(*a, **kw))
    assert lib_eng.graph is graph
