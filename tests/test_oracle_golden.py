"""Pins the CPU oracle (oracle/real3d_oracle.py) against fixtures produced by the reference's own modules
(tests/golden/make_golden.py).  CPU only."""
import pytest
import torch

from oracle import real3d_oracle as orc
from real3dportrait_b200 import synthetic as syn
from conftest import mlp_of

TOL = 2e-5          # fp32 re-association noise between two CPU implementations


def _maxdiff(a, b):
    return float((a.float() - b.float()).abs().max())


@pytest.mark.parametrize('name', ['render_small', 'render_small_imp', 'render_small_wb'])
def test_render_small(golden, name):
    g = golden(name)
    c2w, K = syn.split_camera(g['camera'])
    o, d = orc.gen_rays(c2w, K, g['res'])
    assert _maxdiff(o, g['ray_o']) < 1e-6 and _maxdiff(d, g['ray_d']) < 1e-6
    rgb, depth, wsum, valid = orc.render(g['planes'], mlp_of(g), g['ray_o'], g['ray_d'], S=g['S'], S_imp=g['S_imp'],
                                         white_back=bool(g['white_back']), u_coarse=g['u_coarse'], u_fine=g.get('u_fine'))
    assert torch.equal(valid, g['valid'])
    assert _maxdiff(rgb, g['rgb']) < TOL
    assert _maxdiff(wsum, g['wsum']) < TOL
    assert _maxdiff(depth, g['depth']) < 1e-4


def test_sample_small(golden):
    g = golden('sample_small')
    planes = golden('render_small')['planes']                 # the fixtures share their planes
    f = orc.sample_planes(planes, g['coords'], 1.0)
    assert _maxdiff(f, g['feat']) < 1e-5
    assert _maxdiff(orc.sample_planes_lib(planes, g['coords'], 1.0), g['feat']) < 1e-5
    rgb, sigma = orc.decode(f, mlp_of(g))
    assert _maxdiff(rgb, g['rgb']) < TOL and _maxdiff(sigma, g['sigma']) < 1e-4


def test_sr_layers(golden):
    g = golden('sr_layers')
    for name, up in (('up', 2), ('same', 1)):
        p = {k[len(name) + 1:]: v for k, v in g.items() if k.startswith(name + '.')}
        y = orc.synthesis_layer(g['x'], g['w'], p, '', up)
        assert _maxdiff(y, g[name + '.y']) < 1e-4
    p = {k[6:]: v for k, v in g.items() if k.startswith('torgb.')}
    assert _maxdiff(orc.to_rgb(g['x'], g['w'], p, ''), g['torgb.y']) < 1e-4
    assert _maxdiff(orc.upsample2x(g['img']), g['img_up']) < 1e-5
    assert _maxdiff(orc.resize_bilinear(g['x'], 24), g['x_resized']) < 1e-5


@pytest.mark.parametrize('name', ['render_full48', 'render_full48_48'])
def test_render_full(golden, name):
    g = golden(name)
    planes, cam = syn.make_planes(1, seed=0), syn.make_cameras(1, seed=1)
    u_c, u_f = syn.make_jitter(1, 4096, 48, g['S_imp'], seed=2)
    c2w, K = syn.split_camera(cam)
    o, d = orc.gen_rays(c2w, K, 64)
    assert _maxdiff(o[:, ::97], g['ray_o']) < 1e-6 and _maxdiff(d[:, ::97], g['ray_d']) < 1e-6
    rgb, depth, wsum, valid = orc.render(planes, syn.make_decoder_params(seed=4), o, d, S=48, S_imp=g['S_imp'],
                                         u_coarse=u_c, u_fine=u_f, lib=True)
    assert bool(valid.all())
    assert _maxdiff(rgb, g['rgb']) < TOL
    assert _maxdiff(wsum, g['wsum']) < TOL
    assert _maxdiff(depth, g['depth']) < 1e-4


def test_sr_full(golden):
    g = golden('render_full48')
    fimg = orc.feature_image(g['rgb'], 64)
    img = orc.superres(fimg[:, :3], fimg, torch.ones(1, 14, 512), syn.make_sr_params(seed=5))[..., ::2, ::2]
    ref = golden('sr_full')['image_s2']
    assert _maxdiff(img, ref) < 2e-4 * float(ref.abs().max())


def test_sr_warp_full(golden):
    """Torso head (SuperresolutionHybrid8XDC_Warp, fuse mode v2) at N=1 vs the reference class run with the stub torso model."""
    g = golden('render_full48')
    fimg = orc.feature_image(g['rgb'], 64)
    wimg = orc.feature_image(g['wsum'], 64)
    inp = syn.make_warp_inputs(1, seed=7)
    # the antialiased 1/2 resize restated == the library op the reference calls
    lib = torch.nn.functional.interpolate(inp['ref_bg_rgb'], size=(256, 256), mode='bilinear', align_corners=False, antialias=True)
    assert _maxdiff(orc.aa_down2(inp['ref_bg_rgb']), lib) < 1e-5
    img, _ = orc.superres_warp(fimg[:, :3], fimg, torch.ones(1, 14, 512), inp['ref_torso_rgb'], inp['ref_bg_rgb'], wimg, inp['segmap'],
                               inp['kp_s'], inp['kp_d'], syn.make_sr_warp_params(seed=6), syn.StubTorsoModel())
    img, ref = img[..., ::2, ::2], golden('sr_warp_full')['image_s2']
    assert _maxdiff(img, ref) < 2e-4 * float(ref.abs().max())


@pytest.mark.parametrize('mode', ['v1', 'v3'])
def test_sr_warp_other_fuse_modes(golden, mode):
    """htbsr_head_weight_fuse_mode v1 (plain alpha blend) and v3 (conv-predicted head mask + batch quantile threshold), sr_with_ref.py:96-104,126-152,
    vs the reference class in that mode (stub torso model; stretched weights image stored in the fixture)."""
    g, fx = golden('render_full48'), golden('sr_warp_' + mode)
    fimg = orc.feature_image(g['rgb'], 64)
    inp = syn.make_warp_inputs(1, seed=7)
    img, _ = orc.superres_warp(fimg[:, :3], fimg, torch.ones(1, 14, 512), inp['ref_torso_rgb'], inp['ref_bg_rgb'], fx['weights_img'], inp['segmap'],
                               inp['kp_s'], inp['kp_d'], syn.make_sr_warp_params(seed=6, fuse_mode=mode), syn.StubTorsoModel(), mode=mode)
    img, ref = img[..., ::2, ::2], fx['image_s2']
    assert _maxdiff(img, ref) < 2e-4 * float(ref.abs().max())



def test_trigrid_sample_and_render(golden):
    """`trigrid_v2` (depth-3 tri-grids, 3-D grid_sample; renderer.py:78-89) against the reference's sample_from_trigrids / ImportanceRenderer."""
    g = golden('render_trigrid')
    D = g['depth_slices']
    grids = torch.randn(2, 3, 32 * D, 32, 32, generator=torch.Generator().manual_seed(g['planes_seed']))
    f = orc.sample_trigrids(grids, g['coords'], 1.0, D)
    assert _maxdiff(f, g['feat']) < 1e-5
    assert _maxdiff(orc.sample_trigrids_lib(grids, g['coords'], 1.0, D), g['feat']) < 1e-5
    c2w, K = syn.split_camera(g['camera'])
    o, d = orc.gen_rays(c2w, K, g['res'])
    for tag, S_imp in (('a', 0), ('b', 12)):
        rgb, depth, wsum, valid = orc.render(grids, mlp_of(g), o, d, S=g['S'], S_imp=S_imp, u_coarse=g[tag + '.u_coarse'],
                                             u_fine=g.get(tag + '.u_fine'), trigrid_depth=D)
        assert torch.equal(valid, g[tag + '.valid'])
        assert _maxdiff(rgb, g[tag + '.rgb']) < TOL and _maxdiff(wsum, g[tag + '.wsum']) < TOL and _maxdiff(depth, g[tag + '.depth']) < 1e-4


def test_large_sr(golden):
    """SuperresolutionHybrid8XDC(large_sr=True) (ResBlock2d + to_rgb tails, superresolution.py:263-345) against the reference class."""
    fimg = orc.feature_image(golden('render_full48')['rgb'], 64)
    out = orc.superres_large(fimg[:, :3], fimg, torch.ones(1, 14, 512), syn.make_sr_large_params(seed=8, n_res=2), 2)[..., ::2, ::2]
    ref = golden('sr_large')['image_s2']
    assert _maxdiff(out, ref) < 1e-4 * float(ref.abs().max())
