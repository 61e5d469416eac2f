"""FrameEngine(secc2plane=...): the SECC -> plane backbone inside the step.  Graph replay (whole-step graph, torso split graphs, prepare()'s
zero-copy graphs) is bit-identical to the eager step; a second begin_planes() renders the new clip through the graphs captured for the first;
the uint8 frames equal those of an engine fed the backbone's planes directly."""
import pytest
import torch

import secc2plane_reference as ref
import real3dportrait_b200 as r3
from real3dportrait_b200 import engine, synthetic as syn

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
B = 2


def _backbone(seed=7):
    m = r3.SegFormerSECC2PlaneBackbone()
    m.load_state_dict(ref.make_params({k: v.shape for k, v in m.state_dict().items()}, seed), strict=True)
    return m.to(DEV).eval()


def _plain(**kw):
    eng = engine.FrameEngine(batch=B, sr_mode='tc', hp={'num_samples_fine': 0}, out_uint8=True, **kw)
    eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_params(seed=5))
    return eng


def _clip(seed):
    cano, src, _ = ref.make_inputs(1, 512, seed)
    return syn.make_planes(1, seed=seed).to(DEV), cano.to(DEV), src.to(DEV)


def _frames(n, seed=40):
    out = []
    for s in range(n):
        _, _, tgt = ref.make_inputs(B, 512, seed + s)
        u_c, _ = syn.make_jitter(B, 4096, 48, 0, seed=seed + s + 100)
        out.append((tgt.to(DEV), syn.make_cameras(B, seed=seed + s + 200).to(DEV), u_c.to(DEV)))
    return out


def test_rejections():
    with pytest.raises(NotImplementedError):
        engine.FrameEngine(batch=B, hp={'phase1_plane_fusion_mode': 'mul'}, secc2plane=r3.SegFormerSECC2PlaneBackbone())
    eng = _plain(secc2plane=_backbone())
    tgt, cams, u = _frames(1)[0]
    with pytest.raises(RuntimeError, match='begin_planes'):
        eng.step(None, cams, u, cond_tgt=tgt)
    with pytest.raises(ValueError):
        eng.step(syn.make_planes(B).to(DEV), cams, u, cond_tgt=tgt)
    with pytest.raises(ValueError):
        _plain().step(syn.make_planes(B).to(DEV), cams, u, cond_tgt=tgt)


@torch.no_grad()
def test_plain_engine_graphs_match_eager_and_direct_planes():
    g_eng, e_eng, direct = _plain(secc2plane=_backbone()), _plain(secc2plane=_backbone(), use_graph=False), _plain(use_graph=False)
    frames = _frames(3)
    cano, c_cano, c_src = _clip(1)
    for e in (g_eng, e_eng):
        e.begin_planes(cano, c_cano, c_src)
    bb = _backbone()
    bb.begin_clip(c_cano, c_src)
    cano_cl = r3.canonical_planes_cl(cano)
    for f in frames:
        got = g_eng.step(None, f[1], f[2], cond_tgt=f[0]).clone()
        want = e_eng.step(None, f[1], f[2], cond_tgt=f[0]).clone()
        assert got.dtype == torch.uint8 and got.shape == (B, 512, 512, 3)
        assert torch.equal(got, want)
        assert torch.equal(direct.step((cano_cl, bb.planes_cl(f[0])), f[1], f[2]), want)
    graph = g_eng.graph
    assert graph is not None
    # prepare(): zero-copy graphs over (cond_tgt, cameras, u_coarse) tuples
    assert g_eng.prepare(frames) == len(frames)
    for f in frames:
        assert torch.equal(g_eng.step(None, f[1], f[2], cond_tgt=f[0]), e_eng.step(None, f[1], f[2], cond_tgt=f[0]))
    # a second clip: refilled in place, rendered by the graphs captured for the first
    cano2, c_cano2, c_src2 = _clip(2)
    g_eng.begin_planes(cano2, c_cano2, c_src2)
    e_eng.begin_planes(cano2, c_cano2, c_src2)
    assert g_eng.graph is graph and len(g_eng.inplace) == len(frames)
    for f in frames:
        a = g_eng.step(None, f[1], f[2], cond_tgt=f[0]).clone()
        b = e_eng.step(None, f[1], f[2], cond_tgt=f[0]).clone()
        assert torch.equal(a, b)
    static = _frames(1, seed=90)[0]                                  # a fresh tuple: the whole-step graph with its static inputs
    assert torch.equal(g_eng.step(None, static[1], static[2], cond_tgt=static[0]), e_eng.step(None, static[1], static[2], cond_tgt=static[0]))
    assert g_eng.graph is graph


@torch.no_grad()
@pytest.mark.parametrize('warper_in_graph', [False, True])
def test_torso_engine_graphs_match_eager(warper_in_graph):
    hp = dict(syn.WARP_HPARAMS, htbsr_head_weight_fuse_mode='v2', num_samples_fine=48, neural_rendering_resolution=64)

    def mk(**kw):
        eng = engine.FrameEngine(batch=B, sr_mode='tc', hp=hp, torso_model=syn.StubTorsoModel(), out_uint8=True, secc2plane=_backbone(), **kw)
        eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_warp_params(seed=6, fuse_mode='v2'))
        inp = syn.make_warp_inputs(1, seed=3)
        eng.begin_clip(*(inp[k].to(DEV) for k in ('ref_torso_rgb', 'ref_bg_rgb', 'segmap', 'kp_s')))
        eng.begin_planes(*_clip(1))
        return eng
    g_eng, e_eng = mk(warper_in_graph=warper_in_graph), mk(use_graph=False)
    frames = []
    for s, (tgt, cams, _) in enumerate(_frames(2, seed=60)):
        u_c, u_f = syn.make_jitter(B, 64 * 64, 48, 48, seed=70 + s)
        kp_d = torch.rand(B, 68, 3, generator=torch.Generator().manual_seed(80 + s)) * 2 - 1
        frames.append((tgt, cams, u_c.to(DEV), u_f.to(DEV), kp_d.to(DEV)))
    for f in frames:
        a = g_eng.step(None, *f[1:4], kp_d=f[4], cond_tgt=f[0]).clone()
        b = e_eng.step(None, *f[1:4], kp_d=f[4], cond_tgt=f[0]).clone()
        assert torch.equal(a, b)
    assert g_eng.prepare(frames) == len(frames)
    for f in frames:
        assert torch.equal(g_eng.step(None, *f[1:4], kp_d=f[4], cond_tgt=f[0]), e_eng.step(None, *f[1:4], kp_d=f[4], cond_tgt=f[0]))
    g_eng.begin_planes(*_clip(2))
    e_eng.begin_planes(*_clip(2))
    for f in frames:
        assert torch.equal(g_eng.step(None, *f[1:4], kp_d=f[4], cond_tgt=f[0]), e_eng.step(None, *f[1:4], kp_d=f[4], cond_tgt=f[0]))


@torch.no_grad()
def test_step_host_takes_the_driving_image():
    eng, e_eng = _plain(secc2plane=_backbone()), _plain(secc2plane=_backbone(), use_graph=False)
    for e in (eng, e_eng):
        e.begin_planes(*_clip(1))
    tgt, cams, u = _frames(1)[0]
    h = [t.cpu().pin_memory() for t in (tgt, cams, u)]
    h_out = torch.empty(B, 512, 512, 3, dtype=torch.uint8).pin_memory()
    eng.step_host(*h, h_out)
    eng.sync_host()
    assert torch.equal(h_out, e_eng.step(None, cams, u, cond_tgt=tgt).cpu())
