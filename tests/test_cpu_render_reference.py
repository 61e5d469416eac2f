"""Self-check of tests/render_reference.py without a GPU: the float64 render reproduces the fp32 oracle to fp32 rounding, CPU simulations
of the kernels' decoders pass every bound, and a decoder that lost any one of its partial products fails them by at least 3x on the inputs
tests/test_gpu_render_conformance.py uses."""
import pytest
import torch

import render_reference as rr
from oracle import real3d_oracle as orc

DROPS = ('x_lo', 'w1_lo', 'h_lo', 'w2_lo', 'all_lo')


def _maxdiff(a, b):
    return float((a.double() - b.double()).abs().max())


@pytest.mark.parametrize('S,S_imp,wb,depth', [(7, 0, False, 0), (24, 9, False, 0), (12, 12, True, 0), (10, 0, False, 2), (9, 6, False, 4)])
def test_render64_matches_fp32_oracle(S, S_imp, wb, depth):
    """Importance, white_back, rays that miss the box, tri-grids: float64 and the fp32 oracle agree to fp32 rounding."""
    N, M, H, W = 2, 60, 20, 12
    g = torch.Generator().manual_seed(S * 10 + S_imp)
    planes = torch.randn(N, 3, 32 * max(depth, 1), H, W, generator=g)
    o, d = rr.scatter_rays(N, M, 3)
    u_c = torch.rand(N, M, S, 1, generator=g)
    u_f = torch.rand(N * M, S_imp, generator=g) if S_imp else None
    mlp = rr.transparent_decoder()
    ref = rr.render64(planes, mlp, o, d, S=S, S_imp=S_imp, white_back=wb, u_coarse=u_c, u_fine=u_f, trigrid_depth=depth)
    got = orc.render(planes, mlp, o, d, S=S, S_imp=S_imp, white_back=wb, u_coarse=u_c, u_fine=u_f, trigrid_depth=depth)
    assert torch.equal(got[3], ref[3]) and 0 < int(ref[3].sum()) < ref[3].numel()
    assert _maxdiff(got[0], ref[0]) < 3e-6 and _maxdiff(got[2], ref[2]) < 2e-6 and _maxdiff(got[1], ref[1]) < 3e-6


def _probe(scale, decoder):
    planes = rr.probe_planes(1, 64, 48, scale, seed=3)
    o, _ = rr.probe_rays(1, 4096, seed=5)
    f, q, sg = rr.gather64(planes, o, 1.0)
    f32 = orc.sample_planes(planes, o, 1.0).mean(1)
    return f, f32, rr.gather_bound(q, sg)


@pytest.mark.parametrize('scale', [1.0, 8.0, 1e-3])
def test_decoder_bound_holds_for_split_and_fp32_simulations(scale):
    for name, mlp in rr.decoder_set():
        f, f32, eg = _probe(scale, mlp)
        assert float(((f32.double() - f).abs() / eg).max()) <= 1.0
        cref, sref = rr.decode64(f, mlp)
        for split, (c, s) in ((True, rr.decode_split(f32, mlp)), (False, rr.decode_fp32(f32, mlp))):
            ec, es = rr.decoder_bound(f32, mlp, eg, split)
            rc, rs = float(((c - cref).abs() / ec).max()), float(((s - sref).abs() / es).max())
            assert rc <= 0.25 and rs <= 0.25, (name, split, rc, rs)          # the GPU's accumulation order gets the rest


def test_each_dropped_partial_product_fails_the_decoder_bound_3x():
    """On the probe inputs of the GPU suite (feature scales x1 and x8, opaque decoders), every defect exceeds the colour bound >= 3x."""
    worst = {k: 0.0 for k in DROPS}
    for scale in (1.0, 8.0):
        for name, mlp in rr.decoder_set():
            f, f32, eg = _probe(scale, mlp)
            cref, _ = rr.decode64(f, mlp)
            ec, _ = rr.decoder_bound(f32, mlp, eg, True)
            for dr in DROPS:
                c, _ = rr.decode_split(f32, mlp, dr)
                worst[dr] = max(worst[dr], float(((c - cref).abs() / ec).max()))
    print('defect error / bound:', {k: round(v, 1) for k, v in worst.items()})
    assert min(worst.values()) >= 3.0, worst


def test_each_dropped_partial_product_fails_tau_3x():
    """Whole renders with opaque decoders (the GPU suite's ragged cases): the split simulation stays within TAU_RGB / 3 and every defect
    moves rgb by >= 3 TAU_RGB."""
    worst = {k: float('inf') for k in DROPS}
    sim = 0.0
    for (N, M, S, S_imp, H, W) in [(3, 100, 7, 0, 20, 36), (2, 37, 24, 9, 48, 16), (2, 64, 48, 48, 32, 32)]:
        g = torch.Generator().manual_seed(N * 1000 + M)
        planes = torch.randn(N, 3, 32, H, W, generator=g)
        o, d = rr.scatter_rays(N, M, N * 1000 + M + 1)
        u_c = torch.rand(N, M, S, 1, generator=g)
        u_f = torch.rand(N * M, S_imp, generator=g) if S_imp else None
        for name, mlp in rr.decoder_set()[:2]:
            ref = rr.render64(planes, mlp, o, d, S=S, S_imp=S_imp, u_coarse=u_c, u_fine=u_f)
            run = lambda drop: rr.render64(planes, mlp, o, d, S=S, S_imp=S_imp, u_coarse=u_c, u_fine=u_f,
                                           decode=lambda f: rr.decode_split(f, mlp, drop))
            sim = max(sim, _maxdiff(run(None)[0], ref[0]))
            for dr in DROPS:
                worst[dr] = min(worst[dr], _maxdiff(run(dr)[0], ref[0]))
    print(f'split simulation {sim:.2e}; smallest defect error / TAU_RGB:', {k: round(v / rr.TAU_RGB, 1) for k, v in worst.items()})
    assert sim <= rr.TAU_RGB / 3
    assert min(worst.values()) >= 3 * rr.TAU_RGB, worst
