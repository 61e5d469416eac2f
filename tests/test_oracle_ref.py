"""The oracle computes what the reference's own modules compute (rays -> ImportanceRenderer -> OSGDecoder, small size, seeded
inputs): fixture render_ref_head.npz, written by tests/golden/make_golden.py from the reference project."""
import torch

from oracle import real3d_oracle as orc
from real3dportrait_b200 import synthetic as syn


def test_stock_reference_render_matches_oracle_small(golden):
    g = golden('render_ref_head')
    N, res, S = 1, 16, 12
    planes = syn.make_planes(N, h=32, w=32, seed=0)
    cam = syn.make_cameras(N, seed=1)
    mlp = syn.make_decoder_params(seed=4)
    for S_imp in (0, 12):
        u_c, u_f = syn.make_jitter(N, res * res, S, S_imp, seed=2)
        feat, wsum, valid = g[f'imp{S_imp}.feat'], g[f'imp{S_imp}.wsum'], g[f'imp{S_imp}.valid']
        c2w, K = syn.split_camera(cam)
        o, d = orc.gen_rays(c2w, K, res)
        ref = orc.render(planes, mlp, o, d, S=S, S_imp=S_imp, u_coarse=u_c, u_fine=u_f)
        assert float((feat - ref[0]).abs().max()) < 2e-5 and float((wsum - ref[2]).abs().max()) < 2e-5
        assert torch.equal(valid, ref[3])
