"""The plain-C restatement (oracle/r3dp_oracle.c) against the reference fixtures and the torch oracle.  CPU only."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import real3d_oracle as orc
from real3dportrait_b200 import synthetic as syn
from conftest import mlp_of, ROOT


@pytest.fixture(scope='module')
def clib():
    subprocess.run(['make', '-C', os.path.join(ROOT, 'oracle'), '-s'], check=True)
    return C.CDLL(os.path.join(ROOT, 'oracle', '_build', 'libr3dp_oracle.so'))


def _p(t):
    return t.ctypes.data_as(C.c_void_p)


def _c_render(lib, planes, mlp, o, d, S, Ni, wb, u_c, u_f):
    N, _, _, H, W = planes.shape
    M = o.shape[1]
    a = lambda t: np.ascontiguousarray(t.numpy(), dtype=np.float32)
    pl, ro, rd, uc = a(planes), a(o), a(d), a(u_c)
    uf = a(u_f) if u_f is not None else np.zeros(1, np.float32)
    w1, b1, w2, b2 = (a(mlp[k]) for k in ('net.0.weight', 'net.0.bias', 'net.2.weight', 'net.2.bias'))
    rgb, depth, wsum = np.zeros((N, M, 32), np.float32), np.zeros((N, M, 1), np.float32), np.zeros((N, M, 1), np.float32)
    valid = np.zeros((N, M, 1), np.uint8)
    lib.orc_render(_p(pl), N, H, W, _p(ro), _p(rd), M, S, Ni, C.c_float(1.0), int(wb), _p(uc), _p(uf), _p(w1), _p(b1), _p(w2), _p(b2),
                   _p(rgb), _p(depth), _p(wsum), _p(valid))
    return torch.from_numpy(rgb), torch.from_numpy(depth), torch.from_numpy(wsum), torch.from_numpy(valid.astype(bool))


@pytest.mark.parametrize('name', ['render_small', 'render_small_imp', 'render_small_wb'])
def test_c_render_vs_reference_fixture(clib, golden, name):
    g = golden(name)
    rgb, depth, wsum, valid = _c_render(clib, g['planes'], mlp_of(g), g['ray_o'], g['ray_d'], g['S'], g['S_imp'], bool(g['white_back']),
                                        g['u_coarse'], g.get('u_fine'))
    assert torch.equal(valid, g['valid'])
    assert float((rgb - g['rgb']).abs().max()) < 2e-5 and float((wsum - g['wsum']).abs().max()) < 2e-5
    assert float((depth - g['depth']).abs().max()) < 1e-4


def test_c_rays_and_gather_vs_reference_fixture(clib, golden):
    g = golden('render_small')
    c2w, K = syn.split_camera(g['camera'])
    N, res = c2w.shape[0], g['res']
    ro, rd = np.zeros((N, res * res, 3), np.float32), np.zeros((N, res * res, 3), np.float32)
    clib.orc_gen_rays(_p(np.ascontiguousarray(c2w.numpy().reshape(N, 16))), _p(np.ascontiguousarray(K.numpy().reshape(N, 9))), N, res, _p(ro), _p(rd))
    assert float(np.abs(ro - g['ray_o'].numpy()).max()) < 1e-6 and float(np.abs(rd - g['ray_d'].numpy()).max()) < 1e-6
    s = golden('sample_small')
    pl, co = np.ascontiguousarray(g['planes'].numpy()), np.ascontiguousarray(s['coords'].numpy())     # the fixtures share their planes
    out = np.zeros((2, 3, 500, 32), np.float32)
    clib.orc_sample_planes(_p(pl), 2, 32, 32, _p(co), 500, C.c_float(1.0), _p(out))
    assert float(np.abs(out - s['feat'].numpy()).max()) < 1e-5


def test_c_vs_torch_oracle_random_rays(clib):
    """Same ragged case the GPU suite runs: rays that partly miss the box, importance pass with S_imp != S."""
    g = torch.Generator().manual_seed(2037)
    N, M, S, Ni, H, W = 2, 37, 24, 9, 48, 16
    planes = torch.randn(N, 3, 32, H, W, generator=g)
    o = torch.tensor([0.0, 0.0, 1.6]).expand(N, M, 3).contiguous() + 0.05 * torch.randn(N, M, 3, generator=g)
    d = torch.nn.functional.normalize(torch.tensor([0.0, 0.0, -1.0]) + 0.45 * torch.randn(N, M, 3, generator=g), dim=-1)
    u_c, u_f = torch.rand(N, M, S, 1, generator=g), torch.rand(N * M, Ni, generator=g)
    mlp = syn.make_decoder_params(seed=4)
    ref = orc.render(planes, mlp, o, d, S=S, S_imp=Ni, u_coarse=u_c, u_fine=u_f)
    got = _c_render(clib, planes, mlp, o, d, S, Ni, False, u_c, u_f)
    assert torch.equal(got[3], ref[3])
    assert float((got[0] - ref[0]).abs().max()) < 2e-5 and float((got[2] - ref[2]).abs().max()) < 2e-5
