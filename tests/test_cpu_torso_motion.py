"""torso_motion='cuda' without a GPU: option validation, the unchanged state_dict, the float64 folding of the motion-field estimator against the
reference's own sub-blocks (where oracle/_ref is staged), the 3-D nearest-up parity composition, and a float64 restatement of the estimator's
input construction and deformation at a toy size."""
import pytest
import torch
import torch.nn.functional as F

import real3dportrait_b200 as r3
from real3dportrait_b200 import synthetic as syn, torso_warp as tw
import torso_warper_ref as twr


def _head(**kw):
    return r3.SuperresolutionHybrid8XDC_Warp(channels=32, img_resolution=512, sr_num_fp16_res=0, sr_antialias=True, hp=syn.WARP_HPARAMS, **kw)


def test_option_validation():
    with pytest.raises(ValueError):
        _head(torso_motion='cuda')                                   # needs torso_stage2='cuda'
    with pytest.raises(ValueError):
        _head(torso_stage2='cuda', torso_motion='cudnn')
    m = _head(torso_stage2='cuda', torso_motion='cuda')
    assert m.torso_motion == 'cuda'
    with pytest.raises(ValueError):
        m.set_torso_stage2('torch')                                  # the estimator on the kernels needs the restated stage 1
    m.set_torso_motion('torch')
    m.set_torso_stage2('torch')
    with pytest.raises(NotImplementedError):
        r3.SuperresolutionHybrid8XDC_Warp(channels=32, img_resolution=512, sr_num_fp16_res=0, sr_antialias=True, torso_motion='cuda',
                                          hp=dict(syn.WARP_HPARAMS, torso_model_version='v1'))
    assert _head().torso_motion == 'torch'


def _ref_mfe_cls():
    if twr.ref_classes() is None:
        pytest.skip('the reference warper modules are not staged under oracle/_ref')
    from modules.real3d.facev2v_warp.network2 import MotionFieldEstimator
    return MotionFieldEstimator


def test_shape_validation():
    MFE = _ref_mfe_cls()
    assert tw.estimator_shape_error(MFE('standard', 34, 4)) is None
    assert tw.estimator_shape_error(MFE('standard', 34, 9)) is None
    assert tw.estimator_shape_error(MFE('small', 34, 4)) is not None
    assert tw.estimator_shape_error(MFE('standard', 34, 4, predict_multiref_occ=False)) is not None
    assert tw.estimator_shape_error(MFE('standard', 34, 6)) is not None
    with pytest.raises(NotImplementedError):
        tw.MotionWeights(MFE('small', 34, 4), split=False)


def test_fold_kp9_layout():
    """torso_kp_num 9: 50 input channels padded to 64, a 128-channel fuser input (input | pad | up output | head features), 10 mask logits."""
    MFE = _ref_mfe_cls()
    w = tw.MotionWeights(twr.randomize(MFE('standard', 34, 9), seed=3), split=False)
    assert (w.K, w.c0, w.P0, w.CF) == (9, 50, 64, 128)
    assert w.down[0][0].shape[-1] == 64 and w.fuser[0].shape[-1] == 128 and w.mask[2:] == (10, 16)
    fu = twr.randomize(MFE('standard', 34, 9), seed=3).tgt_head_fuser.weight.detach()
    got = w.fuser[0][0].double()                                    # [343, 32, 128]
    ref = fu.double().permute(2, 3, 4, 0, 1).reshape(343, 32, 114)
    assert torch.equal(got[..., 50:64], torch.zeros_like(got[..., 50:64]))
    assert float((got[..., :50] - ref[..., :50]).abs().max()) <= 2 ** -11 * float(ref.abs().max())
    assert float((got[..., 64:] - ref[..., 50:]).abs().max()) <= 2 ** -11 * float(ref.abs().max())


def test_state_dict_unchanged():
    a, b = _head(torso_stage2='cuda'), _head(torso_stage2='cuda', torso_motion='cuda')
    assert list(a.state_dict()) == list(b.state_dict())


def test_compose_nearest_up3d():
    g = torch.Generator().manual_seed(0)
    w = torch.randn(5, 3, 3, 3, 3, generator=g, dtype=torch.float64)
    x = torch.randn(2, 3, 4, 5, 6, generator=g, dtype=torch.float64)
    ref = F.conv3d(F.interpolate(x, scale_factor=(1, 2, 2), mode='nearest'), w, padding=1)
    G = tw.compose_nearest_up3d(w)
    out = torch.zeros_like(ref)
    for p in range(2):
        for q in range(2):
            out[..., p::2, q::2] = F.conv3d(F.pad(x, (1 - q, q, 1 - p, p, 1, 1)), G[p * 2 + q])
    assert float((out - ref).abs().max()) < 1e-12


def test_folding_matches_reference_blocks():
    """The float64 folds (conv + eval BatchNorm, nearest-up phases, the pre-activation ResBlock2D) reproduce the reference's sub-blocks."""
    MFE = _ref_mfe_cls()
    torch.manual_seed(0)
    mfe = twr.randomize(MFE('standard', 34, 4), seed=7).double()
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        x = torch.randn(1, 64, 4, 8, 8, generator=g, dtype=torch.float64)
        w, b = tw.fold_cna(mfe.down[1].layers[0])
        assert float((torch.relu(F.conv3d(x, w, b, padding=1)) - mfe.down[1].layers[0](x)).abs().max()) < 1e-10
        x = torch.randn(1, 128, 4, 4, 4, generator=g, dtype=torch.float64)
        w, b = tw.fold_cna(mfe.up[3].layers[1])
        G = tw.compose_nearest_up3d(w)
        out = torch.zeros(1, 64, 4, 8, 8, dtype=torch.float64)
        for p in range(2):
            for q in range(2):
                out[..., p::2, q::2] = F.conv3d(F.pad(x, (1 - q, q, 1 - p, p, 1, 1)), G[p * 2 + q], b)
        assert float((torch.relu(out) - mfe.up[3](x)).abs().max()) < 1e-10
        enc = mfe.tgt_head_encoder
        x = torch.randn(1, 4, 16, 16, generator=g, dtype=torch.float64)
        w, b = tw.fold_cna(enc[0])
        h = torch.relu(F.conv2d(x, w, b, padding=3))
        assert float((h - enc[0](x)).abs().max()) < 1e-10
        rb = enc[1]
        nac1, nac2 = rb.layers[0].layers, rb.layers[1].layers
        s1, t1 = tw.bn_affine(nac1[0])
        s2, t2 = tw.bn_affine(nac2[0])
        a = torch.relu(h * s1[:, None, None] + t1[:, None, None])
        a = torch.relu(F.conv2d(a, nac1[2].weight * s2[:, None, None, None], nac1[2].bias * s2 + t2, padding=1))
        y = h + F.conv2d(a, nac2[2].weight, nac2[2].bias, padding=1)
        assert float((y - rb(h)).abs().max()) < 1e-10


def _grid(D, H, W):
    lin = lambda n: 2 * (torch.arange(n, dtype=torch.float64) / (n - 1)) - 1        # noqa: E731
    z, y, x = torch.meshgrid(lin(D), lin(H), lin(W), indexing='ij')
    return torch.stack([x, y, z], -1)


def _trilinear_zeros(vol, p):
    """vol [C,D,H,W], p (x, y, z) in [-1, 1] (align_corners=True, zero padding) -> [C]; written per corner."""
    C, D, H, W = vol.shape
    ix, iy, iz = (p[0] + 1) / 2 * (W - 1), (p[1] + 1) / 2 * (H - 1), (p[2] + 1) / 2 * (D - 1)
    x0, y0, z0 = int(torch.floor(ix)), int(torch.floor(iy)), int(torch.floor(iz))
    out = torch.zeros(C, dtype=torch.float64)
    for dz in (0, 1):
        for dy in (0, 1):
            for dx in (0, 1):
                xx, yy, zz = x0 + dx, y0 + dy, z0 + dz
                if 0 <= xx < W and 0 <= yy < H and 0 <= zz < D:
                    wgt = (1 - abs(ix - xx)) * (1 - abs(iy - yy)) * (1 - abs(iz - zz))
                    out += wgt * vol[:, zz, yy, xx]
    return out


def test_input_and_deformation_restatement():
    """The estimator's input channels (k*5 + j) and the softmax-weighted deformation, restated voxel by voxel in float64, against the
    tensor formulas the GPU tests use (F.grid_sample, broadcast Gaussians); toy size 3 x 4 x 5, K = 2."""
    g = torch.Generator().manual_seed(2)
    K, D, H, W = 2, 3, 4, 5
    vol = torch.randn(4, D, H, W, generator=g, dtype=torch.float64)
    kp_s, kp_d = 0.9 * (2 * torch.rand(K, 3, generator=g, dtype=torch.float64) - 1), 0.9 * (2 * torch.rand(K, 3, generator=g, dtype=torch.float64) - 1)
    grid = _grid(D, H, W)
    sm = torch.stack([grid] + [grid - kp_d[k] + kp_s[k] for k in range(K)])                      # [K+1,D,H,W,3]
    deformed = F.grid_sample(vol[None].expand(K + 1, -1, -1, -1, -1), sm, align_corners=True)     # [K+1,4,D,H,W]
    gauss = lambda kp: torch.exp(-0.5 * ((grid - kp) ** 2).sum(-1) / 0.01)                       # noqa: E731
    logits = torch.randn(K + 1, D, H, W, generator=g, dtype=torch.float64)
    deform = (sm * torch.softmax(logits, 0)[..., None]).sum(0)
    for d in range(D):
        for h in range(H):
            for w in range(W):
                p = grid[d, h, w]
                m = torch.softmax(logits[:, d, h, w], 0)
                acc = m[0] * p
                for k in range(K + 1):
                    q = p if k == 0 else p - kp_d[k - 1] + kp_s[k - 1]
                    assert float((_trilinear_zeros(vol, q) - deformed[k, :, d, h, w]).abs().max()) < 1e-12
                    if k > 0:
                        hm = torch.exp(-0.5 * ((p - kp_d[k - 1]) ** 2).sum() / 0.01) - torch.exp(-0.5 * ((p - kp_s[k - 1]) ** 2).sum() / 0.01)
                        assert abs(float(hm - (gauss(kp_d[k - 1]) - gauss(kp_s[k - 1]))[d, h, w])) < 1e-12
                        acc = acc + m[k] * q
                assert float((acc - deform[d, h, w]).abs().max()) < 1e-12
