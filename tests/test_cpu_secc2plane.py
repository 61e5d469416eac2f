"""SegFormerSECC2PlaneBackbone on the host: the float64 restatement against the reference's own fixture, state_dict compatibility with the
reference class, the float64 folds, the flip index map and the rejected configurations."""
import os

import pytest
import torch
import torch.nn.functional as F

import secc2plane_reference as ref
from conftest import load_golden
from real3dportrait_b200 import secc2plane as sp
from real3dportrait_b200.secc2plane import SegFormerSECC2PlaneBackbone

REF_ROOT = os.environ.get('R3DP_REFERENCE', '/root/reference')
HAS_REF = os.path.isdir(os.path.join(REF_ROOT, 'modules', 'real3d'))


def _params(m, seed):
    return ref.make_params({k: v.shape for k, v in m.state_dict().items()}, seed)


def test_restatement_matches_reference_fixture():
    g = load_golden('secc2plane_small')
    m = SegFormerSECC2PlaneBackbone()
    sd = ref.to64(_params(m, int(g['param_seed'])))
    cano, src, tgt = ref.make_inputs(1, int(g['size']), int(g['input_seed']))
    with torch.no_grad():
        out = ref.forward(sd, torch.cat([cano, src, tgt], 1).double())
    want = g['planes_s2'].double()
    got = out[..., ::2, ::2]
    assert got.shape == want.shape
    err = float((got - want).abs().max())
    assert err <= 1e-6 * float(want.abs().max()) + 1e-7, err     # float32 storage of a float64 run


@pytest.mark.skipif(not HAS_REF, reason='needs a reference checkout (R3DP_REFERENCE)')
@pytest.mark.parametrize('mode', ['cano_src_tgt', 'cano_tgt'])
def test_state_dict_round_trip_with_reference_class(mode):
    Ref = ref.reference_class(REF_ROOT)
    theirs = Ref(mode='b0', out_channels=96, pncc_cond_mode=mode)
    ours = SegFormerSECC2PlaneBackbone(pncc_cond_mode=mode)
    assert {k: tuple(v.shape) for k, v in theirs.state_dict().items()} == {k: tuple(v.shape) for k, v in ours.state_dict().items()}
    sd = _params(ours, 3)
    ours.load_state_dict(sd, strict=True)
    theirs.load_state_dict(ours.state_dict(), strict=True)
    ours2 = SegFormerSECC2PlaneBackbone(pncc_cond_mode=mode)
    ours2.load_state_dict(theirs.state_dict(), strict=True)
    for k, v in ours2.state_dict().items():
        assert torch.equal(v, sd[k]), k


def test_prenet_split_equals_full_prenet():
    m = SegFormerSECC2PlaneBackbone()
    sd = ref.to64(_params(m, 5))
    m.load_state_dict(_params(m, 5))
    cano, src, tgt = (t.double() for t in ref.make_inputs(2, 64, 2))
    full = ref.prenet(sd, torch.cat([cano.expand(2, -1, -1, -1), src.expand(2, -1, -1, -1), tgt], 1))
    w, b = sp.fold_prenet(m.prenet.weight, m.prenet.bias)
    base = torch.einsum('cj,njhw->nchw', w[:, :6], torch.cat([cano, src], 1)) + b[None, :, None, None]
    split = base + torch.einsum('cj,njhw->nchw', w[:, 6:], tgt)
    assert float((split - full).abs().max()) < 1e-12


def test_bn_and_head_fold_equal_unfolded_head():
    m = SegFormerSECC2PlaneBackbone()
    m.load_state_dict(_params(m, 9))
    sd = ref.to64(m.state_dict())
    g = torch.Generator().manual_seed(0)
    feats = [torch.randn(2, c, s, s, generator=g, dtype=torch.float64) for c, s in zip(ref.EMBED, (32, 16, 8, 4))]
    want = ref.head(sd, feats)
    G, bias = sp.fold_head(m.fuse_head)
    acc = bias[None, :, None, None].expand(2, -1, 32, 32).clone()
    for Gi, c in zip(G, feats):
        t = torch.einsum('oc,nchw->nohw', Gi, c)
        acc += F.interpolate(t, size=(32, 32), mode='bilinear', align_corners=False) if t.shape[-1] != 32 else t
    got = torch.relu(acc)
    assert float((got - want).abs().max()) < 1e-10 * float(want.abs().max())
    # the BN fold alone
    wf, shift = sp.fold_bn(m.fuse_head.linear_fuse.conv.weight, m.fuse_head.linear_fuse.bn)
    z = torch.randn(3, 1024, 2, 2, generator=g, dtype=torch.float64)
    p = 'fuse_head.linear_fuse.bn'
    bn = F.batch_norm(F.conv2d(z, sd['fuse_head.linear_fuse.conv.weight']), sd[p + '.running_mean'], sd[p + '.running_var'], sd[p + '.weight'],
                      sd[p + '.bias'], False, 0.0, 1e-5)
    assert float((torch.einsum('oc,nchw->nohw', wf, z) + shift[None, :, None, None] - bn).abs().max()) < 1e-12


def test_mirrored_taps_give_mirrored_conv():
    """The last conv runs on mirrored images with mirrored taps; that is the mirrored conv (zero padding is symmetric)."""
    g = torch.Generator().manual_seed(1)
    x = torch.randn(1, 8, 10, 10, generator=g, dtype=torch.float64)
    w = torch.randn(6, 8, 3, 3, generator=g, dtype=torch.float64)
    y = F.conv2d(x, w, padding=1)
    assert torch.allclose(F.conv2d(x.flip(2), w.flip(2), padding=1), y.flip(2), atol=1e-12)
    assert torch.allclose(F.conv2d(x.flip(2, 3), w.flip(2, 3), padding=1), y.flip(2, 3), atol=1e-12)
    # the align_corners=True x2 upsample commutes with the mirrors too
    u = F.interpolate(x, scale_factor=2.0, mode='bilinear', align_corners=True)
    assert torch.allclose(F.interpolate(x.flip(2, 3), scale_factor=2.0, mode='bilinear', align_corners=True), u.flip(2, 3), atol=1e-12)


def test_plane_index_map_matches_reference_flips():
    H = W = 6
    conv_out = torch.arange(96 * H * W, dtype=torch.float64).reshape(1, 96, H, W)
    p = conv_out.view(1, 3, 32, H, W)
    planes = torch.stack([torch.flip(p[:, 0], [2]), torch.flip(p[:, 1], [2]), torch.flip(p[:, 2], [2, 3])], 1)
    where = sp.plane_index_map(H, W)
    for co in (0, 31, 32, 63, 64, 95):
        for y in range(H):
            for x in range(W):
                pl, c, yy, xx = where(co, y, x)
                assert planes[0, pl, c, yy, xx] == conv_out[0, co, y, x]


@pytest.mark.parametrize('kw', [{'mode': 'b1'}, {'mode': 'b3'}, {'out_channels': 96 * 3}, {'out_channels': 32}])
def test_unbuilt_configurations_raise(kw):
    with pytest.raises(NotImplementedError):
        SegFormerSECC2PlaneBackbone(**kw)


def test_cpu_tensor_and_bad_shapes_raise():
    m = SegFormerSECC2PlaneBackbone()
    with pytest.raises(RuntimeError, match='CUDA'):
        m(torch.zeros(1, 9, 128, 128))
    with pytest.raises(RuntimeError, match='CUDA'):
        m.begin_clip(torch.zeros(1, 3, 64, 64), torch.zeros(1, 3, 64, 64))
    with pytest.raises(RuntimeError, match='CUDA'):
        sp.canonical_planes_cl(torch.zeros(1, 3, 32, 8, 8))
    # shapes: H == W, a multiple of 32, 32 <= H <= 512 (every attention sees at most 256 keys); 9 channels in 'cano_src_tgt'
    for shape in [(1, 9, 128, 96), (1, 9, 100, 100), (1, 9, 544, 544), (1, 9, 16, 16), (1, 6, 128, 128), (9, 128, 128)]:
        with pytest.raises(ValueError):
            m(torch.zeros(shape))
    m6 = SegFormerSECC2PlaneBackbone(pncc_cond_mode='cano_tgt')
    with pytest.raises(ValueError):
        m6(torch.zeros(1, 9, 128, 128))
    with pytest.raises(RuntimeError, match='begin_clip'):
        m.planes_cl(torch.zeros(1, 3, 128, 128))
