"""SegFormerSECC2PlaneBackbone(precision='tc_exact') on the host: the launch plan (one launch per `tc` launch, the split entry point of each
stage, buffers passed as fp32 or split rows only), the precision argument, the state_dict, and the split weight packing bit for bit against
a float64 fold written from the state_dict."""
import pytest
import torch

import secc2plane_exact_reference as xref
import secc2plane_reference as ref
from real3dportrait_b200 import _capi as capi, secc2plane as sp
from real3dportrait_b200.secc2plane import SegFormerSECC2PlaneBackbone

SIZES = [(512, 4), (512, 1), (480, 3), (96, 3), (32, 3)]
#: tc entry point -> the ones its stage may use in tc_exact
EXACT_OF = {'r3dp_sp_embed': {'r3dp_sp_embed'},
            'r3dp_sp_layernorm': {'r3dp_sp_layernorm', 'r3dp_hb_layernorm', 'r3dp_sp_layernorm_split'},
            'r3dp_sp_patches': {'r3dp_sp_patches_split'}, 'r3dp_sp_attention': {'r3dp_sp_attention_split'},
            'r3dp_sp_dwconv_gelu': {'r3dp_sp_dwconv_gelu_split'}, 'r3dp_sp_head_fuse': {'r3dp_sp_head_fuse_split'},
            'r3dp_sp_leaky': {'r3dp_sp_leaky_split'}, 'r3dp_sp_upsample2_flip': {'r3dp_sp_upsample2_flip_split'},
            'r3dp_sr_tc_conv': {'r3dp_sr_tcx_conv'}, 'r3dp_mf_conv3d': {'r3dp_mf_conv3d'}}


def _module(seed=3, **kw):
    m = SegFormerSECC2PlaneBackbone(**kw)
    m.load_state_dict(ref.make_params({k: v.shape for k, v in m.state_dict().items()}, seed), strict=True)
    return m


@pytest.mark.parametrize('H,B', SIZES)
@pytest.mark.parametrize('cin', [9, 6])
def test_plan_mirrors_the_tc_plan_stage_by_stage(H, B, cin):
    tc, ex = ref.launch_plan(H, B, cin), xref.launch_plan_exact(H, B, cin)
    assert len(ex) == len(tc)
    for (tag, f, a), (xtag, xf, xa) in zip(tc, ex):
        assert xtag == tag
        assert xf in EXACT_OF[f], (tag, f, xf)
        if f == 'r3dp_mf_conv3d':
            d = dict(zip(('xs', 'xlo', 'cin'), xa[:3]))
            assert xa[-1] == 1 and d['xs'] == 2 * d['cin'] and d['xlo'] == d['cin'], (tag, xa)        # split operands
            assert xa[3:14] == a[3:14], tag                                                          # same grid, taps, couts
            ys, yc0, ylo, out_f32 = xa[14:18]
            assert out_f32 == 1 or (ylo == a[14] and ys == 2 * a[14]), tag                         # fp32 or split output
        if xf == 'r3dp_sp_layernorm':
            assert tag.endswith('.pe_norm'), tag                                                     # fp32 output only
    n = {f: sum(1 for _, g, _ in ex if g == f) for f in {g for _, g, _ in ex}}
    levels = 4
    assert n['r3dp_sp_attention_split'] == n['r3dp_sp_dwconv_gelu_split'] == 2 * levels
    assert n['r3dp_sp_layernorm_split'] == 2 * 2 * levels                                           # norm2, next norm1 / final norm
    assert n['r3dp_hb_layernorm'] == levels + 2 * 3                                                  # first norm1, 6 sr_norms
    assert n['r3dp_sp_patches_split'] == 3 + 2 * 3
    h1 = (H - 1) // 4 + 1
    assert n.get('r3dp_sr_tcx_conv', 0) == (3 if h1 % 128 == 0 else 0)
    assert n.get('r3dp_sp_leaky_split', 0) == (0 if h1 % 128 == 0 else 3)


@pytest.mark.parametrize('H,B', SIZES)
def test_plan_buffer_flow(H, B):
    """Every buffer a launch reads was written earlier in the same form and width; nothing crosses a launch as plain fp16."""
    written = {'x': ('f32', 9)}
    for tag, fn, _, reads, writes in xref.exact_flow(H, B):
        for name, form, width in reads:
            assert name in written, f'{tag}: reads {name} before any launch writes it'
            assert written[name] == (form, width), (tag, name, written[name], (form, width))
        for name, form, width in writes:
            assert form in ('f32', 'split'), (tag, name, form)
            written[name] = (form, width)
    assert written['planes'] == ('f32', 96)


def test_every_split_entry_point_is_declared_and_planned():
    header = open(capi.HEADER).read()
    planned = {f for H, B in SIZES for _, f, _ in xref.launch_plan_exact(H, B)}
    for fn in xref.SPLIT_ENTRY_POINTS:
        assert fn in capi._SIGNATURES and f'int {fn}(' in header, fn
        assert fn in planned, fn


def test_precision_argument():
    assert SegFormerSECC2PlaneBackbone().precision == 'tc'
    assert SegFormerSECC2PlaneBackbone(precision='tc_exact').precision == 'tc_exact'
    for bad in ('fp32', 'TC', 'exact', None, ''):
        with pytest.raises(ValueError):
            SegFormerSECC2PlaneBackbone(precision=bad)
    with pytest.raises(TypeError):
        SegFormerSECC2PlaneBackbone('b0', 96, 'cano_src_tgt', 'tc_exact')                           # keyword-only
    for kw in ({'mode': 'b1'}, {'out_channels': 288}):                                               # unbuilt configurations still raise
        with pytest.raises(NotImplementedError):
            SegFormerSECC2PlaneBackbone(precision='tc_exact', **kw)
    m = SegFormerSECC2PlaneBackbone(pncc_cond_mode='cano_tgt', precision='tc_exact')
    assert m.prenet.weight.shape[1] == 6
    with pytest.raises(RuntimeError, match='CUDA'):
        m(torch.zeros(1, 6, 64, 64))


@pytest.mark.parametrize('mode', ['cano_src_tgt', 'cano_tgt'])
def test_state_dict_is_the_same_in_both_precisions(mode):
    a, b = _module(pncc_cond_mode=mode), _module(pncc_cond_mode=mode, precision='tc_exact')
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb)
    for k in sa:
        assert sa[k].shape == sb[k].shape and sa[k].dtype == sb[k].dtype and torch.equal(sa[k], sb[k]), k
    b.load_state_dict(sa, strict=True)                                                               # and one loads the other's
    a.load_state_dict(b.state_dict(), strict=True)


def test_split_packing_equals_float64_fold_bit_for_bit():
    m = _module(seed=5, precision='tc_exact')
    want = xref.exact_packs(ref.to64(m.state_dict()))
    P = sp.fold_and_pack(m, 'cpu', True)
    got = {}
    for s, st in enumerate(P['stages']):
        if s > 0:
            got[f's{s + 1}.pe'] = st['pe']
        for bi, b in enumerate(st['blocks']):
            for n, key in (('attn.q', 'q'), ('attn.kv', 'kv'), ('attn.proj', 'proj'), ('mlp.fc1', 'fc1'), ('mlp.fc2', 'fc2'), ('attn.sr', 'sr')):
                if key in b:
                    got[f's{s + 1}.{bi}.{n}'] = b[key]
    for i, g in enumerate(P['G']):
        got[f'G{i + 1}'] = g
    for i, cv in zip((0, 2, 4), P['convs']):
        got[f'to_plane_cnn.{i}'] = cv['mf']
    got['last_r'], got['last_rc'] = P['last_r'], P['last_rc']
    assert set(got) == set(want)
    for k, pk in got.items():
        assert pk.w.dtype == torch.float16 and pk.w.shape == want[k].shape, (k, tuple(pk.w.shape), tuple(want[k].shape))
        assert torch.equal(pk.w.view(torch.int16), want[k].view(torch.int16)), k
        assert pk.w.shape[-2 if pk.w.ndim == 3 else 0] == pk.cop and pk.bias.dtype == torch.float32
    # the biases and the fp32 tensors do not depend on the precision
    Pt = sp.fold_and_pack(m, 'cpu', False)
    assert torch.equal(P['stages'][2]['blocks'][1]['fc1'].bias, Pt['stages'][2]['blocks'][1]['fc1'].bias)
    assert torch.equal(P['head_bias'], Pt['head_bias']) and torch.equal(P['wpre'], Pt['wpre'])
    # tc packs are the plain fp16 of the same fold: the hi half of the split pack is fp16(w * 2^10)
    q_tc, q_ex = Pt['stages'][0]['blocks'][0]['q'].w, P['stages'][0]['blocks'][0]['q'].w
    assert q_ex.shape[1] == 2 * q_tc.shape[1]
    assert torch.equal(q_tc, m.mix_vit.block1[0].attn.q.weight.detach().double().half())
