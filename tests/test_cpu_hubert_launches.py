"""HuBERT's launch plan and the end-to-end bar, on the host.

* launch_plan's invariants for hubert-large and the small fixture config at T = 1 ... 30 000: the stats launch once and 186 launches per
  group for hubert-large (32 for the small config); the segment lengths of the groups sum to T; every split row keeps its lo half past the
  channels a launch reads or writes, so the columns between the halves are never written; Cp is a multiple of 64 and >= C; the conv GEMMs
  read windows of k frames at a stride of s frames of their input rows, which the previous launch wrote; HubertModel.forward on B items is
  B groups of one segment without stats.
* The plan's GEMM, attention and positional-conv tags are exactly forward_folded's sites.
* The discrimination check (hubert-large at T = 49, the small config at T = 1031): forward_folded with every operand rounded as the kernels
  read it (split fp16) sits at least 10x below E2E_BAR and with every launch reading fp16 hi halves alone at least 3x above it.  A single
  launch that loses its lo halves moves hubert-large's output by about 1e-6 ... 3e-5 of its range, the size of the library's own fp32
  accumulation error, so the end-to-end bar cannot promise to see one launch: each site's margin is printed, not asserted, and the
  per-launch rows of tests/test_gpu_hubert_launches.py each assert that hi-only operands break their own bar."""
import pytest
import torch

import hubert_reference as hr
from real3dportrait_b200 import hubert as hb

CONFIGS = {'large': hr.LARGE, 'small': hr.small_config()}
PER_GROUP = {'large': 186, 'small': 32}
TS = [1, 999, 1000, 4000, 4001, 30000]


def _clip(T):
    return 320 * T + 80 + (T % 7) * 37


def _groups(plan):
    """{group prefix: [(tag, fn, args)]} in launch order."""
    out = {}
    for tag, fn, a in plan:
        if '.' in tag:
            out.setdefault(tag.split('.', 1)[0], []).append((tag, fn, a))
    return out


def _check_group(cfg, launches, segs):
    C, H, I = cfg['conv_dim'][0], cfg['hidden_size'], cfg['intermediate_size']
    Cp = (C + 63) // 64 * 64
    assert Cp % 64 == 0 and Cp >= C
    Fg = sum(segs)
    F, width = None, None                                      # rows and row width of the split rows the next launch reads
    for tag, fn, a in launches:
        site = tag.split('.', 1)[1]
        if fn == 'r3dp_hb_conv0':
            F, c, _, ys, ylo = a
            assert c == C and ylo >= C and ys >= ylo + C and ylo == Cp, tag
            assert 5 * (F - 1) + 10 <= 320 * (Fg - 1) + 400, tag            # conv0 reads only the group's samples
            width = ys
        elif fn == 'r3dp_hb_gemm':
            M, w, s, seg, N, Kp, epi, ldy, ylo = a
            assert seg % 64 == 0 and Kp % seg == 0 and w == Kp // seg * 2 * seg, tag    # each tap reads hi [0, seg) and lo [seg, 2 seg)
            if site.startswith('conv'):
                i = int(site[4])
                k, st = hr.KERNELS[i], hr.STRIDES[i]
                assert (seg, Kp, w, s) == (Cp, k * Cp, k * 2 * Cp, st * 2 * Cp), tag
                assert M == (F - k) // st + 1 and (M - 1) * st + k <= F and width == 2 * Cp, tag
                assert (N, epi, ldy, ylo) == (C, 3, C, 0), tag
                F = M
            else:
                assert M == Fg and w == s == width, tag                     # dense rows: the launch reads the whole split row
                K = {'proj': C, 'qkv': H, 'out': H, 'ffn1': H, 'ffn2': I}[site.split('.')[-1]]
                assert seg >= K and Kp == seg, tag
                if epi in (0, 1):
                    assert ylo >= N and ldy >= ylo + N, tag                 # lo past the hi half: no column between them is written
                    width = ldy
                else:
                    assert ldy >= N and ylo == 0, tag
        elif fn == 'r3dp_hb_layernorm':
            R, c, _, gelu, yfs, yhs, yhlo = a
            assert R == F if site.startswith('conv') else R == Fg, tag
            assert (yfs == 0) != (yhs == 0), tag                            # one output form per launch
            if yhs:
                assert yhlo >= c and yhs >= yhlo + c, tag
                width = yhs
            assert gelu == int(site.startswith('conv')), tag
        elif fn == 'r3dp_a2m_split':
            assert a == (Fg, H), tag
        elif fn == 'r3dp_hb_pos_conv':
            nseg, Ls, M, h = a
            assert (nseg, Ls, M, h) == (len(segs), max(segs), Fg, H) and (nseg - 1) * Ls < M <= nseg * Ls, tag
        elif fn == 'r3dp_hb_attention':
            rows, ld, lo, heads, lens, nseg, os_, olo = a
            assert lens == tuple(segs) and nseg == len(segs) and sum(lens) == rows == Fg, tag
            assert heads * 64 == H and lo == 3 * H and ld == 6 * H and width == ld and olo >= H and os_ >= olo + H, tag
            width = os_
        else:
            raise AssertionError(f'{tag}: unexpected entry point {fn}')


@pytest.mark.parametrize('name', CONFIGS)
@pytest.mark.parametrize('T', TS)
def test_plan_invariants(name, T):
    cfg = CONFIGS[name]
    L = _clip(T)
    assert hr.frames(L) == hb.hubert_frames(L) == T
    plan = hr.launch_plan(cfg, L)
    assert plan[0] == ('stats', 'r3dp_hb_stats', (L,))
    assert len({tag for tag, _, _ in plan}) == len(plan)
    grp = hr.groups(T)
    assert sum(sum(s) for _, s in grp) == T and all(len(s) <= hr.GROUP and max(s) <= hr.SEG for _, s in grp)
    assert [f0 for f0, _ in grp] == [sum(sum(s) for _, s in grp[:g]) for g in range(len(grp))]
    assert all(f0 % (hr.SEG * hr.GROUP) == 0 for f0, _ in grp)
    launches = _groups(plan)
    assert len(plan) == 1 + PER_GROUP[name] * len(grp) and len(launches) == len(grp)
    for (_, segs), (_, ls) in zip(grp, launches.items()):
        assert len(ls) == PER_GROUP[name]
        _check_group(cfg, ls, segs)
    assert plan[-1][2][4] == cfg['hidden_size']                              # ln_f into contiguous [T, H] rows
    assert hr.launch_plan(cfg, L, ldo=1032)[-1][2][4] == 1032


@pytest.mark.parametrize('name', CONFIGS)
def test_plan_forward_items(name):
    cfg = CONFIGS[name]
    Lx = 320 * 48 + 400 + 11
    plan = hr.launch_plan(cfg, Lx, B=2)
    launches = _groups(plan)
    assert list(launches) == ['b0', 'b1'] and len(plan) == 2 * PER_GROUP[name]
    for ls in launches.values():
        _check_group(cfg, ls, [49])
    assert [a for _, _, a in launches['b0']] == [a for _, _, a in launches['b1']]


@pytest.mark.parametrize('name', CONFIGS)
def test_plan_tags_cover_folded_sites(name):
    cfg = CONFIGS[name]
    for T in (1, 4001):
        plan = hr.launch_plan(cfg, _clip(T))
        for g in _groups(plan):
            sites = [hr.site_of(tag, fn) for tag, fn, _ in plan if tag.startswith(g + '.') and hr.site_of(tag, fn)]
            assert sites == hr.folded_sites(cfg)
    if name == 'small':
        m, _ = hr.formula_model(cfg)
        P = hb.fold_weights(m)
        x = hr.normalise(hr.wave(_clip(3)))
        for site in hr.folded_sites(cfg):
            assert torch.isfinite(hr.forward_folded(P, cfg, x, operands='hi', site=site)).all()
        for bad in ('split', 'l0.ln1', 'conv0', 'l9.qkv'):
            with pytest.raises(ValueError, match='no launch'):
                hr.forward_folded(P, cfg, x, operands='hi', site=bad)


@pytest.fixture(scope='module')
def folded():
    out = {}
    for name, cfg in CONFIGS.items():
        m, _ = hr.formula_model(cfg)
        out[name] = hb.fold_weights(m)
        del m
    return out


@pytest.mark.parametrize('name,T', [('large', 49), ('small', 1031)])
@torch.no_grad()
def test_end_to_end_bar_discriminates(folded, name, T):
    """The formula weights and waveform of tests/test_gpu_hubert.py; one segment (T <= 1031 frames, two for the small config)."""
    cfg, P = CONFIGS[name], folded[name]
    L = _clip(T)
    x = hr.normalise(hr.wave(L))[:320 * (T - 1) + 400]
    segs = hr.segments(T)
    exact = hr.forward_folded(P, cfg, x, segs)
    scale = float(exact.abs().max())

    def ratio(**k):
        return float((hr.forward_folded(P, cfg, x, segs, **k) - exact).abs().max()) / scale

    split = ratio(operands='split')
    print(f'{name} T={T}: all split {split:.2e} = bar / {hr.E2E_BAR / split:.0f}')
    assert split * 10 <= hr.E2E_BAR
    every = ratio(operands='hi')
    print(f'{name} T={T}: all hi-only {every:.2e} = bar x {every / hr.E2E_BAR:.1f}')
    assert every >= 3 * hr.E2E_BAR
    for site in hr.folded_sites(cfg):
        r = ratio(operands='hi', site=site)
        print(f'{name} T={T}: {site} hi-only {r:.2e} = bar x {r / hr.E2E_BAR:.2f}')
