"""Every r3dp_mf_conv3d launch of SegFormerSECC2PlaneBackbone('b0') at its exact arguments against float64, and a recorded-launch check that
keeps the per-launch tables of the backbone equal to what the module launches.

* CONV3D holds one row per distinct r3dp_mf_conv3d launch of `forward` at 512^2 (B = 4 and 1), 480^2 (B = 3), 96^2 and 32^2 (B = 3): the
  token GEMMs (q, kv, proj, fc1, fc2, sr, the patch embeds of stages 2-4, the head maps G_i) on 1x1x1 taps with xs = K and ys = O, the
  to_plane_cnn convs below 512^2 (1x3x3, 256 -> 256 fp16) and the last conv (1x3x3, fp32 into a 96-wide slice).  The rows come from
  secc2plane_reference.launch_plan; the weights from the module's own packers, so the padded couts (cop > cout) carry its zero rows.
  The bound is sr_conv_reference's |got - ref| <= alpha |ref| + extra + beta S, S the same GEMM / conv on |x|, |w| and |b|, with BETA
  per tap count below (measured on the card).  Every output sits between sentinel guards of at least (cop - cout) ys
  elements: every element of the slice is written and nothing else is.  Bit-exact: the last rows of a GEMM equal a launch on those rows
  alone, the last image of a conv its N = 1 launch.
* test_backbone_launches_have_rows records every r3dp_mf_conv3d, r3dp_sr_tc_conv and r3dp_sp_* call of `forward` at 512^2 (B = 4, 1)
  and 480^2 (B = 3), requires the recorded sequence to equal launch_plan's, and each launch to have a row: CONV3D here, CASES of
  test_gpu_sr_conv_conformance.py for r3dp_sr_tc_conv (SECC_PRODUCTION there), the r3dp_sp_* tables of test_gpu_secc2plane_kernels.py.
  Every 512^2 row must still be launched."""
import pytest
import torch

import real3dportrait_b200 as r3
from real3dportrait_b200 import _capi as capi, secc2plane as sp
import secc2plane_reference as ref
import sr_conv_reference as scr
import test_gpu_secc2plane_kernels as kern
import test_gpu_sr_conv_conformance as srcc
from launch_harness import GUARD, Recorder, assert_plan, assert_rows, assert_written, call_signature, conv3d, guarded, inside
from torso_motion_reference import ref_conv

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
F16, F32 = torch.float16, torch.float32
#: (H, B) of the forward calls the table covers; the first three are the ones the recorded-launch test runs
PLAN_SIZES = [(512, 4), (512, 1), (480, 3), (96, 3), (32, 3)]
RECORDED = PLAN_SIZES[:3]
#: beta per taps (1: the token GEMMs, 9: the 1x3x3 convs).  Worst ratio over the rows on an H100 80GB HBM3 (700 W power limit): GEMMs
#: 4.4e-7 (s4.pe, K = 1440, fp32 out), convs 6.7e-7 (the 480^2 last conv, K = 2304, fp32 out); the fp16-output rows measure lower (GEMMs
#: 4.8e-8, convs 1.7e-7) because the store's 2^-11 rounding absorbs most of the accumulation error.  A skipped K chunk or cout tile costs
#: O(S), far outside either bar.  The estimator's table (BETA3, 2^-18) measures 343-tap sums; these are shorter.
BETA = {1: 1e-6, 9: 1.5e-6}


def _rows(fn):
    """{signature: tag} of one entry point over PLAN_SIZES, the first tag of each distinct launch."""
    out = {}
    for H, B in PLAN_SIZES:
        for tag, f, a in ref.launch_plan(H, B):
            if f == fn:
                out.setdefault(ref.launch_signature(f, a), f'{H}^2 B{B} {tag}')
    return out


CONV3D = _rows('r3dp_mf_conv3d')
CONV3D_KEYS = list(CONV3D)


def _id(key):
    a = key[1]
    kind = 'gemm' if a[8] == 1 else 'conv'
    return f'{CONV3D[key].replace(" ", "-")}-{kind}-K{a[2]}-N{a[3]}x{a[5]}x{a[6]}-O{a[11]}cop{a[12]}-ys{a[14]}c{a[15]}-{"f32" if a[17] else "f16"}'


# ---- operands and one launch ---------------------------------------------------------------------------------------------------------------
def _weights(tag, cin, O, taps, g):
    """The module's packing of seeded float64 weights: _pack_gemm of a Linear / _conv_rows of a patch-embed or sr conv / G_i (no bias), or
    _pack_taps of a 3x3 conv.  -> (packed fp16, fp32 bias, cop)."""
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV, dtype=torch.float64)      # noqa: E731
    if taps == 9:
        wp, b, _, cop = sp._pack_taps(rn(O, cin, 3, 3) / (9 * cin) ** 0.5, 0.1 * rn(O), DEV)
        return wp, b, cop
    st = tag.rsplit(' ', 1)[-1]
    if st.endswith('.pe') or st.endswith('.sr'):
        k = 3 if st.endswith('.pe') else ref.SR[int(st[1]) - 1]
        w = sp._conv_rows(rn(O, cin // (k * k), k, k) / cin ** 0.5)
    else:
        w = rn(O, cin) / cin ** 0.5
    wp, b, _, cop = sp._pack_gemm(w, None if st.startswith('G') else 0.1 * rn(O), DEV)
    return wp, b, cop


@torch.no_grad()
@pytest.mark.parametrize('key', CONV3D_KEYS, ids=[_id(k) for k in CONV3D_KEYS])
def test_conv3d_launch_vs_float64(key):
    a = key[1]
    xs, _, cin, N, D, H, W, kd, kh, kw, _, O, cop, _, ys, yc0, _, out_f32, _ = a
    taps = kd * kh * kw
    tag = CONV3D[key]
    g = torch.Generator(device=DEV).manual_seed(CONV3D_KEYS.index(key) + 500)
    wp, b, cop_mod = _weights(tag, cin, O, taps, g)
    assert cop_mod == cop, (tag, cop_mod, cop)                                  # the module's packing pads to the launch's cop
    M = N * D * H * W
    x = torch.randn(N, D, H, W, xs, generator=g, device=DEV).half()
    dt = F32 if out_f32 else F16
    buf, y = guarded(M * ys, dt, tail=max(GUARD, (cop - O) * ys), device=DEV)
    conv3d(a, x, wp, b, None, y)
    mask = inside(ys, yc0, O, device=DEV)
    assert_written(buf, y, ys, mask, tag)
    yv = y.view(M, ys)
    got = yv[:, yc0:yc0 + O].view(N, D, H, W, O)
    # a 256^2 last conv is checked on its last image: the float64 reference of all four would take several GB
    k0 = N - 1 if taps == 9 and H >= 256 else 0
    xd = x[k0:].double().permute(0, 4, 1, 2, 3)[:, :cin]
    wd = (wp.double().view(taps, cop, cin) if taps == 9 else wp.double().view(1, cop, cin))[None, :, :O]
    tp = (kd, kh, kw)
    want = ref_conv(xd, wd, tp, False, b[:O])
    S = ref_conv(xd.abs(), wd.abs(), tp, False, b[:O].abs())
    alpha = scr.ALPHA_F32 if out_f32 else scr.ALPHA_F16
    extra = 0.0 if out_f32 else 2 * scr.FLOOR_F16                              # fp16 subnormal floor of the store
    scr.check_bound(got[k0:].permute(0, 4, 1, 2, 3), want, S, alpha, BETA[taps], extra, tag=_id(key))
    # bit-exact: the last image of a conv equals its N = 1 launch; the last rows of a GEMM equal a launch on those rows alone
    if taps == 9:
        if N > 1:
            _, one = guarded(D * H * W * ys, dt, device=DEV)
            conv3d(a, x[N - 1:].contiguous(), wp, b, None, one, N=1)
            assert torch.equal(one.view(H * W, ys)[:, mask], yv[-H * W:, mask]), f'{tag}: last image vs its N=1 launch'
    else:
        r = min(W, 300)
        tail = torch.empty(r * ys, device=DEV, dtype=dt)
        conv3d(a, x[:, :, :, W - r:].contiguous(), wp, b, None, tail, N=1, H=1, W=r)
        assert torch.equal(tail.view(r, ys), yv[-r:]), f'{tag}: last {r} rows vs a launch on them alone'


# ---- the recorded launches -----------------------------------------------------------------------------------------------------------------
@torch.no_grad()
def test_backbone_launches_have_rows():
    m = r3.SegFormerSECC2PlaneBackbone()
    m.load_state_dict(ref.make_params({k: v.shape for k, v in m.state_dict().items()}, 3), strict=True)
    m = m.to(DEV).eval()
    m._prepared()                                                # the weight packing launches r3dp_sr_tc_pack_weights, not recorded
    launched = {}
    with Recorder(capi.lib(), lambda n: n.startswith('r3dp_sp_') or n in ('r3dp_mf_conv3d', 'r3dp_sr_tc_conv')) as rec:
        for H, B in RECORDED:
            cano, src, tgt = ref.make_inputs(B, H, 11)
            rec.calls.clear()
            m(torch.cat([cano.expand(B, -1, -1, -1), src.expand(B, -1, -1, -1), tgt], 1).to(DEV))
            got = [call_signature(n, a) for n, a in rec.calls]
            assert_plan(got, [ref.launch_signature(f, a) for _, f, a in ref.launch_plan(H, B)], f'{H}^2 B={B}')
            for s in got:
                launched.setdefault(s, (H, B))
        torch.cuda.synchronize()
    sr_rows = {srcc.row_signature(row) for row in srcc.CASES}
    sp_rows = kern.sp_signatures()
    missing = []
    for (fn, a), (H, B) in launched.items():
        if fn == 'r3dp_mf_conv3d':
            ok = (fn, a) in CONV3D
        elif fn == 'r3dp_sr_tc_conv':
            N, Nw, I, O, h, w, ksize, act = a
            ok = srcc.row_signature(('conv_res', N, Nw, I, O, h, w, {'ksize': ksize, 'act': act})) in sr_rows
        else:
            ok = (fn, a) in sp_rows
        if not ok:
            missing.append(f'{H}^2 B={B}: {fn}{a}')
    stale = [f'{CONV3D[k]}: {k}' for k in CONV3D if CONV3D[k].startswith('512^2') and k not in launched]
    stale += [f'{fn}{a} ({H}^2 B={B})' for fn, a, (H, B) in kern.sp_rows_at(512) if (fn, a) not in launched]
    stale += [f'SECC_PRODUCTION {row}' for row in srcc.SECC_PRODUCTION
              if ('r3dp_sr_tc_conv', (*row[1:7], row[7].get('ksize', 3), row[7]['act'])) not in launched]
    assert_rows(missing, stale, 'the 512^2 backbone')
