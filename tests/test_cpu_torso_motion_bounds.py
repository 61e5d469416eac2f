"""The bars of tests/torso_motion_reference.py have teeth (no GPU needed): a float32 restatement of each kernel around the motion-field
estimator's convolutions (csrc/conv3d_tc.cu) and of r3dp_tw_affine_relu passes its bar at a toy size, and the same restatement with one
plausible defect fails it."""
import pytest
import torch

import sr_conv_reference as scr
import torso_motion_reference as tmr
import torso_warper_ref as twr


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _split(v):
    """fp32 -> (hi, lo) fp16, the kernels' put()."""
    hi = v.half()
    return hi, (v - hi.float()).half()


def _join(hl):
    return hl[0].double() + hl[1].double()


def _get(hl, split=True):
    """The kernels' get(): hi + lo summed in fp32."""
    return hl[0].float() + hl[1].float() if split else hl[0].float()


def _fma(a, b, c):
    """fp32 fmaf through float64: the product of two fp32 values is exact in float64, one rounding to fp32 remains."""
    return (a.double() * b.double() + c.double()).float()


def _fails(fn):
    with pytest.raises(AssertionError):
        fn()


# ---- pool / head_bcast / head_input ---------------------------------------------------------------------------------------------------------
def _mean2x2_f32(a, rows=(0, 1), cols=(0, 1)):
    """((a + b) + (c + d)) * 0.25 on [.., 2H, 2W, C] fp32; rows / cols: the offsets of the pair inside each block."""
    r0, r1 = rows
    c0, c1 = cols
    return ((a[..., r0::2, c0::2, :] + a[..., r0::2, c1::2, :]) + (a[..., r1::2, c0::2, :] + a[..., r1::2, c1::2, :])) * 0.25


def test_pool_bar_and_wrong_pair():
    x = _split(3 * torch.randn(2, 3, 8, 10, 16, generator=_g(1)))
    ref, S = tmr.pool(_join(x))
    ok = _join(_split(_mean2x2_f32(_get(x))))
    scr.check_bound(ok, ref, S, scr.ALPHA_SPLIT, tmr.BETA_POOL, scr.FLOOR_F16, 'pool sim')
    bad = _join(_split(_mean2x2_f32(_get(x), rows=(0, 0))))                     # rows (2y, 2y) instead of (2y, 2y + 1)
    _fails(lambda: scr.check_bound(bad, ref, S, scr.ALPHA_SPLIT, tmr.BETA_POOL, scr.FLOOR_F16))


def test_head_bcast_bar_and_lo_half_ignored():
    x = _split(torch.randn(2, 8, 8, 32, generator=_g(2)))
    ref, S = tmr.pool(_join(x))
    ok = _join(_split(_mean2x2_f32(_get(x))))
    scr.check_bound(ok, ref, S, scr.ALPHA_SPLIT, tmr.BETA_POOL, scr.FLOOR_F16, 'head_bcast sim')
    bad = _join(_split(_mean2x2_f32(_get(x, split=False))))                    # the lo half of the input ignored
    _fails(lambda: scr.check_bound(bad, ref, S, scr.ALPHA_SPLIT, tmr.BETA_POOL, scr.FLOOR_F16))


def test_head_input_bar_and_wrong_pair():
    g = _g(3)
    rgb, wt = 2 * torch.rand(2, 3, 8, 12, generator=g) - 1, torch.rand(2, 1, 8, 12, generator=g)
    ref, S = tmr.head_input(rgb.double(), wt.double())
    x = torch.cat([rgb, wt], 1).permute(0, 2, 3, 1)
    for split in (False, True):
        st = (lambda v: _join(_split(v))) if split else (lambda v: v.half().double())      # noqa: E731
        alpha = scr.alpha_store(split)
        scr.check_bound(st(_mean2x2_f32(x)), ref, S, alpha, tmr.BETA_HEAD_INPUT, scr.FLOOR_F16, f'head_input sim split={split}')
        _fails(lambda: scr.check_bound(st(_mean2x2_f32(x, cols=(1, 1))), ref, S, alpha, tmr.BETA_HEAD_INPUT, scr.FLOOR_F16))


# ---- affine_relu ------------------------------------------------------------------------------------------------------------------------------
def test_affine_relu_bar_and_scale_index():
    g = _g(4)
    C = 32
    x = _split(3 * torch.randn(2, 5, 6, C, generator=g))
    s, t = 0.5 + torch.rand(C, generator=g), 0.3 * torch.randn(C, generator=g)
    ref, S = tmr.affine_relu(_join(x), s, t)

    def sim(idx):
        return _join(_split(torch.relu(_fma(_get(x), s[idx], t[idx]))))
    c = torch.arange(C)
    scr.check_bound(sim(c), ref, S, scr.ALPHA_SPLIT, tmr.BETA_AFFINE, scr.FLOOR_F16, 'affine_relu sim')
    _fails(lambda: scr.check_bound(sim(c & ~7), ref, S, scr.ALPHA_SPLIT, tmr.BETA_AFFINE, scr.FLOOR_F16))     # scale / shift at c & ~7


# ---- mf_input -------------------------------------------------------------------------------------------------------------------------------
def _grid_f32(n):
    i = torch.arange(n, dtype=torch.float32)
    return 2.0 * (i / float(n - 1)) - 1.0


def _mf_input_f32(fc, kp_s, kp_d):
    """r3dp_mf_input for one frame in fp32: fc [D,H,W,4] fp32, kp [K,3] -> [D,H,W,(K+1)*5] fp32 (before the store)."""
    D, H, W, _ = fc.shape
    K = kp_s.shape[0]
    gz, gy, gx = torch.meshgrid(_grid_f32(D), _grid_f32(H), _grid_f32(W), indexing='ij')
    out = []
    for k in range(K + 1):
        sx, sy, sz, hm = gx, gy, gz, torch.zeros_like(gx)
        if k > 0:
            ps, pd = kp_s[k - 1], kp_d[k - 1]
            ddx, ddy, ddz = gx - pd[0], gy - pd[1], gz - pd[2]
            dsx, dsy, dsz = gx - ps[0], gy - ps[1], gz - ps[2]
            c = torch.tensor(0.01, dtype=torch.float32)
            hm = torch.exp(-0.5 * (ddx * ddx + ddy * ddy + ddz * ddz) / c) - torch.exp(-0.5 * (dsx * dsx + dsy * dsy + dsz * dsz) / c)
            sx, sy, sz = ddx + ps[0], ddy + ps[1], ddz + ps[2]
        out.append(hm[..., None])
        ix, iy, iz = (sx + 1.0) / 2.0 * float(W - 1), (sy + 1.0) / 2.0 * float(H - 1), (sz + 1.0) / 2.0 * float(D - 1)
        fx, fy, fz = torch.floor(ix), torch.floor(iy), torch.floor(iz)
        acc = torch.zeros(D, H, W, 4)
        for cnr in range(8):
            dz, dy, dx = cnr >> 2, (cnr >> 1) & 1, cnr & 1
            xx, yy, zz = fx.long() + dx, fy.long() + dy, fz.long() + dz
            ok = (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H) & (zz >= 0) & (zz < D)
            wt = (ix - fx if dx else fx + 1.0 - ix) * (iy - fy if dy else fy + 1.0 - iy) * (iz - fz if dz else fz + 1.0 - iz)
            v = fc[zz.clamp(0, D - 1), yy.clamp(0, H - 1), xx.clamp(0, W - 1)]
            acc = torch.where(ok[..., None], _fma(v, wt[..., None], acc), acc)
        out.append(acc)
    return torch.cat(out, -1)


def test_mf_input_bar_and_shared_volume_misread():
    g = _g(5)
    N, K, D, H, W = 2, 3, 5, 9, 11
    fc = torch.randn(N, D, H, W, 4, generator=g)
    kp_s, kp_d = [0.9 * (2 * torch.rand(N, K, 3, generator=g) - 1) for _ in range(2)]
    for n in range(N):
        ref, S, extra = tmr.mf_input(fc[n].double(), kp_s[n].double(), kp_d[n].double())
        ex = extra * (1 + 2.0 ** -10) + scr.FLOOR_F16
        got = _join(_split(_mf_input_f32(fc[n], kp_s[n], kp_d[n])))
        r = scr.check_bound(got, ref, S, scr.ALPHA_SPLIT, tmr.BETA_SAMPLE, ex, f'mf_input sim frame {n}')
        assert r <= tmr.BETA_SAMPLE
    bad = _join(_split(_mf_input_f32(fc[0], kp_s[1], kp_d[1])))                 # frame 1 reading frame 0's volume, as if fc_shared were set
    ref, S, extra = tmr.mf_input(fc[1].double(), kp_s[1].double(), kp_d[1].double())
    _fails(lambda: scr.check_bound(bad, ref, S, scr.ALPHA_SPLIT, tmr.BETA_SAMPLE, extra * (1 + 2.0 ** -10) + scr.FLOOR_F16))


def test_mf_input_coordinate_term_is_needed():
    """Without the coordinate term the fp32 restatement fails on the Gaussians' flanks: the term is what lets the bar stay tight."""
    g = _g(6)
    D, H, W, K = 5, 33, 33, 4
    fc = torch.randn(D, H, W, 4, generator=g)
    kp_s, kp_d = [0.9 * (2 * torch.rand(K, 3, generator=g) - 1) for _ in range(2)]
    ref, S, extra = tmr.mf_input(fc.double(), kp_s.double(), kp_d.double())
    got = _join(_split(_mf_input_f32(fc, kp_s, kp_d)))
    scr.check_bound(got, ref, S, scr.ALPHA_SPLIT, tmr.BETA_SAMPLE, extra * (1 + 2.0 ** -10) + scr.FLOOR_F16, 'mf_input sim 33^2')
    _fails(lambda: scr.check_bound(got, ref, S, scr.ALPHA_SPLIT, tmr.BETA_SAMPLE, scr.FLOOR_F16))


# ---- mf_deform --------------------------------------------------------------------------------------------------------------------------------
def _deform_f32(logits, kp_s, kp_d):
    D, H, W, K1 = logits.shape
    gz, gy, gx = torch.meshgrid(_grid_f32(D), _grid_f32(H), _grid_f32(W), indexing='ij')
    g = [gx, gy, gz]
    mx = logits.amax(-1)
    den = torch.zeros(D, H, W)
    for k in range(K1):
        den = den + torch.exp(logits[..., k] - mx)
    o = [torch.zeros(D, H, W) for _ in range(3)]
    for k in range(K1):
        m = torch.exp(logits[..., k] - mx) / den
        for c in range(3):
            s = g[c] if k == 0 else (g[c] - kp_d[k - 1, c]) + kp_s[k - 1, c]
            o[c] = _fma(s, m, o[c])
    return torch.stack(o, -1)


def test_mf_deform_bar_and_swapped_keypoints():
    g = _g(7)
    D, H, W, K = 4, 6, 7, 4
    logits = 3 * torch.randn(D, H, W, K + 1, generator=g)
    kp_s, kp_d = [0.9 * (2 * torch.rand(K, 3, generator=g) - 1) for _ in range(2)]
    ref, S, extra = tmr.deform(logits.double(), kp_s.double(), kp_d.double())
    scr.check_bound(_deform_f32(logits, kp_s, kp_d).double(), ref, S, 0.0, scr.gamma(K + 2), extra, 'deform sim')
    _fails(lambda: scr.check_bound(_deform_f32(logits, kp_d, kp_s).double(), ref, S, 0.0, scr.gamma(K + 2), extra))   # kp_s / kp_d swapped


# ---- mf_occlusion -----------------------------------------------------------------------------------------------------------------------------
def _occlusion_f32(x, wk, bk, order='cD+d'):
    """The kernel's fma chain per output pixel over (d, ky, kx, c); x fp32 [D,H,W,C] (hi + lo summed), wk [D,49,C,2].  order 'dC+c':
    the weights of input channel d*C + c read for channel c*D + d (the other view of the fuser output)."""
    D, H, W, C = x.shape
    if order == 'dC+c':
        full = wk.permute(2, 0, 1, 3).reshape(C * D, 49, 2)                  # [c*D + d] as the kernel's layout holds it
        wk = full.reshape(D, C, 49, 2).permute(0, 2, 1, 3)                    # read back as if the channel were d*C + c
    xp = torch.nn.functional.pad(x, (0, 0, 3, 3, 3, 3))
    out = []
    for o in range(2):
        acc = torch.zeros(H, W)
        for d in range(D):
            for ky in range(7):
                for kx in range(7):
                    for c in range(C):
                        v = xp[d, ky:ky + H, kx:kx + W, c]
                        nz = torch.zeros(H + 6, W + 6, dtype=torch.bool)
                        nz[3:3 + H, 3:3 + W] = True
                        ok = nz[ky:ky + H, kx:kx + W]
                        acc = torch.where(ok, _fma(v, wk[d, ky * 7 + kx, c, o], acc), acc)
        out.append(1.0 / (1.0 + torch.exp(-(acc + bk[o]))))
    return out


def test_mf_occlusion_bar_and_channel_order():
    g = _g(8)
    D, H, W, C = 3, 5, 6, 8
    x = _split(torch.randn(D, H, W, C, generator=g))
    wk = 3 * torch.randn(D, 49, C, 2, generator=g) / (D * 49 * C) ** 0.5
    bk = 0.1 * torch.randn(2, generator=g)
    bounds = tmr.occlusion(_join(x), wk, bk, True)
    for got, (ref, S, extra) in zip(_occlusion_f32(_get(x), wk, bk), bounds):
        scr.check_bound(got.double(), ref, S, 0.0, tmr.BETA_OCC, extra, 'occlusion sim')
    bad = _occlusion_f32(_get(x), wk, bk, order='dC+c')
    _fails(lambda: [scr.check_bound(b.double(), r, S, 0.0, tmr.BETA_OCC, e) for b, (r, S, e) in zip(bad, bounds)])


# ---- the launch plan -------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('K', [4, 9])
def test_launch_plan_layout(K):
    """launch_plan's fuser-input slices tile the voxel: input channels [0, P0), the last up block [P0, P0 + 32), the head features
    [P0 + 32, P0 + 64) = CF; the conv chain's channel counts follow one another; the per-clip volume is shared only when N > 1."""
    P0 = ((K + 1) * 5 + 31) // 32 * 32
    for split in (0, 1):
        wide = 2 if split else 1
        plan = {tag: a for tag, _, a in twr.launch_plan(K, 4, split)}
        assert plan['mf.input'][6:9] == (P0, (P0 + 64) * wide, P0 + 64)
        up4, bc = plan['mf.up.4'], plan['mf.head_bcast']
        assert (up4[11], up4[14], up4[15], up4[16]) == (32, (P0 + 64) * wide, P0, P0 + 64)
        assert bc[7:10] == ((P0 + 64) * wide, P0 + 32, P0 + 64)
        assert plan['mf.fuser'][:3] == ((P0 + 64) * wide, P0 + 64, P0 + 64) and plan['mf.down.0'][:3] == ((P0 + 64) * wide, P0 + 64, P0)
        assert plan['mf.mask'][11] == K + 1 and plan['mf.deform'][0] == plan['mf.mask'][14]
    assert twr.launch_plan(K, 4, 0)[0][2][0] == 1 and twr.launch_plan(K, 1, 0)[0][2][0] == 0 and twr.launch_plan(K, 4, 0, clip=False)[0][2][0] == 0
