"""Float64 references and element-wise error bounds for the kernels around the motion-field estimator's 3-D convolutions (csrc/conv3d_tc.cu
r3dp_mf_input, _pool, _head_input, _head_bcast, _deform, _occlusion) and for r3dp_tw_affine_relu (csrc/torso_warp.cu), for
tests/test_gpu_torso_warper_launches.py.  Test infrastructure: it does not import the library, so it also runs without a GPU
(tests/test_cpu_torso_motion.py shows there that each bar passes a float32 restatement of its kernel and fails a plausible defect).

Every reference is computed from the operands the kernel reads, converted exactly to float64 (hi + lo of split [hi | lo] tensors), and every
bound is sr_conv_reference.check_bound's  |got - ref| <= alpha |ref| + extra + beta S,  S the same operation on absolute values.  alpha is
the store's rounding (alpha_store and FLOOR_F16 for fp16 / split outputs, 0 for fp32 outputs).  Nothing here is measured: the kernels are
short chains of fp32 operations, so every term follows from the arithmetic.  u = 2^-24; the library is built without --use_fast_math
(divisions correctly rounded, expf within 2 ulp = 4u relative, subnormals kept), and first-order terms carry a factor 1.01 for the
second-order ones (every relative error below is under 1e-3).

  * pool / head_bcast:  ((a + b) + (c + d)) * 0.25 with a = fl(hi + lo) (split) or hi: every input passes through at most 3 roundings
    (its hi + lo and two adds), x 0.25 is exact: beta = gamma_3 on S = the 2x2 mean of |x|.
  * head_input:  the same mean of four fp32 inputs (the bilinear 256 -> 128 resize at exactly 1/2, align_corners=False): beta = gamma_2.
    The channels past the four real ones are written as exact zeros.
  * affine_relu:  fmaf(fl(hi + lo), s, t) then ReLU (1-Lipschitz): u |x| |s| from hi + lo, u |x s + t| from the fma: beta = gamma_2 on
    S = |x| |s| + |t|.
  * input (heatmaps):  the kernel's grid coordinate g' = fl(fl(2 fl(i / (n - 1))) - 1) is within 3u of the exact g.  The Gaussian argument
    a = -50 |g - kp|^2 is computed from d' = fl(g' - kp) with 3 squares, 2 adds, x -0.5 (exact) and / 0.01f (0.01f = 0.01 (1 - 2.2e-8),
    0.38u): a' = a(g') (1 + eta), |eta| <= 8u, and |a(g') - a(g)| <= 100 sum_i |d_i| 3u: the coordinate term, one grid-coordinate error
    times the local gradient |da/dd| of the steep (variance 0.01) flanks.  expf adds 4u, so |G' - G| <= G (1.01 |da| + 4u), and the
    difference of the two Gaussians rounds once more: extra = (E_d + E_s)(1 + u) + u |hm| + 2 x 2^-126 (expf results in the fp32 subnormal
    range), then the store.
  * input (deformed source):  s = g - kp_d + kp_s is computed as fl(fl(g' - kp_d) + kp_s): ds = 3u + u (|g - kp_d| + |s|) (k = 0: the
    identity grid, 3u).  ix = fl(fl(s + 1) / 2 * (n - 1)) adds u |s + 1| (n - 1) / 2 and u |ix|.  The trilinear interpolant of the zero-padded
    volume moves by at most sum_axis dix_axis L_axis, L_axis the largest |difference of two voxels neighbouring along that axis| over the
    cells within one voxel of the sample (the perturbed point may sit in a neighbouring cell): extra = 1.01 of that.  At the computed point
    each 1-D weight is within u (fx + 1 - ix is the one inexact subtraction), a corner weight within 5u, and the 8-term sum adds gamma_9:
    beta = gamma_15 on S = the same trilinear interpolation of |volume|.  Pad channels up to cpad are exact zeros.
  * deform:  m_k = softmax over the K + 1 fp32 logits.  fl(l_k - mx) and expf give e_k' = e_k (1 + r_k), r_k = 4u + 1.01 u |l_k - mx|;
    the K adds of the denominator gamma_K; the division u: m_k' = m_k (1 + q_k), q_k = r_k + max_j r_j + gamma_K + u.  The sparse motions
    s_k carry ds_k as above and the (K + 1)-term fma sum gamma_{K+1} (+ u of a product): extra = 1.01 sum_k m_k (|s_k| q_k + ds_k),
    beta = gamma_{K+2} on S = sum_k m_k |s_k|.  fp32 output, alpha = 0.
  * occlusion:  each output is sigmoid(v), v = b + sum over (d, ky, kx, c) of x[c, d] w, accumulated by one fma chain per output in that
    order (out-of-range taps skipped), x = fl(hi + lo).  An fma chain's error is at most u sum_i |P_i| over its exact partial sums P_i; the
    reference evaluates that sum in the kernel's order with the skipped taps as zero terms (a zero term repeats a partial sum and only
    loosens the bound), and the rounding of hi + lo adds u sum |x| |w|.  The bias add rounds once (u |v|).  Then, as for the torso head's
    gate (tests/torso_fusion_reference.py), s' = sigmoid(v') (1 + d) with |d| <= 6u: beta = 7u on S = sigmoid(v), and
    extra = 1.01 s (1 - s) |v' - v| + 2^-126."""
import torch
import torch.nn.functional as F

from sr_conv_reference import FLOOR_F16, U_F32, gamma  # noqa: F401  (re-exported)

U = U_F32
BETA_POOL = gamma(3)
BETA_HEAD_INPUT = gamma(2)
BETA_AFFINE = gamma(2)
BETA_SAMPLE = gamma(15)
BETA_OCC = 7 * U
FLOOR_EXP = 2.0 ** -126
SIGMA2 = 0.01                      # the heatmap Gaussians' variance (func_utils.py: kp_variance=0.01)
# Accumulation term of the 3-D conv (see sr_conv_reference.py for the bound): fp32 sums of up to 343 x 96 fp16 products per output (x3
# with split operands).  Worst ratio measured over the cases of tests/test_gpu_torso_motion.py on an H100 80GB HBM3 (700 W power limit):
# fp16 1.61e-6 (the K = 9 fuser, 114 -> 32, 7^3), split 6.84e-6 (the K = 4 fuser, 89 -> 32).  beta = 2^-18 = 3.8e-6 (2.4x) and 2^-16 = 1.5e-5 (2.2x).
BETA3 = {False: 2.0 ** -18, True: 2.0 ** -16}


def ref_conv(x, w, taps, up, bias=None):
    """float64 reference: x [N,C,D,H,W], w [nph,taps,O,C] -> [N,O,D,H',W'] (up: the 4 parity phases of (kd,2,2) taps)."""
    kd, kh, kw = taps
    nph, _, O, C = w.shape
    wk = w.reshape(nph, kd, kh, kw, O, C).permute(0, 4, 5, 1, 2, 3)
    if not up:
        y = F.conv3d(x, wk[0], padding=(kd // 2, kh // 2, kw // 2))
    else:
        N, _, D, H, W = x.shape
        y = x.new_zeros(N, O, D, 2 * H, 2 * W)
        for p in range(2):
            for q in range(2):
                xp = F.pad(x, (1 - q, q, 1 - p, p, kd // 2, kd // 2))
                y[..., p::2, q::2] = F.conv3d(xp, wk[p * 2 + q])
    return y if bias is None else y + bias.double()[None, :, None, None, None]


def mean2x2(x: torch.Tensor) -> torch.Tensor:
    """[..., 2H, 2W, C] -> [..., H, W, C]: the mean of each 2x2 block (AvgPool (1, 2, 2), the exact-1/2 bilinear resize)."""
    return 0.25 * ((x[..., 0::2, 0::2, :] + x[..., 0::2, 1::2, :]) + (x[..., 1::2, 0::2, :] + x[..., 1::2, 1::2, :]))


def pool(x: torch.Tensor):
    """(ref, S) of r3dp_mf_pool / r3dp_mf_head_bcast's mean: x float64 [..., 2H, 2W, C]."""
    return mean2x2(x), mean2x2(x.abs())


def head_input(rgb: torch.Tensor, wts: torch.Tensor):
    """(ref, S) of r3dp_mf_head_input: rgb [N,3,2H,2W], wts [N,1,2H,2W] float64 -> [N,H,W,4]."""
    x = torch.cat([rgb, wts], 1).permute(0, 2, 3, 1)
    return pool(x)


def affine_relu(x: torch.Tensor, s: torch.Tensor, t: torch.Tensor):
    """(ref, S) of r3dp_tw_affine_relu on x float64 [..., C] with the fp32 scale / shift s, t [C]."""
    s, t = s.double(), t.double()
    return torch.relu(x * s + t), x.abs() * s.abs() + t.abs()


def grid(n: int, dev) -> torch.Tensor:
    """make_coordinate_grid's exact coordinates 2 i / (n - 1) - 1 (float64)."""
    return 2 * (torch.arange(n, device=dev, dtype=torch.float64) / (n - 1)) - 1


def _grid3(D, H, W, dev):
    z, y, x = torch.meshgrid(grid(D, dev), grid(H, dev), grid(W, dev), indexing='ij')
    return torch.stack([x, y, z], -1)                                            # components (W, H, D)


def _motion_coord_error(g, kd, s):
    """ds of the sparse motion s = fl(fl(g' - kd) + ks) (module docstring); kd None: the identity grid."""
    if kd is None:
        return torch.full_like(g, 3 * U)
    return 1.01 * (3 * U + U * ((g - kd).abs() + s.abs()))


def _local_slopes(vol: torch.Tensor, P: int):
    """vol [C,D,H,W] float64 zero-padded by P -> per axis (x, y, z) the [D+2P, H+2P, W+2P] max over channels and over the cells within one
    voxel of cell (z0, y0, x0) of the |difference of two neighbours| along that axis: window z0-1..z0+2 x y0-1..y0+2 x x0-1..x0+1 (x)."""
    v = F.pad(vol, (P, P + 1, P, P + 1, P, P + 1))                             # one extra voxel past the end: every edge has its pair
    out = []
    for ax in (3, 2, 1):                                                       # x (W), y (H), z (D)
        e = (v.narrow(ax, 1, v.shape[ax] - 1) - v.narrow(ax, 0, v.shape[ax] - 1)).abs().amax(0)   # [D', H', W'] one shorter along ax
        e = F.pad(e, [0, 1 if ax == 3 else 0, 0, 1 if ax == 2 else 0, 0, 1 if ax == 1 else 0])
        k = [4, 4, 4]
        k[ax - 1] = 3
        e = F.pad(e[None, None], (1, k[2] - 2, 1, k[1] - 2, 1, k[0] - 2))      # window starts one voxel before the cell
        out.append(F.max_pool3d(e, tuple(k), stride=1)[0, 0])
    return out


def mf_input(fc: torch.Tensor, kp_s: torch.Tensor, kp_d: torch.Tensor):
    """r3dp_mf_input for ONE frame: fc float64 [D,H,W,4] (the volume that frame reads), kp_s / kp_d float64 [K,3] (the fp32 values) ->
    (ref, S, extra) [D,H,W,(K+1)*5] before the store (module docstring); channel k*5 is the heatmap, k*5 + 1..4 the sampled source."""
    D, H, W, _ = fc.shape
    K = kp_s.shape[0]
    dev = fc.device
    g = _grid3(D, H, W, dev)
    vol = fc.permute(3, 0, 1, 2)[None]
    P = 40
    Lx, Ly, Lz = _local_slopes(vol[0], P)
    n1 = torch.tensor([W - 1, H - 1, D - 1], device=dev, dtype=torch.float64)
    refs, Ss, extras = [], [], []
    for k in range(K + 1):
        if k == 0:
            hm = torch.zeros(D, H, W, dtype=torch.float64, device=dev)
            e_hm = torch.zeros_like(hm)
            s, ds = g, _motion_coord_error(g, None, g)
        else:
            Es, Gs = [], []
            for kp in (kp_d[k - 1], kp_s[k - 1]):
                d = g - kp
                a = -0.5 * (d * d).sum(-1) / SIGMA2
                G = torch.exp(a)
                da = 8 * U * a.abs() + 100 * d.abs().sum(-1) * 3 * U
                Gs.append(G)
                Es.append(G * (1.01 * da + 4 * U))
            hm = Gs[0] - Gs[1]
            e_hm = (Es[0] + Es[1]) * (1 + U) + U * hm.abs() + 2 * FLOOR_EXP
            s = g - kp_d[k - 1] + kp_s[k - 1]
            ds = _motion_coord_error(g, kp_d[k - 1], s)
        samp = F.grid_sample(vol, s[None], mode='bilinear', padding_mode='zeros', align_corners=True)[0].permute(1, 2, 3, 0)
        S = F.grid_sample(vol.abs(), s[None], mode='bilinear', padding_mode='zeros', align_corners=True)[0].permute(1, 2, 3, 0)
        ix = (s + 1) / 2 * n1
        dix = 1.01 * (n1 / 2 * (ds + U * (s + 1).abs()) + U * ix.abs())
        i0 = torch.floor(ix).long() + P                                          # cell index in the padded volume
        i0 = torch.minimum(torch.maximum(i0, torch.zeros_like(i0)), torch.tensor([W + 2 * P - 1, H + 2 * P - 1, D + 2 * P - 1], device=dev))
        lip = sum(dix[..., a] * L[i0[..., 2], i0[..., 1], i0[..., 0]] for a, L in enumerate((Lx, Ly, Lz)))
        refs += [hm[..., None], samp]
        Ss += [torch.zeros_like(hm)[..., None], S]
        extras += [e_hm[..., None], (1.01 * lip)[..., None].expand(-1, -1, -1, 4)]
    return torch.cat(refs, -1), torch.cat(Ss, -1), torch.cat(extras, -1)


def deform(logits: torch.Tensor, kp_s: torch.Tensor, kp_d: torch.Tensor):
    """r3dp_mf_deform for ONE frame: logits float64 [D,H,W,K+1] (the fp32 values), kp_s / kp_d [K,3] -> (ref, S, extra) [D,H,W,3]."""
    D, H, W, K1 = logits.shape
    K = K1 - 1
    g = _grid3(D, H, W, logits.device)
    m = torch.softmax(logits, -1)
    r = 4 * U + 1.01 * U * (logits - logits.amax(-1, keepdim=True)).abs()
    q = r + r.amax(-1, keepdim=True) + gamma(K) + U
    ref, S, extra = 0, 0, 0
    for k in range(K + 1):
        if k == 0:
            s, ds = g, _motion_coord_error(g, None, g)
        else:
            s = g - kp_d[k - 1] + kp_s[k - 1]
            ds = _motion_coord_error(g, kp_d[k - 1], s)
        mk = m[..., k:k + 1]
        ref = ref + mk * s
        S = S + mk * s.abs()
        extra = extra + mk * (s.abs() * q[..., k:k + 1] + ds)
    return ref, S, 1.01 * extra


def occlusion(x: torch.Tensor, wk: torch.Tensor, bk: torch.Tensor, split: bool):
    """r3dp_mf_occlusion for ONE frame: x float64 [D,H,W,C] (hi + lo), wk fp32 [D,49,C,2], bk [2] -> [(ref, S, extra)] for occ and occ2,
    each [H,W].  The bound follows the kernel's fma chain (module docstring)."""
    D, H, W, C = x.shape
    out = []
    for o in range(2):
        v = torch.zeros(H * W, dtype=torch.float64, device=x.device)
        sabs = torch.zeros_like(v)
        psum = torch.zeros_like(v)
        for d in range(D):
            xu = F.unfold(x[d:d + 1].permute(0, 3, 1, 2), 7, padding=3).view(C, 49, H * W).transpose(0, 1).reshape(49 * C, H * W)  # (tap, c)
            prod = xu * wk[d, ..., o].double().reshape(49 * C, 1)               # the chain's terms of this depth slice, in its order
            cs = v[None] + prod.cumsum(0)
            psum = psum + cs.abs().sum(0)
            v = cs[-1]
            sabs = sabs + prod.abs().sum(0)
        b = float(bk[o])
        v = v + b
        dv = 1.01 * U * psum + (U * sabs if split else 0) + U * v.abs()
        s = torch.sigmoid(v)
        out.append((s.view(H, W), s.view(H, W), (1.01 * s * (1 - s) * dv + FLOOR_EXP).view(H, W)))
    return out
