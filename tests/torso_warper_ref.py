"""Reference modules of the torso warper for the stage-2 tests: the reference's own network2.Generator and model2 classes as staged under
oracle/_ref/ by oracle/make_ref.py (None when not staged), seeded synthetic weights for them, and a float64 restatement of stage 2 built from
the host-side folding of real3dportrait_b200.torso_warp."""
import torch
import torch.nn.functional as F

from oracle import ref_runner
from real3dportrait_b200 import torso_warp as tw
from secc2plane_reference import cop_of, launch_signature  # noqa: F401  (launch_signature re-exported for the launch tests)


def ref_classes():
    """(Generator, WarpBasedTorsoModelMediaPipe) of the staged reference, or None."""
    if not ref_runner.available():
        return None
    try:
        m = ref_runner.modules()
        m['hparams'].update({'torso_kp_num': 4, 'torso_inp_mode': 'rgb_alpha'})
        from modules.real3d.facev2v_warp.network2 import Generator
        from modules.real3d.facev2v_warp.model2 import WarpBasedTorsoModelMediaPipe
    except Exception:                                   # noqa: BLE001  (staged without the warper's modules)
        return None
    return Generator, WarpBasedTorsoModelMediaPipe


def make_predictor():
    """model2.py:212-219 (a plain nn.Sequential; built here so a test needs no reference module for it)."""
    nn = torch.nn
    return nn.Sequential(nn.Conv2d(65, 32, 3, 1, 1), nn.ReLU(), nn.Conv2d(32, 32, 3, 1, 1), nn.ReLU(), nn.Conv2d(32, 1, 3, 1, 1), nn.Sigmoid())


def randomize(module: torch.nn.Module, seed: int) -> torch.nn.Module:
    """Seeded values for every parameter and buffer a trained checkpoint would carry: conv weights (fan-in scaled), biases, BatchNorm affine
    and running statistics, spectral-norm u / v (the top singular pair of each weight).  Eval mode."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, t in sorted(list(module.named_parameters()) + list(module.named_buffers()), key=lambda kv: kv[0]):
            if name.endswith('num_batches_tracked'):
                continue
            leaf = name.rsplit('.', 1)[-1]
            if leaf in ('weight', 'weight_orig') and t.dim() > 1:
                t.copy_(torch.randn(t.shape, generator=g) / (t[0].numel() ** 0.5))
            elif leaf in ('weight_u', 'weight_v'):
                v = torch.randn(t.shape, generator=g)
                t.copy_(v / v.norm())
            elif leaf == 'running_var':
                t.copy_(0.5 + torch.rand(t.shape, generator=g))
            elif leaf == 'weight':                                   # BatchNorm gamma
                t.copy_(0.8 + 0.4 * torch.rand(t.shape, generator=g))
            else:                                                    # biases, BatchNorm beta, running_mean
                t.copy_(0.1 * torch.randn(t.shape, generator=g))
        # a trained checkpoint carries the converged power iteration: u, v = the top singular pair, so sigma = u . (W v) is the spectral norm
        # (random u, v give a random, possibly near-zero sigma and activations that overflow)
        for m in module.modules():
            if hasattr(m, 'weight_orig'):
                U, S, Vh = torch.linalg.svd(m.weight_orig.detach().double().reshape(m.weight_orig.shape[0], -1), full_matrices=False)
                m.weight_u.copy_(U[:, 0].to(m.weight_u.dtype))
                m.weight_v.copy_(Vh[0].to(m.weight_v.dtype))
    return module.eval()


def make_stage2_inputs(N: int, h: int, seed: int):
    """fs [N,32,16,h,h] (the masked appearance volume), deformation [N,16,h,h,3] with coordinates past [-1, 1] (the border padding), occlusion_2
    [N,1,h,h] in (0, 1)."""
    g = torch.Generator().manual_seed(seed)
    fs = torch.randn(N, 32, 16, h, h, generator=g)
    deformation = 1.15 * (2 * torch.rand(N, 16, h, h, 3, generator=g) - 1)
    occ = torch.sigmoid(torch.randn(N, 1, h, h, generator=g))
    return fs, deformation, occ


def reference_stage2(gen, pred, fs, deformation, occ2):
    """The reference's Generator(..., return_hid=True) and the predictor on its hidden features (model2.py:260-262)."""
    rgb, hid = gen(fs, deformation, None, return_hid=True)
    occ = pred(torch.cat([hid, F.interpolate(occ2, size=hid.shape[-2:], mode='bilinear')], dim=1))
    return rgb, hid, occ


def folded_stage2_f64(gen, pred, fs, deformation, occ2):
    """Stage 2 restated in float64 from the folded weights (eval spectral norm + BatchNorm folded, BN1 of each ResBlock as an affine map,
    nearest-up + 3x3 as four parity phases of 2x2 taps): the computation the kernels run, without their rounding."""
    d = lambda t: t.double()                                                   # noqa: E731
    fs, deformation, occ2 = d(fs), d(deformation), d(occ2)
    N, _, D, h, w = fs.shape
    x = F.grid_sample(fs, deformation, align_corners=True, padding_mode='border').reshape(N, -1, h, w)
    wi, bi = tw.fold_cna(gen.in_conv)
    x = F.leaky_relu(F.conv2d(x, wi, bi, padding=1), 0.2)
    x = F.conv2d(x, d(gen.mid_conv.weight.detach()), d(gen.mid_conv.bias.detach()))
    for rb in gen.res:
        nac1, nac2 = rb.layers[0].layers, rb.layers[1].layers
        s1, t1 = tw.bn_affine(nac1[0])
        s2, t2 = tw.bn_affine(nac2[0])
        w1 = tw.sn_weight(nac1[2]) * s2[:, None, None, None]
        b1 = d(nac1[2].bias.detach()) * s2 + t2
        a = torch.relu(x * s1[:, None, None] + t1[:, None, None])
        a = torch.relu(F.conv2d(a, w1, b1, padding=1))
        x = x + F.conv2d(a, tw.sn_weight(nac2[2]), d(nac2[2].bias.detach()), padding=1)
    for ub in gen.up:
        wu, bu = tw.fold_cna(ub.layers[1])
        x = torch.relu(conv_up_nearest_phases(x, tw.compose_nearest_up(wu), bu))
    rgb = F.conv2d(x, d(gen.out_conv.weight.detach()), d(gen.out_conv.bias.detach()), padding=3)
    t = torch.cat([x, F.interpolate(occ2, size=x.shape[-2:], mode='bilinear')], dim=1)
    for i, act in ((0, torch.relu), (2, torch.relu), (4, torch.sigmoid)):
        t = act(F.conv2d(t, d(pred[i].weight.detach()), d(pred[i].bias.detach()), padding=1))
    return rgb, x, t


# ---- the library's launch sequence, restated from the architecture ----------------------------------------------------------------------
#: the optional operands of the entry points that take one: whether each is given is part of a launch's arguments (see launch_plan)
OPTIONAL_OPERANDS = {'r3dp_mf_conv3d': ('res',), 'r3dp_tw_conv': ('residual',), 'r3dp_tw_narrow_conv': ('xa', 'xf', 'ex')}
MF_DOWN = [64, 128, 256, 512, 1024]                     # network2.py MotionFieldEstimator('standard'): down_seq[1:], up_seq[1:]
MF_UP = [512, 256, 128, 64, 32]
MF_ENC_RES = 3                                          # tgt_head_encoder: ConvBlock2D 7x7 4 -> 32, then three ResBlock2D(32)
GEN_RES = 6                                             # Generator('standard'): six ResBlock2D(256), up_seq [256, 128, 64]


def launch_plan(K, N, split, clip=True):
    """Every r3dp_mf_* / r3dp_tw_* launch of one warper call with torso_motion='cuda' and torso_stage2='cuda' (torso_warp.motion, stage2,
    hid_to_nchw) on N frames, torso_kp_num K, split = tc_exact, as (tag, C entry point, args).  args are the non-pointer arguments in C
    order, then for the entry points of OPTIONAL_OPERANDS whether each optional operand is given.  clip: the appearance volume and the
    estimator's compressed source come from the per-clip cache (one volume read by every frame when N > 1); otherwise each frame has its own.
    Written from the architecture (network2.py MotionFieldEstimator('standard') and Generator, model2.py:212-263) and the layouts the
    kernels document (NDHWC / NHWC, [hi | lo] halves when split, 32-channel K steps), not from the module's code."""
    plan = []
    wide = 2 if split else 1
    sp = int(bool(split))
    shared = int(bool(clip) and N > 1)
    D, S = 16, 64                                        # the estimator's volume: 16 x 64 x 64
    c0 = (K + 1) * 5                                     # heatmap + 4 deformed source channels per keypoint and the identity
    P0 = (c0 + 31) // 32 * 32
    CF = P0 + 64                                         # fuser input: [input | pad | last up block 32 | head features 32]

    def add(tag, fn, *args):
        plan.append((tag, fn, tuple(args)))

    def conv3d(tag, xs, xlo, cin, dims, taps, up, O, relu, ys, yc0, ylo, out_f32=0, res=False):
        add(tag, 'r3dp_mf_conv3d', xs, xlo, cin, *dims, *taps, up, O, cop_of(O), relu, ys, yc0, ylo, out_f32, sp, bool(res))

    # motion(): the estimator (network2.py:211-244)
    add('mf.input', 'r3dp_mf_input', shared, N, K, D, S, S, P0, CF * wide, CF, sp)
    xs, xlo, cin, hw = CF * wide, CF, P0, S
    for i, O in enumerate(MF_DOWN):                      # DownBlock3D: conv 3x3x3 + BN + ReLU, AvgPool3d (1, 2, 2)
        conv3d(f'mf.down.{i}', xs, xlo, cin, (N, D, hw, hw), (3, 3, 3), 0, O, 1, O * wide, 0, O)
        hw //= 2
        add(f'mf.down.{i}.pool', 'r3dp_mf_pool', N, D, hw, hw, O, O * wide, O, O * wide, O, sp)
        xs, xlo, cin = O * wide, O, O
    for i, O in enumerate(MF_UP):                        # UpBlock3D: nearest (1, 2, 2) + conv 3x3x3 + BN + ReLU as 4 phases of 3x2x2 taps
        last = i + 1 == len(MF_UP)                       # the last block writes its 32 channels at P0 of the fuser input
        ys, yc0, ylo = (CF * wide, P0, CF) if last else (O * wide, 0, O)
        conv3d(f'mf.up.{i}', xs, xlo, cin, (N, D, hw, hw), (3, 2, 2), 1, O, 1, ys, yc0, ylo)
        xs, xlo, cin, hw = O * wide, O, O, 2 * hw
    H2 = 2 * S                                           # the tgt-head encoder at 128^2 (depth 1), 32 channels
    add('mf.head_input', 'r3dp_mf_head_input', N, H2, H2, 32, 32 * wide, 32, sp)
    e = (32 * wide, 32, 32)
    conv3d('mf.enc.0', *e, (N, 1, H2, H2), (1, 7, 7), 0, 32, 1, 32 * wide, 0, 32)
    for r in range(MF_ENC_RES):                          # ResBlock2D: BN1 + ReLU, conv1 (BN2 folded) + ReLU, conv2 + residual
        add(f'mf.enc.{r + 1}.bn1', 'r3dp_tw_affine_relu', N, H2, H2, 32, sp)
        conv3d(f'mf.enc.{r + 1}.conv1', *e, (N, 1, H2, H2), (1, 3, 3), 0, 32, 1, 32 * wide, 0, 32)
        conv3d(f'mf.enc.{r + 1}.conv2', *e, (N, 1, H2, H2), (1, 3, 3), 0, 32, 0, 32 * wide, 0, 32, res=True)
    add('mf.head_bcast', 'r3dp_mf_head_bcast', N, D, S, S, 32, 32 * wide, 32, CF * wide, P0 + 32, CF, sp)
    conv3d('mf.fuser', CF * wide, CF, CF, (N, D, S, S), (7, 7, 7), 0, 32, 0, 32 * wide, 0, 32)
    ls = (K + 2) // 2 * 2                                # K + 1 mask logits per voxel at an even fp32 stride
    conv3d('mf.mask', 32 * wide, 32, 32, (N, D, S, S), (7, 7, 7), 0, K + 1, 0, ls, 0, 0, out_f32=1)
    add('mf.deform', 'r3dp_mf_deform', ls, N, K, D, S, S)
    add('mf.occlusion', 'r3dp_mf_occlusion', N, D, S, S, 32, 32 * wide, 32, sp)
    # stage2(): Generator (network2.py:248-301) and the occlusion_2 predictor (model2.py:212-219, 260-263)
    add('tw.gather3d', 'r3dp_tw_gather3d', shared, N, 32, D, S, S, sp)

    def tw_conv(tag, I, O, k, slope, res=False):
        add(tag, 'r3dp_tw_conv', N, I, O, S, S, k, slope, sp, bool(res))
    tw_conv('tw.in_conv', 32 * D, 256, 3, 0.2)
    tw_conv('tw.mid_conv', 256, 256, 1, 1.0)
    for r in range(GEN_RES):
        add(f'tw.res.{r}.bn1', 'r3dp_tw_affine_relu', N, S, S, 256, sp)
        tw_conv(f'tw.res.{r}.conv1', 256, 256, 3, 0.0)
        tw_conv(f'tw.res.{r}.conv2', 256, 256, 3, 1.0, res=True)
    add('tw.up.0', 'r3dp_tw_conv_up_nearest', N, 256, 128, S, S, 0.0, sp)
    add('tw.up.1', 'r3dp_tw_conv_up_nearest', N, 128, 128, 2 * S, 2 * S, 0.0, sp)      # 64 couts packed with zero filters to 128
    H = 4 * S
    hs, lo = 128 * wide, 128 if split else 0                                           # hid: 128 channels per half, 64 real
    add('tw.out_conv', 'r3dp_tw_narrow_conv', hs, 64, lo, 0, 0, 0, 0, N, H, H, 7, 3, 0, 1, True, False, False)
    add('tw.pred.0', 'r3dp_tw_narrow_conv', hs, 64, lo, 0, 0, S, S, N, H, H, 3, 32, 1, 0, True, False, True)
    add('tw.pred.1', 'r3dp_tw_narrow_conv', 0, 0, 0, 32, 32, 0, 0, N, H, H, 3, 32, 1, 0, False, True, False)
    add('tw.pred.2', 'r3dp_tw_narrow_conv', 0, 0, 0, 32, 32, 0, 0, N, H, H, 3, 1, 2, 1, False, True, False)
    add('tw.hid_to_nchw', 'r3dp_tw_hid_to_nchw', N, 64, H, H, hs, lo)
    return plan


def conv_up_nearest_phases(x, w4, b):
    """Output parity (p, q) of upsample(x2, nearest) -> conv3x3, computed as 2x2 taps of w4[p*2+q] on x: taps (dy, dx) with dy in {p-1, p}."""
    N, _, H, W = x.shape
    out = x.new_zeros(N, w4.shape[1], 2 * H, 2 * W)
    xp = F.pad(x, (1, 1, 1, 1))
    for p in range(2):
        for q in range(2):
            acc = 0
            for dy in (p - 1, p):
                for dx in (q - 1, q):
                    tap = w4[p * 2 + q][:, :, dy + 1, dx + 1]
                    acc = acc + torch.einsum('oi,nihw->nohw', tap, xp[:, :, 1 + dy:1 + dy + H, 1 + dx:1 + dx + W])
            out[:, :, p::2, q::2] = acc + b[None, :, None, None]
    return out
