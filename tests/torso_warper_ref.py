"""Reference modules of the torso warper for the stage-2 tests: the reference's own network2.Generator and model2 classes as staged under
oracle/_ref/ by oracle/make_ref.py (None when not staged), seeded synthetic weights for them, and a float64 restatement of stage 2 built from
the host-side folding of real3dportrait_b200.torso_warp."""
import torch
import torch.nn.functional as F

from oracle import ref_runner
from real3dportrait_b200 import torso_warp as tw


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
