"""The torso warper (modules/real3d/facev2v_warp/model2.py:199-287, WarpBasedTorsoModelMediaPipe, torso_model_version v2) with its stage 2 on
this library's kernels: the deformation-based Generator (network2.py:248-301) and the occlusion_2_predictor (model2.py:212-219, 260-263).

Stage 1 (model2.py:222-258) is restated here and calls the caller's `appearance_extractor` and `motion_field_estimator` children, which stay
PyTorch; with torso_motion='cuda' the motion_field_estimator runs on the 3-D convolutions of csrc/conv3d_tc.cu instead (MotionWeights,
motion()).  Stage 2 reads its weights from the caller's `deform_based_generator` and `occlusion_2_predictor`: eval spectral norm and eval
BatchNorm are folded on the host in float64, then packed once (Stage2Weights, cached by the SR head until its parameters are reloaded).

Layout of stage 2 (N images; tc: fp16 NHWC activations, tc_exact: [hi | lo] halves):
  gather3d  fs [N,16,64,64,32] fp32 NDHWC + deformation -> [N,64,64,512]
  in_conv   3x3 512 -> 256 + BN + LeakyReLU(0.2)                 (conv_tc3, 64-wide maps)
  mid_conv  1x1 256 -> 256                                       -> x (the residual stream)
  res x6    x += conv2(relu(bn2(conv1(relu(bn1(x))))))            bn1 + relu: affine_relu launch; bn2 folded into conv1 (ReLU epilogue)
  up.0/1    nearest x2 + 3x3 + BN + ReLU: 256 -> 128 at 128^2, 128 -> 64 (packed as 128 with zero filters) at 256^2
  out_conv  7x7 64 -> 3 -> rgb_torso [N,3,256,256] fp32           (CUDA cores, fp32)
  predictor cat[hid, bilinear_up(occlusion_2)] 65 -> 32 ReLU -> 32 ReLU -> 1 sigmoid (CUDA cores, fp32; the 65th channel is resized on the fly)
ret['losses'] (model2.py:266-279) is training-only and is not computed."""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.nn.functional as F

from . import _capi as capi
from . import sr_tc

KP_IDX = {4: [0, 8, 16, 27], 9: [0, 3, 6, 8, 10, 13, 16, 27, 33]}     # model2.py:238-243


# ---- weight folding (host, float64) --------------------------------------------------------------------------------------------------
def sn_weight(conv: torch.nn.Module) -> torch.Tensor:
    """Eval-mode spectral norm (torch.nn.utils.spectral_norm): weight_orig / (u . (W_mat v)) with the stored u, v; no power iteration.
    A conv without the hook returns its weight."""
    if not hasattr(conv, 'weight_orig'):
        return conv.weight.detach().double()
    w = conv.weight_orig.detach().double()
    u, v = conv.weight_u.detach().double(), conv.weight_v.detach().double()
    sigma = torch.dot(u, w.reshape(w.shape[0], -1) @ v)
    return w / sigma


def bn_affine(bn: torch.nn.Module):
    """Eval BatchNorm / SyncBatchNorm as y = s * x + t (float64)."""
    s = bn.weight.detach().double() / torch.sqrt(bn.running_var.detach().double() + bn.eps)
    return s, bn.bias.detach().double() - bn.running_mean.detach().double() * s


def fold_cna(block) -> tuple:
    """ConvBlock2D / ConvBlock3D 'CNA' (conv -> BN -> act): (W [O,I,k,k(,k)], b [O]) float64 with the BN folded in."""
    conv, bn = block.layers[0], block.layers[1]
    w, b = sn_weight(conv), conv.bias.detach().double()
    s, t = bn_affine(bn)
    return w * s.reshape(-1, *[1] * (w.dim() - 1)), b * s + t


def compose_nearest_up(w: torch.Tensor) -> torch.Tensor:
    """3x3 weights [O,I,3,3] of a conv applied after nn.Upsample(x2, nearest) -> [4,O,I,3,3]: set p*2+q holds the 2x2 taps of output
    parity (p, q) on the low-resolution input, at (dy+1, dx+1).  Even output: dy=-1 <- w[0], dy=0 <- w[1]+w[2]; odd output: dy=0 <- w[0]+w[1],
    dy=+1 <- w[2]; the same per axis.  Exact at the borders: the upsampled map's zero padding is the input's."""
    A = w.new_zeros(2, 3, 3)                  # A[p][dy+1][ky]
    A[0, 0, 0] = 1; A[0, 1, 1] = 1; A[0, 1, 2] = 1
    A[1, 1, 0] = 1; A[1, 1, 1] = 1; A[1, 2, 2] = 1
    return torch.einsum('pak,qbl,oikl->pqoiab', A, A, w).reshape(4, *w.shape)


class Stage2Weights:
    """Folded and packed weights of stage 2 for one sr_mode (split = tc_exact)."""

    def __init__(self, gen: torch.nn.Module, occ: torch.nn.Sequential, split: bool):
        self.split = bool(split)
        dev = next(gen.parameters()).device
        f32 = lambda t: t.float().contiguous().to(dev)                                    # noqa: E731

        def pack(w, b, in_ch, nw=1):
            # w [nw,O,I,3,3] float64 -> packed fp16 [nw,9,Opad,Ipad] (Opad = 128 | 256), bias [Opad] fp32
            O, I = w.shape[1:3]
            Op = max(128, (O + 127) // 128 * 128)
            w9 = torch.zeros(nw, Op, in_ch, 3, 3, dtype=torch.float64, device=w.device)
            w9[:, :O, :I] = w
            Ip = (in_ch + 63) // 64 * 64
            out = torch.empty(nw, 9, Op, Ip * (2 if split else 1), device=dev, dtype=torch.float16)
            capi.check(sr_tc._fn('pack_weights', split)(capi.ptr(f32(w9)), nw, Op, in_ch, capi.ptr(out, torch.float16), capi.stream()))
            bias = torch.zeros(Op, device=dev)
            bias[:O] = f32(b)
            return out, bias

        def k1_as_3x3(w):
            w3 = w.new_zeros(w.shape[0], w.shape[1], 3, 3)
            w3[:, :, 1, 1] = w[:, :, 0, 0]
            return w3

        w, b = fold_cna(gen.in_conv)
        self.in_conv = pack(w[None], b, w.shape[1])
        mc = gen.mid_conv
        self.mid_conv = pack(k1_as_3x3(mc.weight.detach().double())[None], mc.bias.detach().double(), mc.in_channels)
        self.res = []
        for rb in gen.res:
            nac1, nac2 = rb.layers[0].layers, rb.layers[1].layers                       # NAC: BN, ReLU, conv
            s1, t1 = bn_affine(nac1[0])
            s2, t2 = bn_affine(nac2[0])
            w1, b1 = sn_weight(nac1[2]), nac1[2].bias.detach().double()
            w2, b2 = sn_weight(nac2[2]), nac2[2].bias.detach().double()
            self.res.append((f32(s1), f32(t1), pack((w1 * s2[:, None, None, None])[None], b1 * s2 + t2, w1.shape[1]), pack(w2[None], b2, w2.shape[1])))
        self.up = []
        for ub in gen.up:
            w, b = fold_cna(ub.layers[1])
            self.up.append((pack(compose_nearest_up(w), b, w.shape[1], nw=4), w.shape[0]))
        oc = gen.out_conv
        self.out_conv = (f32(oc.weight.detach().double().permute(2, 3, 1, 0)), f32(oc.bias.detach().double()), oc.kernel_size[0])
        self.occ = [(f32(c.weight.detach().double().permute(2, 3, 1, 0)), f32(c.bias.detach().double())) for c in (occ[0], occ[2], occ[4])]


def stage2(wts: Stage2Weights, fs_ndhwc: torch.Tensor, deformation: torch.Tensor, occlusion_2: torch.Tensor):
    """Generator(fs, deformation, return_hid=True) + occlusion_2_predictor -> (rgb_torso [N,3,H,W] fp32, hid16 NHWC fp16, occ2 [N,1,H,W] fp32).
    fs_ndhwc [N or 1,D,h,w,C] fp32 (one volume shared by the batch is broadcast), deformation [N,D,h,w,3], occlusion_2 [N,1,h',w']."""
    L, sp, st = capi.lib(), wts.split, capi.stream()
    wide = 2 if sp else 1
    N, D, h, w, _ = deformation.shape
    shared = fs_ndhwc.shape[0] == 1 and N > 1                          # one volume read by every image: no per-frame copies of it
    fs_ndhwc, deformation = capi.f32(fs_ndhwc), capi.f32(deformation)
    C = fs_ndhwc.shape[-1]
    dev = deformation.device
    g = torch.empty(N, h, w, C * D * wide, device=dev, dtype=torch.float16)
    with capi.region('torso_stage2'):
        capi.check(L.r3dp_tw_gather3d(capi.ptr(fs_ndhwc), int(shared), capi.ptr(deformation), N, C, D, h, w, capi.ptr(g, torch.float16), int(sp), st))

        def conv(x, packed, H, W, slope, residual=None, k=3):
            wp, bias = packed
            y = torch.empty(N, H, W, wp.shape[2] * wide, device=dev, dtype=torch.float16)
            capi.check(L.r3dp_tw_conv(capi.ptr(x, torch.float16), capi.ptr(wp, torch.float16), capi.ptr(bias), N, x.shape[-1] // wide, wp.shape[2], H, W,
                                      k, slope, capi.ptr(residual, torch.float16), capi.ptr(y, torch.float16), int(sp), st))
            return y

        x = conv(conv(g, wts.in_conv, h, w, 0.2), wts.mid_conv, h, w, 1.0, k=1)
        C0 = x.shape[-1] // wide
        for s1, t1, c1, c2 in wts.res:
            a = torch.empty_like(x)
            capi.check(L.r3dp_tw_affine_relu(capi.ptr(x, torch.float16), capi.ptr(s1), capi.ptr(t1), N, h, w, C0, int(sp), capi.ptr(a, torch.float16), st))
            x = conv(conv(a, c1, h, w, 0.0), c2, h, w, 1.0, residual=x)
        H, W = h, w
        for (wp, bias), O in wts.up:
            y = torch.empty(N, 2 * H, 2 * W, wp.shape[2] * wide, device=dev, dtype=torch.float16)
            capi.check(L.r3dp_tw_conv_up_nearest(capi.ptr(x, torch.float16), capi.ptr(wp, torch.float16), capi.ptr(bias), N, x.shape[-1] // wide,
                                                 wp.shape[2], H, W, 0.0, capi.ptr(y, torch.float16), int(sp), st))
            x, H, W = y, 2 * H, 2 * W
        hid, Chid = x, wts.up[-1][1]
        pad = hid.shape[-1] // wide                                   # channels of one half (the hi half holds Chid real + zero-filter channels)
        lo = pad if sp else 0
        wk, bk, K = wts.out_conv
        rgb = torch.empty(N, 3, H, W, device=dev)
        capi.check(L.r3dp_tw_narrow_conv(capi.ptr(hid, torch.float16), hid.shape[-1], Chid, lo, None, 0, 0, None, 0, 0, capi.ptr(wk), capi.ptr(bk),
                                         N, H, W, K, 3, 0, 1, capi.ptr(rgb), st))
        occ = capi.f32(occlusion_2)
        (w0, b0), (w1, b1), (w2, b2) = wts.occ
        t0 = torch.empty(N, H, W, 32, device=dev)
        capi.check(L.r3dp_tw_narrow_conv(capi.ptr(hid, torch.float16), hid.shape[-1], Chid, lo, None, 0, 0, capi.ptr(occ), occ.shape[-2], occ.shape[-1],
                                         capi.ptr(w0), capi.ptr(b0), N, H, W, 3, 32, 1, 0, capi.ptr(t0), st))
        t1 = torch.empty_like(t0)
        capi.check(L.r3dp_tw_narrow_conv(None, 0, 0, 0, capi.ptr(t0), 32, 32, None, 0, 0, capi.ptr(w1), capi.ptr(b1), N, H, W, 3, 32, 1, 0, capi.ptr(t1), st))
        occ2 = torch.empty(N, 1, H, W, device=dev)
        capi.check(L.r3dp_tw_narrow_conv(None, 0, 0, 0, capi.ptr(t1), 32, 32, None, 0, 0, capi.ptr(w2), capi.ptr(b2), N, H, W, 3, 1, 2, 1, capi.ptr(occ2), st))
    return rgb, hid, occ2


def compose_nearest_up3d(w: torch.Tensor) -> torch.Tensor:
    """3x3x3 weights [O,I,3,3,3] of a conv applied after nn.Upsample((1,2,2), nearest) -> [4,O,I,3,2,2]: depth untouched, phase p*2+q holds
    the 2x2 (H, W) taps of output parity (p, q) on the low-resolution input; tap (iy, ix) reads input offset (p + iy - 1, q + ix - 1)."""
    O, I = w.shape[:2]
    g = compose_nearest_up(w.reshape(O, I * 3, 3, 3)).reshape(4, O, I, 3, 3, 3)      # [.., kz, dy+1, dx+1]
    out = w.new_zeros(4, O, I, 3, 2, 2)
    for p in range(2):
        for q in range(2):
            out[p * 2 + q] = g[p * 2 + q][..., p:p + 2, q:q + 2]
    return out


# ---- the motion-field estimator (network2.py:162-244) on the 3-D convolutions of csrc/conv3d_tc.cu -------------------------------------
MOTION_D, MOTION_HW = 16, 64


def pack_conv3d(w: torch.Tensor, b: torch.Tensor, cin: int, split: bool, cin_map=None, cout_tile: Optional[int] = None):
    """Folded float64 weights [nph,O,I,kd,kh,kw] -> (packed fp16 [nph, taps, cop, cin (x2 split: [hi | lo] of w * 2^10)], bias [cop] fp32,
    O, cop).  cin: the channels the conv reads (a multiple of 32); cin_map: the physical input channel of each of the I logical channels."""
    nph, O, I = w.shape[:3]
    taps = w.shape[3] * w.shape[4] * w.shape[5]
    tile = cout_tile or (16 if O <= 16 else 32 if O <= 32 else 64 if O <= 64 else 128)
    cop = (O + tile - 1) // tile * tile
    idx = torch.as_tensor(list(range(I)) if cin_map is None else cin_map, dtype=torch.long, device=w.device)
    wt = torch.zeros(nph, taps, cop, cin, dtype=torch.float64, device=w.device)
    wt[:, :, :O].index_copy_(3, idx, w.permute(0, 3, 4, 5, 1, 2).reshape(nph, taps, O, I))
    if split:
        s = wt * 1024.0
        hi = s.half()
        packed = torch.cat([hi, (s - hi.double()).half()], dim=-1)
    else:
        packed = wt.half()
    bias = torch.zeros(cop, dtype=torch.float32, device=w.device)
    bias[:O] = b.float()
    return packed.contiguous(), bias, O, cop


def estimator_shape_error(mfe: torch.nn.Module) -> Optional[str]:
    """Why `mfe` is not the estimator the kernels restate (MotionFieldEstimator('standard', 34, K in {4, 9}), predict_multiref_occ), or None."""
    try:
        if not getattr(mfe, 'predict_multiref_occ', False):
            return 'predict_multiref_occ=False'
        down = [blk.layers[0].layers[0] for blk in mfe.down]
        up = [blk.layers[1].layers[0] for blk in mfe.up]
        c0 = down[0].in_channels
        if c0 % 5 or c0 // 5 - 1 not in (4, 9):
            return f'{c0} input channels (torso_kp_num 4 or 9 are built)'
        if [c.out_channels for c in down] != [64, 128, 256, 512, 1024] or [c.out_channels for c in up] != [512, 256, 128, 64, 32]:
            return "model_scale other than 'standard'"
        if mfe.compress.out_channels != 4 or mfe.tgt_head_fuser.in_channels != c0 + 64 or mfe.mask_conv.out_channels != c0 // 5:
            return 'unexpected estimator layers'
    except AttributeError as e:
        return f'not a MotionFieldEstimator ({e})'
    return None


class MotionWeights:
    """Folded and packed weights of the motion-field estimator for one sr_mode (split = tc_exact).  Every BatchNorm is eval-mode and folds
    into the conv before it (fold_cna); the tgt-head encoder's pre-activation ResBlock2D keeps BN1 as an affine + ReLU (r3dp_tw_affine_relu)."""

    def __init__(self, mfe: torch.nn.Module, split: bool):
        err = estimator_shape_error(mfe)
        if err is not None:
            raise NotImplementedError(f"torso_motion='cuda' is built for MotionFieldEstimator('standard'): {err}")
        self.split = bool(split)
        dev = next(mfe.parameters()).device
        d = lambda t: t.detach().double()                                               # noqa: E731
        c0 = mfe.down[0].layers[0].layers[0].in_channels
        self.K = c0 // 5 - 1
        self.c0, self.P0 = c0, (c0 + 31) // 32 * 32                        # input channels, padded to the 32-channel K step
        self.CF = self.P0 + 64                                             # fuser input: [input c0 | pad | up output 32 | head features 32]
        self.compress = (d(mfe.compress.weight)[:, :, 0, 0, 0], d(mfe.compress.bias))
        self.down = []
        cin = self.P0
        for blk in mfe.down:
            w, b = fold_cna(blk.layers[0])
            self.down.append(pack_conv3d(w[None], b, cin, split))
            cin = w.shape[0]
        self.up = []
        for blk in mfe.up:
            w, b = fold_cna(blk.layers[1])
            self.up.append(pack_conv3d(compose_nearest_up3d(w), b, cin, split))
            cin = w.shape[0]
        enc = mfe.tgt_head_encoder
        w, b = fold_cna(enc[0])
        self.enc0 = pack_conv3d(w[None, :, :, None], b, 32, split)
        self.res = []
        for rb in list(enc)[1:]:
            nac1, nac2 = rb.layers[0].layers, rb.layers[1].layers                   # NAC: BN, ReLU, conv
            s1, t1 = bn_affine(nac1[0])
            s2, t2 = bn_affine(nac2[0])
            w1, b1 = sn_weight(nac1[2]), d(nac1[2].bias)
            w2, b2 = sn_weight(nac2[2]), d(nac2[2].bias)
            self.res.append((s1.float().to(dev), t1.float().to(dev),
                             pack_conv3d((w1 * s2[:, None, None, None])[None, :, :, None], b1 * s2 + t2, 32, split),
                             pack_conv3d(w2[None, :, :, None], b2, 32, split)))
        fu = mfe.tgt_head_fuser
        fmap = list(range(c0)) + [self.P0 + i for i in range(64)]
        self.fuser = pack_conv3d(d(fu.weight)[None], d(fu.bias), self.CF, split, cin_map=fmap)
        mc = mfe.mask_conv
        self.mask = pack_conv3d(d(mc.weight)[None], d(mc.bias), 32, split)
        D = MOTION_D
        occ = [d(c.weight)[0].reshape(32, D, 7, 7).permute(1, 2, 3, 0) for c in (mfe.occlusion_conv, mfe.occlusion_conv2)]
        self.occ_w = torch.stack(occ, dim=-1).reshape(D, 49, 32, 2).float().contiguous().to(dev)
        self.occ_b = torch.cat([d(mfe.occlusion_conv.bias), d(mfe.occlusion_conv2.bias)]).float().contiguous().to(dev)


def compress_volume(wts: MotionWeights, motion_inp: torch.Tensor) -> torch.Tensor:
    """compress(motion_inp): the 1x1x1 conv 34 -> 4 in float64, as the NDHWC fp32 volume [N,D,H,W,4] the input kernel samples."""
    wc, bc = wts.compress
    x = torch.einsum('oi,nidhw->ndhwo', wc.to(motion_inp.device), motion_inp.double()) + bc.to(motion_inp.device)
    return x.float().contiguous()


def motion(wts: MotionWeights, fc: torch.Tensor, kp_s: torch.Tensor, kp_d: torch.Tensor, rgb_256: torch.Tensor, weights_256: torch.Tensor):
    """MotionFieldEstimator.forward with Rs = Rd = I -> (deformation [N,D,64,64,3], occlusion, occlusion_2 [N,1,64,64]) fp32.
    fc [N or 1,D,64,64,4] fp32: the compressed source volume (compress_volume; one volume for the batch is read by every image),
    kp_s / kp_d [N,K,3], rgb_256 [N,3,256,256], weights_256 [N,1,256,256]."""
    L, sp, st = capi.lib(), wts.split, capi.stream()
    wide = 2 if sp else 1
    N, K = kp_s.shape[:2]
    if K != wts.K:
        raise ValueError(f'{K} keypoints for an estimator built for {wts.K}')
    D, S = MOTION_D, MOTION_HW
    fc, kp_s, kp_d = capi.f32(fc), capi.f32(kp_s), capi.f32(kp_d)
    dev = kp_s.device
    f16 = torch.float16
    P0, CF = wts.P0, wts.CF

    def conv(x, xs, xlo, cin, packed, dims, taps, relu, y, ys, yc0, ylo, up=0, res=None, out_f32=0):
        wp, bias, O, cop = packed
        n, dd, h, w = dims
        capi.check(L.r3dp_mf_conv3d(capi.ptr(x, f16), xs, xlo, cin, capi.ptr(wp, f16), capi.ptr(bias), capi.ptr(res, f16), n, dd, h, w, *taps, up, O, cop,
                                    relu, capi.ptr(y, torch.float32 if out_f32 else f16), ys, yc0, ylo, out_f32, int(sp), st))

    with capi.region('torso_motion'):
        xf = torch.empty(N, D, S, S, CF * wide, device=dev, dtype=f16)                 # the fuser input; its first P0 channels feed the down path
        capi.check(L.r3dp_mf_input(capi.ptr(fc), int(fc.shape[0] == 1 and N > 1), capi.ptr(kp_s), capi.ptr(kp_d), N, K, D, S, S, P0,
                                   capi.ptr(xf, f16), CF * wide, CF, int(sp), st))
        x, xs, xlo, cin, hw = xf, CF * wide, CF, P0, S
        for packed in wts.down:
            O = packed[2]
            y = torch.empty(N, D, hw, hw, O * wide, device=dev, dtype=f16)
            conv(x, xs, xlo, cin, packed, (N, D, hw, hw), (3, 3, 3), 1, y, O * wide, 0, O)
            hw //= 2
            x = torch.empty(N, D, hw, hw, O * wide, device=dev, dtype=f16)
            capi.check(L.r3dp_mf_pool(capi.ptr(y, f16), N, D, hw, hw, O, O * wide, O, capi.ptr(x, f16), O * wide, O, int(sp), st))
            xs, xlo, cin = O * wide, O, O
        for i, packed in enumerate(wts.up):
            O = packed[2]
            if i + 1 < len(wts.up):
                y, ys, yc0, ylo = torch.empty(N, D, 2 * hw, 2 * hw, O * wide, device=dev, dtype=f16), O * wide, 0, O
            else:                                                                          # the last up block writes its slice of the fuser input
                y, ys, yc0, ylo = xf, CF * wide, P0, CF
            conv(x, xs, xlo, cin, packed, (N, D, hw, hw), (3, 2, 2), 1, y, ys, yc0, ylo, up=1)
            x, xs, xlo, cin, hw = y, O * wide, O, O, 2 * hw
        # tgt-head encoder at 128^2 (D = 1), then its 2x2 mean broadcast over depth into the fuser input
        if tuple(rgb_256.shape) != (N, 3, 4 * S, 4 * S) or tuple(weights_256.shape) != (N, 1, 4 * S, 4 * S):
            raise ValueError(f'rgb_256 / weights_256 must be [N,3|1,{4 * S},{4 * S}], got {tuple(rgb_256.shape)} / {tuple(weights_256.shape)}')
        H2 = 2 * S
        e = torch.empty(N, 1, H2, H2, 32 * wide, device=dev, dtype=f16)
        capi.check(L.r3dp_mf_head_input(capi.ptr(capi.f32(rgb_256)), capi.ptr(capi.f32(weights_256)), N, H2, H2, 32, capi.ptr(e, f16), 32 * wide, 32,
                                        int(sp), st))
        dims2 = (N, 1, H2, H2)
        x = torch.empty_like(e)
        conv(e, 32 * wide, 32, 32, wts.enc0, dims2, (1, 7, 7), 1, x, 32 * wide, 0, 32)
        for s1, t1, c1, c2 in wts.res:
            a = torch.empty_like(x)
            capi.check(L.r3dp_tw_affine_relu(capi.ptr(x, f16), capi.ptr(s1), capi.ptr(t1), N, H2, H2, 32, int(sp), capi.ptr(a, f16), st))
            t = torch.empty_like(x)
            conv(a, 32 * wide, 32, 32, c1, dims2, (1, 3, 3), 1, t, 32 * wide, 0, 32)
            xn = torch.empty_like(x)
            conv(t, 32 * wide, 32, 32, c2, dims2, (1, 3, 3), 0, xn, 32 * wide, 0, 32, res=x)
            x = xn
        capi.check(L.r3dp_mf_head_bcast(capi.ptr(x, f16), N, D, S, S, 32, 32 * wide, 32, capi.ptr(xf, f16), CF * wide, P0 + 32, CF, int(sp), st))
        # fuser (7^3, no activation), mask logits (fp32), softmax + deformation, the occlusion pair
        fx = torch.empty(N, D, S, S, 32 * wide, device=dev, dtype=f16)
        conv(xf, CF * wide, CF, CF, wts.fuser, (N, D, S, S), (7, 7, 7), 0, fx, 32 * wide, 0, 32)
        ls = (K + 2) // 2 * 2                                                           # K+1 logits per voxel, an even stride
        logits = torch.empty(N, D, S, S, ls, device=dev)
        conv(fx, 32 * wide, 32, 32, wts.mask, (N, D, S, S), (7, 7, 7), 0, logits, ls, 0, 0, out_f32=1)
        deformation = torch.empty(N, D, S, S, 3, device=dev)
        capi.check(L.r3dp_mf_deform(capi.ptr(logits), ls, capi.ptr(kp_s), capi.ptr(kp_d), N, K, D, S, S, capi.ptr(deformation), st))
        occ = torch.empty(N, 1, S, S, device=dev)
        occ2 = torch.empty(N, 1, S, S, device=dev)
        capi.check(L.r3dp_mf_occlusion(capi.ptr(fx, f16), N, D, S, S, 32, 32 * wide, 32, int(sp), capi.ptr(wts.occ_w), capi.ptr(wts.occ_b), capi.ptr(occ),
                                       capi.ptr(occ2), st))
    return deformation, occ, occ2


def hid_to_nchw(hid16: torch.Tensor, C: int, split: bool) -> torch.Tensor:
    """NHWC fp16 hid ([hi | lo] when split) -> [N,C,H,W] fp32."""
    N, H, W, cs = hid16.shape
    y = torch.empty(N, C, H, W, device=hid16.device)
    capi.check(capi.lib().r3dp_tw_hid_to_nchw(capi.ptr(hid16, torch.float16), N, C, H, W, cs, cs // 2 if split else 0, capi.ptr(y), capi.stream()))
    return y


# ---- stage 1 (model2.py:222-258) -----------------------------------------------------------------------------------------------------
def _hp(tm) -> dict:
    # The warper's own copy of the hparams (model2.py:202 deep-copies the global at construction).  The reference's forward reads
    # torso_inp_mode / torso_mask_dilate_ksize / mul_torso_mask from the module-level global at call time (model2.py:226-234); the two agree
    # unless that global is changed after the warper is built.
    return getattr(tm, 'hparams', {}) or {}


def dilate(m: torch.Tensor, ksize: int) -> torch.Tensor:
    """utils/commons/image_utils.py dilate: reflect pad + max-pool."""
    pad = (ksize - 1) // 2
    return F.max_pool2d(F.pad(m, [pad, pad, pad, pad], mode='reflect'), kernel_size=ksize, stride=1, padding=0)


@torch.no_grad()
def appearance(tm, torso_src_img: torch.Tensor, segmap: torch.Tensor, motion_wts: Optional['MotionWeights'] = None) -> Dict[str, torch.Tensor]:
    """What stage 1 derives from the reference torso image and the segmap alone (the per-clip part): the masked appearance volume
    [N,32,16,64,64], the 64^2 torso segmap, the dilated torso mask, the motion estimator's appearance input, and the volume in NDHWC.
    motion_wts: also 'fc', the estimator's compressed source volume [N,16,64,64,4] fp32 (compress_volume)."""
    hp = _hp(tm)
    src = torso_src_img
    if hp.get('torso_inp_mode', 'rgb') == 'rgb_alpha':
        seg = F.interpolate(segmap[:, [2, 4]].float(), size=(src.shape[-2], src.shape[-1]), mode='bilinear', align_corners=False, antialias=False)
        src = torch.cat([src, seg], dim=1)
    feats = tm.appearance_extractor(src)
    seg64 = F.interpolate(segmap[:, [2, 4]].float(), size=(64, 64), mode='bilinear', align_corners=False, antialias=False)
    mask = dilate(seg64.sum(dim=1).unsqueeze(1), hp.get('torso_mask_dilate_ksize', 7))
    if hp.get('mul_torso_mask', True):
        feats = feats * mask.unsqueeze(1)
    motion_inp = torch.cat([feats, seg64.unsqueeze(2).repeat([1, 1, feats.shape[2], 1, 1])], dim=1)
    out = {'feats': feats, 'seg64': seg64, 'mask': mask, 'motion_inp': motion_inp, 'fs_ndhwc': feats.permute(0, 2, 3, 4, 1).contiguous()}
    if motion_wts is not None:
        out['fc'] = compress_volume(motion_wts, motion_inp)
    return out


class TorsoWarper:
    """WarpBasedTorsoModelMediaPipe.forward (model2.py:222-287, eval) around the caller's module `tm`, stage 2 on the kernels.
    `app`: the output of appearance() for this clip (per-clip cache), or None to compute it per call.  `motion_wts`: run the
    motion_field_estimator on the kernels (motion()) instead of calling the caller's module."""

    def __init__(self, tm: torch.nn.Module):
        self.tm = tm
        self._eye = None

    @torch.no_grad()
    def __call__(self, wts: Stage2Weights, torso_src_img, segmap, kp_s, kp_d, tgt_head_img, tgt_head_weights, app: Optional[Dict] = None,
                 motion_wts: Optional[MotionWeights] = None):
        tm, hp = self.tm, _hp(self.tm)
        if app is None:
            app = appearance(tm, torso_src_img, segmap, motion_wts)
        elif motion_wts is not None and 'fc' not in app:
            # a clip begun before torso_motion='cuda' was set: its cached volume lacks the compressed source; add it to the cache once
            app['fc'] = compress_volume(motion_wts, app['motion_inp'])
        B = kp_s.shape[0]
        motion_inp = app['motion_inp']
        if motion_inp.shape[0] != B:
            motion_inp = motion_inp.expand(B, -1, -1, -1, -1)
        kp_num = hp.get('torso_kp_num', 4)
        if kp_num not in KP_IDX:
            raise NotImplementedError(f'torso_kp_num {kp_num}')
        kp_s, kp_d = kp_s[:, KP_IDX[kp_num], :], kp_d[:, KP_IDX[kp_num], :]
        if self._eye is None or self._eye.shape[0] != B or self._eye.device != kp_s.device:
            self._eye = torch.eye(3, 3, device=kp_s.device).unsqueeze(0).repeat([B, 1, 1])          # Rs = Rd = I, made once
        if motion_wts is not None:
            deformation, occlusion, occlusion_2 = motion(motion_wts, app['fc'], kp_s, kp_d, tgt_head_img, tgt_head_weights)
        else:
            deformation, occlusion, occlusion_2 = tm.motion_field_estimator(motion_inp, kp_s, kp_d, self._eye, self._eye, tgt_head_img, tgt_head_weights)
        # the reference's gradient-scaling blend (model2.py:251-257); kept so the values are the reference's bits
        deformation = deformation * 0.1 + deformation.detach() * 0.9
        occlusion = occlusion * 0.1 + occlusion.detach() * 0.9
        occlusion_2 = occlusion_2 * 0.1 + occlusion_2.detach() * 0.9
        ret = {'kp_src': kp_s, 'kp_drv': kp_d, 'occlusion': occlusion, 'occlusion_2': occlusion_2}
        rgb, hid16, occ2 = stage2(wts, app['fs_ndhwc'], deformation, occlusion_2)
        ret['deformed_torso_hid'] = hid_to_nchw(hid16, wts.up[-1][1], wts.split)
        ret['occlusion_2'] = occ2
        return rgb, ret
