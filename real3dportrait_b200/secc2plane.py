"""SegFormerSECC2PlaneBackbone (modules/real3d/segformer.py:673-733) on libr3dp_b200: the per-frame SECC -> tri-plane network that
`cal_secc_plane` runs before the render (modules/real3d/secc_img2plane.py:64-81).

The module keeps the reference's constructor and state_dict (keys and shapes) and is a drop-in for it; the parameters are plain
containers and every forward runs the r3dp_sp_* kernels, r3dp_mf_conv3d (token GEMMs, last conv) and r3dp_sr_tc_conv (to_plane_cnn.0/2/4).
Weights are folded on the host in float64 and packed once per parameter set (refolded after load_state_dict / .to()):
  - prenet (StyleGAN2 Conv2dLayer, 1x1, weight gain 1/sqrt(cin), linear) splits into the per-clip part on (cano, src) and the per-frame tgt part;
  - eval BatchNorm of fuse_head.linear_fuse goes into its weights;
  - head fold: bilinear resize (align_corners=False) is a convex combination per output pixel, so it commutes with channel mixing and passes
    constants through; ReLU(BN(W_fuse cat[R(L4 c4), R(L3 c3), R(L2 c2), L1 c1])) = ReLU(sum_i R_i(G_i c_i) + b) with G_i = diag(s) W_fuse,i L_i.
Precision (`tc`): fp16 GEMM operands with fp32 accumulation; residual stream, LayerNorm, softmax and GELU in fp32.  `tc_exact`: the same
launch sequence with every GEMM / conv operand split into two fp16 halves ([hi | lo], weights as w * 2^10; three MMAs, fp32 accumulation)
and every activation the `tc` path passes between launches as fp16 passed as fp32 (the GEMM outputs the attention and the DWConv read) or as
split rows (the r3dp_sp_*_split entry points, r3dp_hb_layernorm, r3dp_sr_tcx_conv).
"""
from __future__ import annotations

import math
from typing import Optional

import torch
import torch.nn as nn

from . import _capi as capi, conv3d, sr_tc
from .conv3d import pack_gemm as _pack_gemm, pack_taps as _pack_taps
from .prepared import PreparedMixin
from .renderer import PlanesCL, producer_view

F16 = torch.float16
EMBED = [32, 64, 160, 256]          # mit_b0 (segformer.py:383-388)
HEADS = [1, 2, 5, 8]
SR = [8, 4, 2, 1]
DEPTH = 2
HEAD_DIM = 32
EMB = 256                           # SegFormerHead embedding_dim


# ---- parameter containers with the reference's names (segformer.py:60-420,471-498,673-704) --------------------------------------------
class _Prenet(nn.Module):
    def __init__(self, cin):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(3, cin, 1, 1))
        self.bias = nn.Parameter(torch.zeros(3))
        f = torch.tensor([1., 3., 3., 1.])
        f = torch.outer(f, f)
        self.register_buffer('resample_filter', f / f.sum())     # upfirdn2d.setup_filter([1,3,3,1]); unused by a 1x1 layer


class _PatchEmbed(nn.Module):
    def __init__(self, k, stride, cin, c):
        super().__init__()
        self.proj = nn.Conv2d(cin, c, k, stride, k // 2)
        self.norm = nn.LayerNorm(c)                               # eps 1e-5 (segformer.py:216)


class _Attention(nn.Module):
    def __init__(self, c, sr):
        super().__init__()
        self.q = nn.Linear(c, c)
        self.kv = nn.Linear(c, 2 * c)
        self.proj = nn.Linear(c, c)
        if sr > 1:
            self.sr = nn.Conv2d(c, c, sr, sr)
            self.norm = nn.LayerNorm(c)                           # eps 1e-5 (segformer.py:118)


class _DW(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.dwconv = nn.Conv2d(c, c, 3, 1, 1, groups=c)


class _Mlp(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.fc1 = nn.Linear(c, 4 * c)
        self.dwconv = _DW(4 * c)
        self.fc2 = nn.Linear(4 * c, c)


class _Block(nn.Module):
    def __init__(self, c, sr):
        super().__init__()
        self.norm1 = nn.LayerNorm(c, eps=1e-6)
        self.attn = _Attention(c, sr)
        self.norm2 = nn.LayerNorm(c, eps=1e-6)
        self.mlp = _Mlp(c)


class _MiTb0(nn.Module):
    def __init__(self):
        super().__init__()
        cins = [3] + EMBED[:3]
        for s in range(4):
            setattr(self, f'patch_embed{s + 1}', _PatchEmbed(7 if s == 0 else 3, 4 if s == 0 else 2, cins[s], EMBED[s]))
            setattr(self, f'block{s + 1}', nn.ModuleList([_Block(EMBED[s], SR[s]) for _ in range(DEPTH)]))
            setattr(self, f'norm{s + 1}', nn.LayerNorm(EMBED[s], eps=1e-6))


class _HeadMLP(nn.Module):
    def __init__(self, cin):
        super().__init__()
        self.proj = nn.Linear(cin, EMB)


class _ConvModule(nn.Module):
    """mmcv ConvModule(1x1, norm_cfg BN): conv (bias=False, mmcv's bias='auto' with a norm) -> bn -> ReLU."""
    def __init__(self):
        super().__init__()
        self.conv = nn.Conv2d(4 * EMB, EMB, 1, bias=False)
        self.bn = nn.BatchNorm2d(EMB)


class _SegFormerHead(nn.Module):
    def __init__(self):
        super().__init__()
        for i, c in enumerate(EMBED):
            setattr(self, f'linear_c{i + 1}', _HeadMLP(c))
        self.linear_fuse = _ConvModule()


# ---- host-side folding (float64) --------------------------------------------------------------------------------------------------------
def fold_prenet(weight: torch.Tensor, bias: torch.Tensor):
    """Conv2dLayer(cin, 3, 1), linear: y = (W / sqrt(cin)) x + b  ->  (W' [3,cin] float64, b float64)."""
    cin = weight.shape[1]
    return weight.detach().double()[:, :, 0, 0] / math.sqrt(cin), bias.detach().double()


def fold_bn(conv_w, bn: nn.BatchNorm2d):
    """1x1 conv (no bias) -> eval BatchNorm  ->  (W [O,I] float64 scaled by s, shift [O] float64)."""
    s = bn.weight.detach().double() / torch.sqrt(bn.running_var.detach().double() + bn.eps)
    shift = bn.bias.detach().double() - bn.running_mean.detach().double() * s
    return s[:, None] * conv_w.detach().double()[:, :, 0, 0], shift


def fold_head(head: _SegFormerHead):
    """-> ([G_1..G_4] float64 [256, C_i], bias float64 [256]) with ReLU(sum_i R_i(G_i c_i) + bias) = linear_fuse(cat[R(_c4),R(_c3),R(_c2),_c1])."""
    wf, shift = fold_bn(head.linear_fuse.conv.weight, head.linear_fuse.bn)
    G, bias = [], shift.clone()
    for i in range(4):
        lin = getattr(head, f'linear_c{i + 1}').proj
        blk = wf[:, (3 - i) * EMB:(4 - i) * EMB]                 # cat order [_c4, _c3, _c2, _c1] (segformer.py:536)
        G.append(blk @ lin.weight.detach().double())
        bias = bias + blk @ lin.bias.detach().double()
    return G, bias


def _conv_rows(w: torch.Tensor) -> torch.Tensor:
    """Conv weights [O, I, k, k] -> GEMM [O, k*k*I], column (ky*k + kx)*I + c (the r3dp_sp_patches order)."""
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1)


def plane_index_map(H: int, W: int):
    """Where the reference's flips (segformer.py:722-730) take conv output (channel co, row y, col x): (plane co // 32, channel co % 32,
    row H-1-y, col x for planes 0 and 1, W-1-x for plane 2).  Returned as a function of (co, y, x)."""
    def where(co, y, x):
        p = co // 32
        return p, co % 32, H - 1 - y, (W - 1 - x) if p == 2 else x
    return where


def fold_and_pack(m: 'SegFormerSECC2PlaneBackbone', dev, split: bool) -> dict:
    """Every float64 fold of m's parameters and every r3dp_mf_conv3d weight pack, on dev (any device: nothing here launches a kernel).
    split: the packs hold [hi | lo] of w * 2^10 (precision='tc_exact'); the fp32 tensors (prenet, patch embed 1, LayerNorms, DWConv, head
    bias) are the same in both precisions.  The to_plane_cnn.0/2/4 packs of r3dp_sr_tc_conv are made by the module (they need CUDA)."""
    f32 = lambda t: t.detach().to(dev, torch.float32).contiguous()      # noqa: E731
    d = lambda t: t.detach().double()                                   # noqa: E731
    gemm = lambda w, b: _pack_gemm(w, b, dev, split)                    # noqa: E731
    P = {}
    wpre, bpre = fold_prenet(m.prenet.weight, m.prenet.bias)
    nconst = wpre.shape[1] - 3
    P['wpre'], P['bpre'] = f32(wpre), f32(bpre)
    P['wpre_const'], P['wpre_tgt'] = f32(wpre[:, :nconst]), f32(wpre[:, nconst:])
    mv = m.mix_vit
    P['pe1'] = (f32(mv.patch_embed1.proj.weight), f32(mv.patch_embed1.proj.bias))
    ln = lambda n: (f32(n.weight), f32(n.bias), float(n.eps))          # noqa: E731
    stages = []
    for s in range(4):
        pe = getattr(mv, f'patch_embed{s + 1}')
        st = {'pe_norm': ln(pe.norm), 'norm': ln(getattr(mv, f'norm{s + 1}'))}
        if s > 0:
            st['pe'] = gemm(_conv_rows(d(pe.proj.weight)), d(pe.proj.bias))
        blocks = []
        for blk in getattr(mv, f'block{s + 1}'):
            at = blk.attn
            b = {'norm1': ln(blk.norm1), 'norm2': ln(blk.norm2),
                 'q': gemm(d(at.q.weight), d(at.q.bias)), 'kv': gemm(d(at.kv.weight), d(at.kv.bias)),
                 'proj': gemm(d(at.proj.weight), d(at.proj.bias)),
                 'fc1': gemm(d(blk.mlp.fc1.weight), d(blk.mlp.fc1.bias)),
                 'fc2': gemm(d(blk.mlp.fc2.weight), d(blk.mlp.fc2.bias)),
                 'dw': (f32(blk.mlp.dwconv.dwconv.weight.reshape(-1, 9)), f32(blk.mlp.dwconv.dwconv.bias))}
            if SR[s] > 1:
                b['sr'] = gemm(_conv_rows(d(at.sr.weight)), d(at.sr.bias))
                b['sr_norm'] = ln(at.norm)
            blocks.append(b)
        st['blocks'] = blocks
        stages.append(st)
    P['stages'] = stages
    G, hb = fold_head(m.fuse_head)
    P['G'] = [gemm(g, None) for g in G]
    P['head_bias'] = f32(hb)
    P['convs'] = [{'mf': _pack_taps(d(c.weight), d(c.bias), dev, split)} for c in (m.to_plane_cnn[i] for i in (0, 2, 4))]
    last = m.to_plane_cnn[7]
    w7, b7 = d(last.weight), d(last.bias)
    P['last_r'] = _pack_taps(w7[:64].flip(2), b7[:64], dev, split)          # planes 0, 1: rows mirrored
    P['last_rc'] = _pack_taps(w7[64:].flip(2, 3), b7[64:], dev, split)      # plane 2: rows and columns mirrored
    return P


class SegFormerSECC2PlaneBackbone(PreparedMixin, nn.Module):
    """SegFormerSECC2PlaneBackbone(mode='b0', out_channels=96, pncc_cond_mode='cano_src_tgt') (segformer.py:673-733) on sm_90a kernels.

    forward(x [B, 9|6, H, W]) -> [B, 3, 32, H/2, W/2] (the reference's flipped planes), a view of channels-last data;
    begin_clip(cond_cano, cond_src) then planes_cl(cond_tgt) -> PlanesCL('hwpc') [B, H/2, W/2, 3, 32]: the per-clip prenet part folded into
    one cached image, and the planes written by the last conv's epilogue in the render's zero-copy layout.

    precision: 'tc' (fp16 GEMM / conv operands, fp32 accumulation) or 'tc_exact' (fp32-grade: every GEMM and conv operand split into two
    fp16 halves, three MMAs per product; every activation passed between launches as fp32 or split fp16).  The parameters and state_dict
    are the same in both."""

    def __init__(self, mode='b0', out_channels=96, pncc_cond_mode='cano_src_tgt', *, precision='tc'):
        super().__init__()
        if mode != 'b0':
            raise NotImplementedError(f'SegFormerSECC2PlaneBackbone: only MiT-b0 is built (got mode={mode!r})')
        if out_channels != 96:
            raise NotImplementedError(f'SegFormerSECC2PlaneBackbone: only out_channels=96 (tri-planes of 32 channels) is built, got {out_channels}')
        if pncc_cond_mode not in ('cano_src_tgt', 'cano_tgt'):
            raise NotImplementedError(f'pncc_cond_mode={pncc_cond_mode!r}')
        if precision not in ('tc', 'tc_exact'):
            raise ValueError(f"SegFormerSECC2PlaneBackbone: precision must be 'tc' or 'tc_exact', got {precision!r}")
        self.mode, self.pncc_cond_mode, self.precision = mode, pncc_cond_mode, precision
        in_dim = 9 if pncc_cond_mode == 'cano_src_tgt' else 6
        self.prenet = _Prenet(in_dim)
        self.mix_vit = _MiTb0()
        self.fuse_head = _SegFormerHead()
        self.to_plane_cnn = nn.Sequential(
            nn.Conv2d(256, 256, 3, 1, 1), nn.LeakyReLU(0.01, inplace=True),
            nn.Conv2d(256, 256, 3, 1, 1), nn.LeakyReLU(0.01, inplace=True),
            nn.Conv2d(256, 256, 3, 1, 1), nn.LeakyReLU(0.01, inplace=True),
            nn.UpsamplingBilinear2d(scale_factor=2.),
            nn.Conv2d(256, out_channels, 3, 1, 1))

    def _prepared(self):
        return self.prepared('weights', self._build)

    def _build(self):
        split = self.precision == 'tc_exact'
        P = fold_and_pack(self, capi.cuda_device(self.prenet.weight), split)
        for cv, c in zip(P['convs'], (self.to_plane_cnn[i] for i in (0, 2, 4))):
            cv['tc'] = sr_tc.pack_plain(c, EMB, split=split)            # r3dp_sr_tc_conv / r3dp_sr_tcx_conv (act 2) where W % 128 == 0
        return P

    # ---- input checks ------------------------------------------------------------------------------------------------------------------
    @staticmethod
    def _check_image(x: torch.Tensor, ch: int, what: str) -> torch.Tensor:
        if x.ndim != 4 or x.shape[1] != ch:
            raise ValueError(f'{what}: expected [B,{ch},H,W], got {tuple(x.shape)}')
        H, W = x.shape[2:]
        if H != W or H % 32 or H > 512 or H < 32:
            raise ValueError(f'{what}: H == W, a multiple of 32 in [32, 512] (every attention sees at most 256 keys); got {H}x{W}')
        if not x.is_cuda:
            raise RuntimeError('real3dportrait_b200 runs on CUDA tensors only (no CPU fallback); got a CPU tensor')
        return capi.f32(x)

    # ---- public interface --------------------------------------------------------------------------------------------------------------
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """x [B, 9|6, H, W] = cat[cano, (src,) tgt] -> planes [B, 3, 32, H/2, W/2] (segformer.py:705-733)."""
        x = self._check_image(x, self.prenet.weight.shape[1], 'SegFormerSECC2PlaneBackbone.forward')
        P = self._prepared()
        out = self._run(x, P['wpre'], None, P['bpre'])
        return out.permute(0, 3, 4, 1, 2)                         # [B,H,W,3,C] -> [B,3,C,H,W] view (channels-last producer layout)

    def begin_clip(self, cond_cano: torch.Tensor, cond_src: Optional[torch.Tensor] = None) -> None:
        """Fold the prenet's per-clip inputs (cano, and src in 'cano_src_tgt') into one cached image [1,3,H,W]."""
        parts = [cond_cano] + ([cond_src] if self.pncc_cond_mode == 'cano_src_tgt' else [])
        if any(p is None for p in parts):
            raise ValueError('begin_clip: cond_src is required with pncc_cond_mode=cano_src_tgt')
        parts = [self._check_image(p, 3, 'begin_clip') for p in parts]
        if any(p.shape[0] != 1 or p.shape != parts[0].shape for p in parts):
            raise ValueError('begin_clip: one [1,3,H,W] image per condition')
        P = self._prepared()
        xc = torch.cat(parts, 1).contiguous() if len(parts) > 1 else parts[0]
        _, cin, H, W = xc.shape
        base = self.cached('clip')
        if base is None or base.shape[2:] != (H, W) or base.device != xc.device:
            base = self.store('clip', torch.empty(1, 3, H, W, device=xc.device))
        # a later clip of the same size refills the same image in place: CUDA graphs captured over planes_cl() read its address
        capi.check(capi.lib().r3dp_sp_prenet(capi.ptr(xc), 1, cin, H, W, capi.ptr(P['wpre_const']), capi.ptr(P['bpre']), capi.ptr(base),
                                             capi.stream()))

    def planes_cl(self, cond_tgt: torch.Tensor, out: Optional[torch.Tensor] = None) -> PlanesCL:
        """cond_tgt [B,3,H,W] (after begin_clip) -> PlanesCL('hwpc') [B,H/2,W/2,3,32] fp32, the same values as forward(cat[cano, src, tgt])."""
        base = self.cached('clip')
        if base is None:
            raise RuntimeError('planes_cl: call begin_clip(cond_cano, cond_src) first')
        x = self._check_image(cond_tgt, 3, 'planes_cl')
        if x.shape[2:] != base.shape[2:]:
            raise ValueError('planes_cl: cond_tgt must have the size of the clip images')
        P = self._prepared()
        return PlanesCL(self._run(x, P['wpre_tgt'], base, None, out), 'hwpc')

    # ---- the launch sequence -----------------------------------------------------------------------------------------------------------
    def _run(self, x, wpre, base, bpre, out=None):
        P, L, st, dev = self._prepared(), capi.lib(), capi.stream(), x.device
        B, cin, H, W = x.shape
        ptr = capi.ptr
        ex = self.precision == 'tc_exact'
        wide = 2 if ex else 1               # halves per channel of an activation passed as fp16: 2 = split rows [hi C | lo C]

        def act(*shape):
            """An activation the tc path passes as fp16; split rows (twice as wide) in tc_exact."""
            return torch.empty(*shape[:-1], wide * shape[-1], device=dev, dtype=F16)

        def gemm(a, R, pk, out_f32):
            """Token GEMM on r3dp_mf_conv3d.  tc_exact: split operands, and every output fp32 (the attention and the DWConv read q, kv, fc1
            at fp32 grade)."""
            K = pk.w.shape[1] // wide
            y = torch.empty(R, pk.cout, device=dev, dtype=torch.float32 if out_f32 or ex else F16)
            conv3d.launch(pk, a, wide * K, K if ex else 0, K, (1, 1, 1, R), (1, 1, 1), y, pk.cout, stream=st)
            return y

        def layernorm(xv, t, R, C, p, xo=None, yf=None, yh=None):
            g, b, eps = p
            if not ex or yh is None:
                capi.check(L.r3dp_sp_layernorm(ptr(xv), ptr(t), R, C, ptr(g), ptr(b), eps, ptr(xo), ptr(yf), ptr(yh, F16), C, st))
            elif t is None:
                assert xo is None and yf is None
                capi.check(L.r3dp_hb_layernorm(ptr(xv), R, C, ptr(g), ptr(b), eps, 0, None, 0, ptr(yh, F16), 2 * C, C, st))
            else:
                assert yf is None
                capi.check(L.r3dp_sp_layernorm_split(ptr(xv), ptr(t), R, C, ptr(g), ptr(b), eps, ptr(xo), ptr(yh, F16), 2 * C, C, st))

        def patches(a, h, C, k, s, p):
            ho = (h + 2 * p - k) // s + 1
            y = act(B * ho * ho, k * k * C)
            capi.check((L.r3dp_sp_patches_split if ex else L.r3dp_sp_patches)(ptr(a, F16), B, h, h, C, k, s, p, ptr(y, F16), st))
            return y, ho

        with capi.region('secc2plane'):
            h = H // 4
            t0 = torch.empty(B * h * h, EMBED[0], device=dev)
            capi.check(L.r3dp_sp_embed(ptr(x), B, cin, H, W, ptr(wpre), ptr(base), ptr(bpre), ptr(P['pe1'][0]), ptr(P['pe1'][1]), ptr(t0), st))
            feats, prev = [], None
            for s in range(4):
                C, S = EMBED[s], P['stages'][s]
                if s > 0:
                    pt, h = patches(prev, h, EMBED[s - 1], 3, 2, 1)
                    t0 = gemm(pt, B * h * h, S['pe'], True)
                R = B * h * h
                xres = torch.empty(R, C, device=dev)
                layernorm(t0, None, R, C, S['pe_norm'], yf=xres)
                a = act(R, C)
                layernorm(xres, None, R, C, S['blocks'][0]['norm1'], yh=a)
                for bi, bw in enumerate(S['blocks']):
                    q = gemm(a, R, bw['q'], False)
                    if SR[s] > 1:
                        pt, hk = patches(a, h, C, SR[s], SR[s], 0)
                        r = gemm(pt, B * hk * hk, bw['sr'], True)
                        a2 = act(B * hk * hk, C)
                        layernorm(r, None, B * hk * hk, C, bw['sr_norm'], yh=a2)
                        kv, tk = gemm(a2, B * hk * hk, bw['kv'], False), hk * hk
                    else:
                        kv, tk = gemm(a, R, bw['kv'], False), h * h
                    o = act(R, C)
                    if ex:
                        capi.check(L.r3dp_sp_attention_split(ptr(q), C, ptr(kv), 2 * C, B, h * h, tk, HEADS[s], HEAD_DIM ** -0.5, ptr(o, F16), 2 * C,
                                                             C, st))
                    else:
                        capi.check(L.r3dp_sp_attention(ptr(q, F16), C, ptr(kv, F16), 2 * C, B, h * h, tk, HEADS[s], HEAD_DIM ** -0.5, ptr(o, F16), C,
                                                       st))
                    t = gemm(o, R, bw['proj'], True)
                    layernorm(xres, t, R, C, bw['norm2'], xo=xres, yh=a)
                    f1 = gemm(a, R, bw['fc1'], False)
                    f2 = act(R, 4 * C)
                    if ex:
                        capi.check(L.r3dp_sp_dwconv_gelu_split(ptr(f1), B, h, h, 4 * C, ptr(bw['dw'][0]), ptr(bw['dw'][1]), ptr(f2, F16), st))
                    else:
                        capi.check(L.r3dp_sp_dwconv_gelu(ptr(f1, F16), B, h, h, 4 * C, ptr(bw['dw'][0]), ptr(bw['dw'][1]), ptr(f2, F16), st))
                    t = gemm(f2, R, bw['fc2'], True)
                    if bi + 1 < len(S['blocks']):
                        layernorm(xres, t, R, C, S['blocks'][bi + 1]['norm1'], xo=xres, yh=a)
                    else:
                        prev = act(R, C)
                        layernorm(xres, t, R, C, S['norm'], yh=prev)
                feats.append((prev, h))
            g = [(gemm(c, B * hh * hh, P['G'][i], True), hh) for i, (c, hh) in enumerate(feats)]
            h1 = feats[0][1]
            y = act(B, h1, h1, EMB)
            capi.check((L.r3dp_sp_head_fuse_split if ex else L.r3dp_sp_head_fuse)(ptr(g[0][0]), g[0][1], ptr(g[1][0]), g[1][1], ptr(g[2][0]), g[2][1],
                                                                                ptr(g[3][0]), g[3][1], B, ptr(P['head_bias']), ptr(y, F16), st))
            for ci, cv in enumerate(P['convs']):
                with capi.region(f'secc2plane.conv{2 * ci}'):         # per-launch times of the conv stack (tools/bench_secc.py)
                    if h1 % 128 == 0:          # r3dp_sr_tc_conv tiles 128-pixel rows
                        z = sr_tc.conv_plain(y, cv['tc'], 2, split=ex)
                    elif ex:
                        z = torch.empty_like(y)
                        conv3d.launch(cv['mf'], y, 2 * EMB, EMB, EMB, (B, 1, h1, h1), (1, 3, 3), z, 2 * EMB, 0, EMB, stream=st)
                        capi.check(L.r3dp_sp_leaky_split(ptr(z, F16), B * h1 * h1, EMB, 0.01, st))
                    else:
                        z = torch.empty_like(y)
                        conv3d.launch(cv['mf'], y, EMB, 0, EMB, (B, 1, h1, h1), (1, 3, 3), z, EMB, stream=st)
                        capi.check(L.r3dp_sp_leaky(ptr(z, F16), z.numel(), 0.01, st))
                y = z
            H2 = 2 * h1
            ur = act(B, H2, H2, EMB)
            urc = torch.empty_like(ur)
            with capi.region('secc2plane.upsample'):
                capi.check((L.r3dp_sp_upsample2_flip_split if ex else L.r3dp_sp_upsample2_flip)(ptr(y, F16), B, h1, h1, EMB, ptr(ur, F16), ptr(urc, F16),
                                                                                              st))
            if out is None:
                out = torch.empty(B, H2, H2, 3, 32, device=dev)
            elif tuple(out.shape) != (B, H2, H2, 3, 32) or out.dtype != torch.float32 or not out.is_contiguous():
                raise ValueError(f'planes_cl: out must be a contiguous fp32 [{B},{H2},{H2},3,32] tensor')
            with capi.region('secc2plane.conv7'):
                for src, pk, c0 in ((ur, P['last_r'], 0), (urc, P['last_rc'], 64)):
                    conv3d.launch(pk, src, wide * EMB, EMB if ex else 0, EMB, (B, 1, H2, H2), (1, 3, 3), out, 96, c0, stream=st)
        return out


def canonical_planes_cl(cano_planes: torch.Tensor) -> PlanesCL:
    """Canonical planes [1,3,32,H,W] (reference layout) -> PlanesCL('hwpc') with frame stride 0, the partner of planes_cl() in the render's
    (cano, secc) pair: the pair is sampled set by set and summed in-kernel.  Done once per clip."""
    t = cano_planes.detach()
    if not t.is_cuda:
        raise RuntimeError('real3dportrait_b200 runs on CUDA tensors only (no CPU fallback); got a CPU tensor')
    if t.ndim != 5 or t.shape[1] != 3 or t.shape[0] != 1:
        raise ValueError(f'canonical planes: expected [1,3,C,H,W], got {tuple(t.shape)}')
    N, _, Cc, H, W = t.shape
    cl = torch.empty(N, H, W, 3, Cc, device=t.device)
    cl.copy_(t.float().permute(0, 3, 4, 1, 2))
    return producer_view(cl.permute(0, 3, 4, 1, 2))
