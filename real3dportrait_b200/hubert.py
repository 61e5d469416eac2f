"""HuBERT audio features (data_gen/utils/process_audio/extract_hubert.py, transformers' HubertModel) on libr3dp_b200.

`HubertModel(config)` is a drop-in for transformers.HubertModel in eval, for the hubert-large-ls960-ft architecture: a layer-norm conv feature
extractor (kernels 10,3,3,3,3,2,2, strides 5,2,2,2,2,2,2), a feature projection and a stable-layer-norm (pre-LN) encoder with a grouped,
weight-normed positional conv.  Its state_dict keys and shapes are transformers' own.  `get_hubert_from_16k_speech` keeps the reference
function's semantics (T = (L - 80) // 320 rows, each 1000-frame segment encoded on its own) and writes the features straight into a caller's
buffer, e.g. the audio2secc VAE's batch['audio'][0].

Precision: every GEMM and attention operand is split fp16 ([hi | lo], three MMAs, fp32 accumulation).  The split operands are LayerNorm,
GELU and attention outputs, plus the projection output that feeds the positional conv; the residual stream stays fp32.  Host folds (float64,
cached until load_state_dict / .to()): the positional conv's weight norm (dim 2: one norm per kernel tap), the LayerNorm gamma / beta that feed
a GEMM, q / k / v as one [3H, H] GEMM with the 1/8 attention scale in q, weights packed as [hi | lo] of w * 2^10."""
from __future__ import annotations

import ctypes
import json
import os
from types import SimpleNamespace
from typing import Optional

import numpy as np
import torch
import torch.nn as nn

from . import _capi as capi
from .prepared import PreparedMixin

F16 = torch.float16
SEG = 1000                    # frames per encoder segment (extract_hubert.py: clip_length = 320 * 1000)
GROUP = 4                     # segments per launch group: bounds the conv stack's buffers independently of the clip length
KERNELS, STRIDES = (10, 3, 3, 3, 3, 2, 2), (5, 2, 2, 2, 2, 2, 2)
_DEFAULTS = dict(hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072, hidden_act='gelu',
                 layer_norm_eps=1e-5, feat_extract_norm='group', feat_extract_activation='gelu', conv_dim=(512,) * 7, conv_stride=STRIDES,
                 conv_kernel=KERNELS, conv_bias=False, num_conv_pos_embeddings=128, num_conv_pos_embedding_groups=16, conv_pos_batch_norm=False,
                 do_stable_layer_norm=False, feat_proj_layer_norm=True, mask_time_prob=0.05, mask_feature_prob=0.0)


def hubert_frames(L: int) -> int:
    """Rows get_hubert_from_16k_speech returns for L samples: (L - 80) // 320 (L >= 400)."""
    if L < 400:
        raise ValueError(f'hubert_frames: a clip needs at least 400 samples (one frame), got {L}')
    return (L - 80) // 320


def _segments(T: int):
    return [min(SEG, T - s) for s in range(0, T, SEG)]


def _config(config) -> SimpleNamespace:
    get = config.get if isinstance(config, dict) else (lambda k, v: getattr(config, k, v))
    c = {k: get(k, v) for k, v in _DEFAULTS.items()}
    for k in ('conv_dim', 'conv_stride', 'conv_kernel'):
        c[k] = tuple(c[k])
    return SimpleNamespace(**c)


def _check_config(c: SimpleNamespace):
    def no(msg):
        raise NotImplementedError(f'HubertModel: {msg} is not built (only the hubert-large-ls960-ft architecture is)')
    if c.feat_extract_norm != 'layer':
        no(f"feat_extract_norm={c.feat_extract_norm!r} (group norm, hubert-base)")
    if not c.do_stable_layer_norm:
        no('do_stable_layer_norm=False (the post-LN encoder)')
    if c.feat_extract_activation != 'gelu' or c.hidden_act != 'gelu':
        no(f'activations {c.feat_extract_activation!r} / {c.hidden_act!r} (gelu only)')
    if c.conv_pos_batch_norm:
        no('conv_pos_batch_norm=True')
    if c.conv_kernel != KERNELS or c.conv_stride != STRIDES:
        no(f'conv kernels {c.conv_kernel} / strides {c.conv_stride}')
    C = c.conv_dim[0]
    if any(d != C for d in c.conv_dim) or C % 32 or C > 512:
        no(f'conv_dim {c.conv_dim} (all equal, a multiple of 32, at most 512)')
    H = c.hidden_size
    if H % 64 or H > 1024 or H != 64 * c.num_attention_heads:
        no(f'hidden_size {H} with {c.num_attention_heads} heads (head_dim 64, hidden at most 1024)')
    if c.num_conv_pos_embeddings != 128 or H != 64 * c.num_conv_pos_embedding_groups:
        no(f'positional conv k{c.num_conv_pos_embeddings} in {c.num_conv_pos_embedding_groups} groups (k128, 64 channels per group)')
    if c.intermediate_size % 64:
        no(f'intermediate_size {c.intermediate_size} (a multiple of 64)')


# ---- parameter containers with transformers' names ------------------------------------------------------------------------------------
class _ConvLayer(nn.Module):
    def __init__(self, cin, cout, k, s, bias):
        super().__init__()
        self.conv = nn.Conv1d(cin, cout, k, stride=s, bias=bias)
        self.layer_norm = nn.LayerNorm(cout, elementwise_affine=True)


class _FeatureExtractor(nn.Module):
    def __init__(self, c):
        super().__init__()
        dims = (1,) + c.conv_dim
        self.conv_layers = nn.ModuleList([_ConvLayer(dims[i], dims[i + 1], c.conv_kernel[i], c.conv_stride[i], c.conv_bias) for i in range(7)])


class _FeatureProjection(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.feat_proj_layer_norm = c.feat_proj_layer_norm
        if c.feat_proj_layer_norm:
            self.layer_norm = nn.LayerNorm(c.conv_dim[-1], eps=c.layer_norm_eps)
        self.projection = nn.Linear(c.conv_dim[-1], c.hidden_size)


class _PosConv(nn.Module):
    def __init__(self, c):
        super().__init__()
        conv = nn.Conv1d(c.hidden_size, c.hidden_size, c.num_conv_pos_embeddings, padding=c.num_conv_pos_embeddings // 2,
                         groups=c.num_conv_pos_embedding_groups)
        self.conv = nn.utils.parametrizations.weight_norm(conv, name='weight', dim=2)
        self._register_load_state_dict_pre_hook(self._old_weight_norm)

    @staticmethod
    def _old_weight_norm(state_dict, prefix, *args):
        # checkpoints saved with torch.nn.utils.weight_norm store weight_g / weight_v
        for old, new in (('weight_g', 'original0'), ('weight_v', 'original1')):
            k = prefix + 'conv.' + old
            if k in state_dict:
                state_dict[prefix + 'conv.parametrizations.weight.' + new] = state_dict.pop(k)


class _Attention(nn.Module):
    def __init__(self, H):
        super().__init__()
        self.k_proj, self.v_proj, self.q_proj, self.out_proj = (nn.Linear(H, H) for _ in range(4))


class _FeedForward(nn.Module):
    def __init__(self, H, I):
        super().__init__()
        self.intermediate_dense = nn.Linear(H, I)
        self.output_dense = nn.Linear(I, H)


class _Layer(nn.Module):
    def __init__(self, c):
        super().__init__()
        H = c.hidden_size
        self.attention = _Attention(H)
        self.layer_norm = nn.LayerNorm(H, eps=c.layer_norm_eps)
        self.feed_forward = _FeedForward(H, c.intermediate_size)
        self.final_layer_norm = nn.LayerNorm(H, eps=c.layer_norm_eps)


class _Encoder(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.pos_conv_embed = _PosConv(c)
        self.layer_norm = nn.LayerNorm(c.hidden_size, eps=c.layer_norm_eps)
        self.layers = nn.ModuleList([_Layer(c) for _ in range(c.num_hidden_layers)])


# ---- host folds (float64) -------------------------------------------------------------------------------------------------------------
def pos_conv_weight(pc: _PosConv) -> torch.Tensor:
    """weight_norm with dim=2: w[:, :, k] = g[k] v[:, :, k] / |v[:, :, k]| (the norm over output and input channels, per tap); float64."""
    p = pc.conv.parametrizations.weight
    g, v = p.original0.detach().double(), p.original1.detach().double()
    return g * v / v.pow(2).sum(dim=(0, 1), keepdim=True).sqrt()


def fold_ln_into(w: torch.Tensor, b: torch.Tensor, ln: nn.LayerNorm):
    """y = W (gamma z + beta) + b  ->  (W diag(gamma), W beta + b), float64."""
    g, be = ln.weight.detach().double(), ln.bias.detach().double()
    return w * g[None, :], w @ be + b


def fold_weights(model: 'HubertModel') -> dict:
    """Every folded weight, float64 (except the LayerNorms the kernels apply, which stay as they are): 'conv' [(W, bias | None, ln)],
    'proj' (W [H, C], b), 'pos' (W [H, H/G, 128], b), 'layers' [(Wqkv [3H, H], bqkv, Wo, bo, W1, b1, W2, b2)], 'ln_f'."""
    d = lambda t: t.detach().double()                                         # noqa: E731
    P = {'conv': [(d(l.conv.weight), None if l.conv.bias is None else d(l.conv.bias), l.layer_norm)
                  for l in model.feature_extractor.conv_layers]}
    fp = model.feature_projection
    w, b = d(fp.projection.weight), d(fp.projection.bias)
    P['proj'] = fold_ln_into(w, b, fp.layer_norm) if fp.feat_proj_layer_norm else (w, b)
    enc = model.encoder
    P['pos'] = (pos_conv_weight(enc.pos_conv_embed), d(enc.pos_conv_embed.conv.bias))
    layers = []
    for lay in enc.layers:
        a = lay.attention
        wq = torch.cat([d(a.q_proj.weight) * 0.125, d(a.k_proj.weight), d(a.v_proj.weight)])
        bq = torch.cat([d(a.q_proj.bias) * 0.125, d(a.k_proj.bias), d(a.v_proj.bias)])
        wq, bq = fold_ln_into(wq, bq, lay.layer_norm)
        f = lay.feed_forward
        w1, b1 = fold_ln_into(d(f.intermediate_dense.weight), d(f.intermediate_dense.bias), lay.final_layer_norm)
        layers.append((wq, bq, d(a.out_proj.weight), d(a.out_proj.bias), w1, b1, d(f.output_dense.weight), d(f.output_dense.bias)))
    P['layers'] = layers
    P['ln_f'] = enc.layer_norm
    return P


def _ceil64(n: int) -> int:
    return (n + 63) // 64 * 64


def pack_split(w: torch.Tensor, Kp: Optional[int] = None) -> torch.Tensor:
    """W [N, K] float64 -> [N, hi Kp | lo Kp] fp16 of W * 2^10 (K zero-padded to Kp).  Raises ValueError when a (folded) weight is too
    large for fp16's range at that scale (|w| >= 64): the hi half would be inf and every output NaN."""
    N, K = w.shape
    big = float(w.abs().max()) if w.numel() else 0.0
    if not big * 1024.0 < 65504.0:
        raise ValueError(f'pack_split: a weight of magnitude {big:.4g} does not fit split fp16 at scale 2^10 (|w| must be < 63.97); '
                         'a LayerNorm gamma folded into a GEMM can enlarge weights this way')
    Kp = Kp or _ceil64(K)
    s = torch.zeros(N, Kp, dtype=torch.float64, device=w.device)
    s[:, :K] = w * 1024.0
    hi = s.half()
    return torch.cat([hi, (s - hi.double()).half()], 1).contiguous()


def conv_gemm_weight(w: torch.Tensor, Cp: int) -> torch.Tensor:
    """Conv [O, I, k] -> GEMM rows [O, k Cp]: K channel j Cp + i = tap j, input channel i (zero for i >= I), the order of an A window row."""
    O, I, k = w.shape
    g = torch.zeros(O, k, Cp, dtype=torch.float64, device=w.device)
    g[:, :, :I] = w.permute(0, 2, 1)
    return g.reshape(O, k * Cp)


def pos_gemm_weight(w: torch.Tensor) -> torch.Tensor:
    """Grouped pos conv [H, 64, 128] -> [H, 128 * 64]: K channel 64 j + i = tap j, input channel i of the output's group."""
    return w.permute(0, 2, 1).reshape(w.shape[0], -1)


def check_pos_conv_range(P: dict, standardised: bool) -> float:
    """The positional conv's split operand is the projection output y = W x + b, whose input row x is a standardised row z (|z|_2 = sqrt(C),
    the LayerNorm's gamma / beta folded into W) or, without feat_proj_layer_norm, GELU(gamma z + beta) with |GELU(u)| <= |u|.  So
    |y_i| <= |W_i|_2 |x|_2 + |b_i| with |x|_2 <= sqrt(C) (max |gamma| sqrt(C) + |beta|_2): a bound fixed by the weights.  Raises ValueError
    when it reaches fp16's range (the hi half would overflow); returns the bound."""
    w, b = P['proj']
    C = w.shape[1]
    if standardised:
        xn = C ** 0.5
    else:
        ln = P['conv'][-1][2]
        xn = float(ln.weight.detach().double().abs().max()) * C ** 0.5 + float(ln.bias.detach().double().norm())
    bound = float((w.norm(dim=1) * xn + b.abs()).max())
    if not bound < 65504.0:
        raise ValueError(f'HubertModel: the projection output can reach {bound:.4g}, beyond fp16 range for the positional conv\'s split operand')
    return bound


class _Output:
    def __init__(self, h):
        self.last_hidden_state = h

    def __getitem__(self, i):
        return (self.last_hidden_state,)[i]


class HubertModel(PreparedMixin, nn.Module):
    """transformers.HubertModel(config) at inference, for the hubert-large-ls960-ft architecture (see the module docstring)."""

    def __init__(self, config):
        super().__init__()
        c = _config(config)
        _check_config(c)
        self.config = c
        if c.mask_time_prob > 0.0 or c.mask_feature_prob > 0.0:
            self.masked_spec_embed = nn.Parameter(torch.empty(c.hidden_size).uniform_())
        self.feature_extractor = _FeatureExtractor(c)
        self.feature_projection = _FeatureProjection(c)
        self.encoder = _Encoder(c)
        self.eval()

    @classmethod
    def from_pretrained(cls, local_dir: str):
        """A local snapshot: config.json plus model.safetensors or pytorch_model.bin.  A HubertForCTC checkpoint loads its `hubert.` weights
        (lm_head.* is ignored).  Never reaches the network."""
        with open(os.path.join(local_dir, 'config.json')) as f:
            cfg = json.load(f)
        st = os.path.join(local_dir, 'model.safetensors')
        if os.path.exists(st):
            from safetensors.torch import load_file
            sd = load_file(st)
        else:
            sd = torch.load(os.path.join(local_dir, 'pytorch_model.bin'), map_location='cpu', weights_only=True)
        if any(k.startswith('hubert.') for k in sd):
            sd = {k[len('hubert.'):]: v for k, v in sd.items() if k.startswith('hubert.')}
        m = cls(cfg)
        m.load_state_dict(sd, strict=True)
        return m

    @property
    def device(self):
        return self.feature_projection.projection.weight.device

    def _prepared(self):
        return self.prepared('weights', self._build)

    def _build(self):
        dev = capi.cuda_device(self.feature_projection.projection.weight)
        c = self.config
        C, H = c.conv_dim[0], c.hidden_size
        Cp = _ceil64(C)
        f32 = lambda t: None if t is None else t.detach().to(dev, torch.float32).contiguous()   # noqa: E731
        with torch.no_grad():
            P = fold_weights(self)
            Q = {'C': C, 'Cp': Cp, 'H': H, 'I': c.intermediate_size, 'eps': float(c.layer_norm_eps)}
            conv = []
            for i, (w, b, ln) in enumerate(P['conv']):
                wk = f32(w[:, 0, :]) if i == 0 else pack_split(conv_gemm_weight(w, Cp)).to(dev)
                conv.append((wk, f32(b), f32(ln.weight), f32(ln.bias), float(ln.eps)))
            Q['conv'] = conv
            check_pos_conv_range(P, self.config.feat_proj_layer_norm)
            Q['proj'] = (pack_split(P['proj'][0], Cp).to(dev), f32(P['proj'][1]))
            Q['pos'] = (pack_split(pos_gemm_weight(P['pos'][0])).to(dev), f32(P['pos'][1]))
            Q['layers'] = [tuple(pack_split(w).to(dev) if j % 2 == 0 else f32(w) for j, w in enumerate(lay)) for lay in P['layers']]
            Q['ln_f'] = (f32(P['ln_f'].weight), f32(P['ln_f'].bias), float(P['ln_f'].eps))
            Q['unit'] = torch.tensor([0.0, 1.0], dtype=torch.float64, device=dev)
        return Q

    def train(self, mode: bool = True):
        if mode:
            raise NotImplementedError('HubertModel: only inference (eval mode) is built')
        return super().train(False)

    # ---- the launch sequence of one group of consecutive segments ----------------------------------------------------------------------
    def _run(self, wave: torch.Tensor, stats: torch.Tensor, f0: int, segs, out: torch.Tensor):
        """Frames [f0, f0 + sum(segs)) of the clip `wave` (fp32, device; normalised by `stats` = (mean, rstd)) -> out rows [sum(segs), H]
        (fp32, unit column stride).  Each segment is encoded on its own."""
        Q, L, st, dev = self._prepared(), capi.lib(), capi.stream(), wave.device
        ptr, chk = capi.ptr, capi.check
        C, Cp, H, I, eps = Q['C'], Q['Cp'], Q['H'], Q['I'], Q['eps']
        Fg = sum(segs)
        n = 320 * (Fg - 1) + 400                                            # the samples those frames read
        x = wave[320 * f0:320 * f0 + n]
        F = (n - 10) // 5 + 1
        mk = torch.zeros if Cp != C else torch.empty                        # split rows' pad channels stay zero
        w0, b0, g0, be0, e0 = Q['conv'][0]
        a = mk(F, 2 * Cp, device=dev, dtype=F16)
        chk(L.r3dp_hb_conv0(ptr(x), ptr(stats, torch.float64), F, C, ptr(w0), ptr(b0), ptr(g0), ptr(be0), e0, ptr(a, F16), 2 * Cp, Cp, st))
        feat = None
        for i in range(1, 7):
            k, s = KERNELS[i], STRIDES[i]
            Fo = (F - k) // s + 1
            w, b, g, be, e = Q['conv'][i]
            y = torch.empty(Fo, C, device=dev)
            chk(L.r3dp_hb_gemm(ptr(a, F16), Fo, k * 2 * Cp, s * 2 * Cp, Cp, ptr(w, F16), C, k * Cp, ptr(b), 3, ptr(y), C, 0, st))
            if i < 6 or not self.config.feat_proj_layer_norm:
                a = mk(Fo, 2 * Cp, device=dev, dtype=F16)
                chk(L.r3dp_hb_layernorm(ptr(y), Fo, C, ptr(g), ptr(be), e, 1, None, 0, ptr(a, F16), 2 * Cp, Cp, st))
            else:
                feat = y                                                    # in place: each warp reads its whole row before writing it
                chk(L.r3dp_hb_layernorm(ptr(y), Fo, C, ptr(g), ptr(be), e, 1, ptr(feat), C, None, 0, 0, st))
            F = Fo
        assert F == Fg, (F, Fg)
        if feat is not None:
            a = mk(Fg, 2 * Cp, device=dev, dtype=F16)
            chk(L.r3dp_hb_layernorm(ptr(feat), Fg, C, None, None, eps, 0, None, 0, ptr(a, F16), 2 * Cp, Cp, st))
            del feat
        h = torch.empty(Fg, H, device=dev)
        chk(L.r3dp_hb_gemm(ptr(a, F16), Fg, 2 * Cp, 2 * Cp, Cp, ptr(Q['proj'][0], F16), H, Cp, ptr(Q['proj'][1]), 3, ptr(h), H, 0, st))
        del a
        # positional conv: per-segment zero padding through a segment-padded copy of the split hidden rows
        Ls = max(segs)
        xs = torch.zeros(len(segs) * Ls, 2 * H, device=dev, dtype=F16)
        chk(L.r3dp_a2m_split(ptr(h), Fg, H, ptr(xs, F16), None, st))
        chk(L.r3dp_hb_pos_conv(ptr(xs, F16), len(segs), Ls, Fg, H, ptr(Q['pos'][0], F16), ptr(Q['pos'][1]), ptr(h), st))
        del xs
        lens = (ctypes.c_int * len(segs))(*segs)
        a = torch.empty(Fg, 2 * H, device=dev, dtype=F16)
        qkv = torch.empty(Fg, 6 * H, device=dev, dtype=F16)
        f = torch.empty(Fg, 2 * I, device=dev, dtype=F16)
        for wq, bq, wo, bo, w1, b1, w2, b2 in Q['layers']:
            chk(L.r3dp_hb_layernorm(ptr(h), Fg, H, None, None, eps, 0, None, 0, ptr(a, F16), 2 * H, H, st))
            chk(L.r3dp_hb_gemm(ptr(a, F16), Fg, 2 * H, 2 * H, H, ptr(wq, F16), 3 * H, H, ptr(bq), 0, ptr(qkv, F16), 6 * H, 3 * H, st))
            chk(L.r3dp_hb_attention(ptr(qkv, F16), Fg, 6 * H, 3 * H, H // 64, lens, len(segs), ptr(a, F16), 2 * H, H, st))
            chk(L.r3dp_hb_gemm(ptr(a, F16), Fg, 2 * H, 2 * H, H, ptr(wo, F16), H, H, ptr(bo), 2, ptr(h), H, 0, st))
            chk(L.r3dp_hb_layernorm(ptr(h), Fg, H, None, None, eps, 0, None, 0, ptr(a, F16), 2 * H, H, st))
            chk(L.r3dp_hb_gemm(ptr(a, F16), Fg, 2 * H, 2 * H, H, ptr(w1, F16), I, H, ptr(b1), 1, ptr(f, F16), 2 * I, I, st))
            chk(L.r3dp_hb_gemm(ptr(f, F16), Fg, 2 * I, 2 * I, I, ptr(w2, F16), H, I, ptr(b2), 2, ptr(h), H, 0, st))
        g, b, e = Q['ln_f']
        chk(L.r3dp_hb_layernorm(ptr(h), Fg, H, ptr(g), ptr(b), e, 0, ctypes.c_void_p(out.data_ptr()), out.stride(0), None, 0, 0, st))

    @torch.no_grad()
    def forward(self, input_values: torch.Tensor, attention_mask=None, mask_time_indices=None, output_attentions=None,
                output_hidden_states=None, return_dict=None):
        """input_values [B, L] (already normalised, as the feature extractor returns them) -> .last_hidden_state [B, (L - 400) // 320 + 1, H]
        fp32.  The whole input is one segment, as transformers runs it."""
        if attention_mask is not None or mask_time_indices is not None:
            raise NotImplementedError('HubertModel: attention_mask / mask_time_indices are not built')
        if output_attentions or output_hidden_states:
            raise NotImplementedError('HubertModel: output_attentions / output_hidden_states are not built')
        if self.training:
            raise NotImplementedError('HubertModel: only inference (eval mode) is built')
        if not isinstance(input_values, torch.Tensor) or input_values.dim() != 2:
            raise ValueError('HubertModel.forward: input_values must be a [B, L] tensor')
        if not input_values.is_cuda:
            raise RuntimeError('real3dportrait_b200 runs on CUDA tensors only (no CPU fallback); input_values is on the CPU')
        B, Lx = input_values.shape
        if Lx < 400:
            raise ValueError(f'HubertModel.forward: at least 400 samples are needed, got {Lx}')
        T = (Lx - 400) // 320 + 1
        x = capi.f32(input_values)
        out = torch.empty(B, T, self.config.hidden_size, device=x.device)
        Q = self._prepared()
        for b in range(B):
            self._run(x[b], Q['unit'], 0, [T], out[b])
        return _Output(out)


@torch.no_grad()
def get_hubert_from_16k_speech(speech, model: HubertModel, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """extract_hubert.py:19-80 on the library: a 16 kHz waveform ([L] or [L, 2], channel 0; numpy or torch, CPU or CUDA) -> HuBERT features
    [T, H] fp32 on the model's CUDA device, T = (L - 80) // 320 (the reference returns them on the CPU).  The clip is normalised as
    Wav2Vec2FeatureExtractor(do_normalize=True) does, over the whole clip (fp64 statistics on the device); the conv feature extractor runs
    over the whole clip and the encoder over consecutive 1000-frame segments, each with its own positional-conv padding and attention, as
    the reference's chunk loop computes them.  `out`: an fp32 [>= T, H] buffer on that device with unit column stride (e.g. the VAE's
    batch['audio'][0]); rows past T are zeroed (get_hubert's padding) and the return value is out[:T]."""
    if isinstance(speech, np.ndarray):
        speech = torch.from_numpy(speech)
    if not isinstance(speech, torch.Tensor) or speech.dim() not in (1, 2):
        raise ValueError('get_hubert_from_16k_speech: speech must be a [L] or [L, 2] waveform')
    if speech.dim() == 2:
        speech = speech[:, 0]
    L = speech.shape[0]
    T = hubert_frames(L)
    dev = model.device
    if dev.type != 'cuda':
        raise RuntimeError('real3dportrait_b200 runs on CUDA tensors only (no CPU fallback); move the model to a CUDA device')
    H = model.config.hidden_size
    if out is None:
        out = torch.empty(T, H, device=dev)
    elif (out.dim() != 2 or out.shape[0] < T or out.shape[1] != H or out.dtype != torch.float32 or out.device != dev or out.stride(1) != 1):
        raise ValueError(f'get_hubert_from_16k_speech: out must be an fp32 [>= {T}, {H}] tensor on {dev} with unit column stride')
    x = speech.to(dev, torch.float32).contiguous()
    Q, Lb = model._prepared(), capi.lib()
    stats = torch.empty(2, dtype=torch.float64, device=dev)
    capi.check(Lb.r3dp_hb_stats(capi.ptr(x), L, capi.ptr(stats, torch.float64), capi.stream()))
    segs = _segments(T)
    for g0 in range(0, len(segs), GROUP):
        sg = segs[g0:g0 + GROUP]
        f0 = g0 * SEG
        model._run(x, stats, f0, sg, out[f0:f0 + sum(sg)])
    if out.shape[0] > T:
        out[T:].zero_()
    return out[:T]
