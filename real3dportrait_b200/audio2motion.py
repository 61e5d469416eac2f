"""The audio2secc VAE (modules/audio2motion/vae.py) on libr3dp_b200: PitchContourVAEModel (the released audio2motion_vae config: use_pitch,
use_mouth_amp_embed) and VAEModel (use_pitch false), audio features + f0 -> the expression coefficients [B, T_x/2, 64] that
`forward_audio2secc` (inference/real3d_infer.py:365-388) feeds the SECC renderer.

The classes keep the reference's constructors and state_dict (keys and shapes, the unused FVAE encoder and the weight_norm g / v pairs
included) and are drop-ins at inference (`train=False`, eval mode: BatchNorm running statistics, dropout off).  Inference path
(vae.py:398-454, 309-337; FVAE.forward(infer=True) :242-269), T = T_x / 2, all channels-last rows per frame:
  - input pack (r3dp_a2m_input): audio x0.5 (pitch: frame 2i, nearest; VAEModel: the mean of 2i, 2i+1, linear), split fp16, channels padded
    to a multiple of 32; pitch model: f0 -> f0_to_coarse -> pitch_embed row, and a 32-channel block [blink == 0, blink == 1, mouth_amp,
    eye_amp, 0...] through which cond_proj's blink / amplitude columns act (so cond_proj is one GEMM and no per-clip constant needs a sync);
  - mel_encoder / pitch_encoder: k3 convs (BatchNorm folded, exact GELU in the epilogue); cond_proj: a GEMM;
  - g_pre_net (k8, stride 4, pad 2): a k3 conv over groups of four frames (4 C_g channels, zero weights on the unused taps);
  - the prior draw z = Normal(0, 1).sample([B, 16, T/4]) on the CPU generator (as the reference draws it) x temperature;
  - the prior flow reversed: four ResidualCouplingLayers (mean only); the Flips are absorbed into the pre / post weights;
    each layer: pre (GEMM), WN (4 fused r3dp_a2m_wn_layer launches), x1 -= post(h) (a GEMM with the residual in place);
  - the decoder: ConvTranspose1d(k4, s4) as a GEMM whose channels-last output is already the T-frame stream, WN (hidden 256, k5),
    out_proj (GEMM), x y_mask into `out` (r3dp_a2m_store).
Every WN cond_layer of a network is one GEMM with the layer's in_layer bias folded in and its rows paired (tanh, sigmoid) per channel.
Weights are folded on the host in float64 once per parameter set (weight norm g v / |v|, the eval BatchNorms, the Flips, cond_proj's
blink / amplitude columns, the gate pairing) and packed for the kernels (refolded after load_state_dict / .to())."""
from __future__ import annotations

import copy
import ctypes
from typing import Optional

import numpy as np
import torch
import torch.distributions as dist
import torch.nn as nn

from . import _capi as capi, conv3d
from .conv3d import pack_conv3d
from .prepared import PreparedMixin

F16 = torch.float16
LATENT = 16
F0_BIN, F0_MIN, F0_MAX = 256, 50.0, 1100.0                 # utils/commons/pitch_utils.py:4-8
F0_MEL_MIN = 1127 * np.log(1 + F0_MIN / 700)
F0_MEL_MAX = 1127 * np.log(1 + F0_MAX / 700)


def _wn(conv: nn.Module):
    return torch.nn.utils.weight_norm(conv, name='weight')


# ---- parameter containers with the reference's names -------------------------------------------------------------------------------------
class WN(nn.Module):
    """flow_base.py:21-68 (dilation rate 1, no adapters): cond_layer, in_layers, res_skip_layers, all weight-normed."""

    def __init__(self, hidden, k, n_layers, gin):
        super().__init__()
        self.hidden_channels, self.kernel_size, self.n_layers = hidden, k, n_layers
        self.in_layers = nn.ModuleList()
        self.res_skip_layers = nn.ModuleList()
        self.drop = nn.Dropout(0)
        self.cond_layer = _wn(nn.Conv1d(gin, 2 * hidden * n_layers, 1))
        for i in range(n_layers):
            self.in_layers.append(_wn(nn.Conv1d(hidden, 2 * hidden, k, padding=k // 2)))
            self.res_skip_layers.append(_wn(nn.Conv1d(hidden, 2 * hidden if i < n_layers - 1 else hidden, 1)))


class FVAEEncoder(nn.Module):
    """vae.py:99-124; in the state_dict only (the inference path never runs it)."""

    def __init__(self, cin, hidden, latent, k, n_layers, gin):
        super().__init__()
        self.pre_net = nn.Sequential(nn.Conv1d(cin, hidden, kernel_size=8, stride=4, padding=2))
        self.wn = WN(hidden, k, n_layers, gin)
        self.out_proj = nn.Conv1d(hidden, latent * 2, 1)


class FVAEDecoder(nn.Module):
    """vae.py:127-148."""

    def __init__(self, latent, hidden, cout, k, n_layers, gin):
        super().__init__()
        self.pre_net = nn.Sequential(nn.ConvTranspose1d(latent, hidden, kernel_size=4, stride=4))
        self.wn = WN(hidden, k, n_layers, gin)
        self.out_proj = nn.Conv1d(hidden, cout, 1)


class Flip(nn.Module):
    pass


class ResidualCouplingLayer(nn.Module):
    """flow_base.py:614-667, mean_only."""

    def __init__(self, channels, hidden, k, n_layers, gin):
        super().__init__()
        self.half_channels = channels // 2
        self.pre = nn.Conv1d(self.half_channels, hidden, 1)
        self.enc = WN(hidden, k, n_layers, gin)
        self.post = nn.Conv1d(hidden, self.half_channels, 1)


class ResidualCouplingBlock(nn.Module):
    """flow_base.py:670-703: [layer, Flip] x n_flows."""

    def __init__(self, channels, hidden, k, n_layers, n_flows, gin):
        super().__init__()
        self.flows = nn.ModuleList()
        for _ in range(n_flows):
            self.flows.append(ResidualCouplingLayer(channels, hidden, k, n_layers, gin))
            self.flows.append(Flip())


class FVAE(nn.Module):
    """vae.py:150-191 as both audio2secc models build it: hidden 256, latent 16, k 5, encoder 8 / decoder 4 layers, stride 4, prior flow
    of 4 coupling layers (hidden 64, k 3, 4 layers)."""

    def __init__(self, gin, use_prior_glow):
        super().__init__()
        self.latent_size = LATENT
        self.use_prior_glow = use_prior_glow
        self.g_pre_net = nn.Sequential(nn.Conv1d(gin, gin, kernel_size=8, stride=4, padding=2))
        self.encoder = FVAEEncoder(64, 256, LATENT, 5, 8, gin)
        if use_prior_glow:
            self.prior_flow = ResidualCouplingBlock(LATENT, 64, 3, 4, 4, gin)
        self.decoder = FVAEDecoder(LATENT, 256, 64, 5, 4, gin)
        self.prior_dist = dist.Normal(0, 1)


def _encoder(cin, c):
    return nn.Sequential(nn.Conv1d(cin, c, 3, 1, 1, bias=False), nn.BatchNorm1d(c), nn.GELU(), nn.Conv1d(c, c, 3, 1, 1, bias=False))


# ---- host-side folding (float64) ---------------------------------------------------------------------------------------------------------
def wn_weight(m: nn.Module) -> torch.Tensor:
    """torch.nn.utils.weight_norm (dim 0): weight = g v / |v|, the norm over every dim but the output channel; float64."""
    g, v = m.weight_g.detach().double(), m.weight_v.detach().double()
    return g * v / v.flatten(1).norm(dim=1).view(-1, *([1] * (v.dim() - 1)))


def fold_conv_bn(w: torch.Tensor, bn: nn.BatchNorm1d):
    """bias-free conv [O, I, k] -> eval BatchNorm  ->  (W float64 scaled by s, bias), s = gamma / sqrt(var + eps)."""
    s = bn.weight.detach().double() / torch.sqrt(bn.running_var.detach().double() + bn.eps)
    return w.detach().double() * s[:, None, None], bn.bias.detach().double() - bn.running_mean.detach().double() * s


def gate_order(h: int) -> torch.Tensor:
    """Row order of a 2h-row in_layer / cond slice as the WN kernel reads it: row 2c = channel c (tanh half), 2c + 1 = row h + c (sigmoid)."""
    return torch.stack([torch.arange(h), torch.arange(h) + h], 1).reshape(-1)


def fold_cond(wn: WN):
    """The WaveNet's cond_layer with each layer's in_layer bias added and every 2H slice in gate_order: (W [L*2H, C_g], b [L*2H])."""
    H, L = wn.hidden_channels, wn.n_layers
    w = wn_weight(wn.cond_layer)[:, :, 0]
    b = wn.cond_layer.bias.detach().double().clone()
    for i in range(L):
        b[i * 2 * H:(i + 1) * 2 * H] += wn.in_layers[i].bias.detach().double()
    idx = torch.cat([i * 2 * H + gate_order(H) for i in range(L)])
    return w[idx], b[idx]


def pack_wn_layer(w_in: torch.Tensor, w_rs: torch.Tensor) -> torch.Tensor:
    """in_layer [2H, H, k] and res_skip [NO, H] (float64) -> the r3dp_a2m_wn_layer weight steps [S, 2, 64, 32] fp16 ([hi | lo] of w * 2^10):
    in_layer steps (gate chunk j of 32 channels in gate_order, tap, input chunk c), then res_skip steps (output chunk n of 64, input chunk c)."""
    H2, H, k = w_in.shape
    NC = H // 32
    wi = w_in[gate_order(H).to(w_in.device)]                                   # rows paired per channel
    steps = []
    for j in range(H2 // 64):
        for tap in range(k):
            for c in range(NC):
                steps.append(wi[64 * j:64 * (j + 1), 32 * c:32 * (c + 1), tap])
    for n in range(w_rs.shape[0] // 64):
        for c in range(NC):
            steps.append(w_rs[64 * n:64 * (n + 1), 32 * c:32 * (c + 1)])
    s = torch.stack(steps) * 1024.0
    hi = s.half()
    return torch.stack([hi, (s - hi.double()).half()], 1).contiguous()


def fold_weights(model: nn.Module) -> dict:
    """Every folded weight of the inference path, float64, on the parameters' device.  Keys:
      'enc1', 'enc2' (mel_encoder: conv1 + BN [C_g', A, 3] + bias; conv2 [C_g', C_g', 3]), 'penc1', 'penc2' (pitch model),
      'pitch_table' [300, 128], 'cond_proj' (W [128, 288] over [mel | pitch | blink0, blink1, mouth, eye, 0...], bias),
      'g_pre' (W [C_g, 4 C_g, 3] over groups of four frames, bias), 'flow_cond' / 'dec_cond' (fold_cond of every WN, stacked),
      'flows': per coupling layer in reverse order (the order the flow runs) {pre (W [64, 32] over the physical state, b), wn: [(w_in, b_in,
      w_rs, b_rs)], post (W [8, 64] negated, b negated), yc0}, 'dec_pre' (W [1024, 32], b [1024]), 'dec_wn', 'out_proj'."""
    d = lambda t: t.detach().double()                                           # noqa: E731
    P = {}
    pitch = isinstance(model, PitchContourVAEModel)
    w1, b1 = fold_conv_bn(model.mel_encoder[0].weight, model.mel_encoder[1])
    P['enc1'], P['enc2'] = (w1, b1), d(model.mel_encoder[3].weight)
    gin = model.mel_encoder[3].weight.shape[0]
    if pitch:
        w1, b1 = fold_conv_bn(model.pitch_encoder[0].weight, model.pitch_encoder[1])
        P['penc1'], P['penc2'] = (w1, b1), d(model.pitch_encoder[3].weight)
        P['pitch_table'] = d(model.pitch_embed.weight)
        W = d(model.cond_proj.weight)
        wc = torch.zeros(128, 288, dtype=torch.float64, device=W.device)
        wc[:, :256] = W[:, :256]
        E = d(model.blink_embed.weight)                                          # [2, 128]
        wc[:, 256:258] = W[:, 256:384] @ E.t()
        col = 384
        if model.hparams.get('use_mouth_amp_embed', False):
            wc[:, 258] = W[:, col:col + 128] @ d(model.mouth_amp_embed)
            col += 128
        if model.hparams.get('use_eye_amp_embed', False):
            wc[:, 259] = W[:, col:col + 128] @ d(model.eye_amp_embed)
        P['cond_proj'] = (wc, d(model.cond_proj.bias))
    vae = model.vae
    g = vae.g_pre_net[0]
    wg = d(g.weight)                                                             # [C_g, C_g, 8]
    wq = torch.zeros(gin, 4 * gin, 3, dtype=torch.float64, device=wg.device)
    for j in range(8):                                                           # input frame 4t - 2 + j = group t - 1 + (j + 2) // 4
        tap, r = (j + 2) // 4, (j + 2) % 4
        wq[:, r * gin:(r + 1) * gin, tap] = wg[:, :, j]
    P['g_pre'] = (wq, d(g.bias))

    def wn_layers(wn):
        return [(wn_weight(wn.in_layers[i]), wn_weight(wn.res_skip_layers[i])[:, :, 0], d(wn.res_skip_layers[i].bias))
                for i in range(wn.n_layers)]

    if vae.use_prior_glow:
        layers = [f for f in vae.prior_flow.flows if isinstance(f, ResidualCouplingLayer)]
        flows, conds = [], []
        for n, lay in enumerate(reversed(layers)):
            flipped = n % 2 == 0                    # reversed order runs Flip, layer, Flip, layer ...: odd flips before layers 3 and 1
            x0 = [15 - j for j in range(8)] if flipped else list(range(8))
            wp = torch.zeros(64, 32, dtype=torch.float64, device=wg.device)
            wp[:, x0] = d(lay.pre.weight)[:, :, 0]
            # x1 channel j sits at physical 7 - j (flipped) or 8 + j; the post GEMM writes channels [yc0, yc0 + 8)
            wpost, bpost = -d(lay.post.weight)[:, :, 0], -d(lay.post.bias)
            if flipped:
                wpost, bpost = wpost.flip(0), bpost.flip(0)
            flows.append({'pre': (wp, d(lay.pre.bias)), 'wn': wn_layers(lay.enc), 'post': (wpost, bpost), 'yc0': 0 if flipped else 8})
            conds.append(fold_cond(lay.enc))
        P['flows'] = flows
        P['flow_cond'] = (torch.cat([c[0] for c in conds]), torch.cat([c[1] for c in conds]))
    dec = vae.decoder
    wt = d(dec.pre_net[0].weight)                                                # [16, 256, 4]
    wd = torch.zeros(1024, 32, dtype=torch.float64, device=wt.device)
    wd[:, :LATENT] = wt.permute(2, 1, 0).reshape(1024, LATENT)                   # row r * 256 + o: output frame 4u + r, channel o
    P['dec_pre'] = (wd, d(dec.pre_net[0].bias).repeat(4))
    P['dec_cond'] = fold_cond(dec.wn)
    P['dec_wn'] = wn_layers(dec.wn)
    P['out_proj'] = (d(dec.out_proj.weight)[:, :, 0], d(dec.out_proj.bias))
    return P


def f0_to_coarse(f0: torch.Tensor) -> torch.Tensor:
    """utils/commons/pitch_utils.py:17-26 on a float32 tensor (the reference's formula and evaluation order, without its assert)."""
    f0_mel = 1127 * (1 + f0 / 700).log()
    pos = f0_mel > 0
    f0_mel[pos] = (f0_mel[pos] - F0_MEL_MIN) * (F0_BIN - 2) / (F0_MEL_MAX - F0_MEL_MIN) + 1
    f0_mel[f0_mel <= 1] = 1
    f0_mel[f0_mel > F0_BIN - 1] = F0_BIN - 1
    return (f0_mel + 0.5).long()


# ---- the models --------------------------------------------------------------------------------------------------------------------------
class _Audio2Motion(PreparedMixin, nn.Module):
    pitch = False

    def _check_config(self, in_out_dim, audio_in_dim, sqz_prior):
        name = type(self).__name__
        if sqz_prior:
            raise NotImplementedError(f'{name}: sqz_prior=True is a training-time variant and is not built')
        if in_out_dim != 64:
            raise NotImplementedError(f'{name}: only in_out_dim=64 (the expression coefficients) is built, got {in_out_dim}')
        if audio_in_dim not in (1024, 13):
            raise NotImplementedError(f'{name}: audio_in_dim must be 1024 (hubert) or 13 (mfcc), got {audio_in_dim}')

    @property
    def device(self):
        return next(self.vae.parameters()).device

    def _prepared(self):
        return self.prepared('weights', self._build)

    def _build(self):
        dev = capi.cuda_device(next(self.vae.parameters()))
        with torch.no_grad():
            P = fold_weights(self)

            def conv(wb, cin):                                              # [O, I, k] or [O, I] -> r3dp_mf_conv3d taps along W
                w, b = wb
                if w.dim() == 2:
                    w = w[:, :, None]
                return pack_conv3d(w[None, :, :, None, None, :], b, cin, True)

            def wn(layers):
                return [(pack_wn_layer(wi, wr).to(dev), br.to(dev, torch.float32).contiguous()) for wi, wr, br in layers]

            A, Ap = self.audio_in_dim, conv3d.ceil32(self.audio_in_dim)
            Q = {'A': A, 'Ap': Ap, 'gin': P['enc2'].shape[0]}
            Q['enc1'] = conv(P['enc1'], Ap)
            Q['enc2'] = conv((P['enc2'], None), P['enc2'].shape[1])
            if self.pitch:
                Q['penc1'] = conv(P['penc1'], 128)
                Q['penc2'] = conv((P['penc2'], None), 128)
                Q['pitch_table'] = P['pitch_table'].to(torch.float32).contiguous()
                Q['cond_proj'] = conv(P['cond_proj'], 288)
            Q['g_pre'] = conv(P['g_pre'], 4 * Q['gin'])
            if 'flows' in P:
                Q['flow_cond'] = conv(P['flow_cond'], Q['gin'])
                Q['flows'] = [{'pre': conv(f['pre'], 32), 'wn': wn(f['wn']), 'post': conv(f['post'], 64), 'yc0': f['yc0']} for f in P['flows']]
            Q['dec_pre'] = conv(P['dec_pre'], 32)
            Q['dec_cond'] = conv(P['dec_cond'], Q['gin'])
            Q['dec_wn'] = wn(P['dec_wn'])
            Q['out_proj'] = conv(P['out_proj'], 256)
        return Q

    # ---- input checks --------------------------------------------------------------------------------------------------------------
    def _inputs(self, batch, z):
        name = type(self).__name__
        for key in ('audio', 'f0', 'y_mask'):
            if key not in batch:
                raise KeyError(f'{name}.forward: batch[{key!r}] is required')
        audio, f0, mask = batch['audio'], batch['f0'], batch['y_mask']
        if audio.dim() != 3 or audio.shape[2] != self.audio_in_dim:
            raise ValueError(f'{name}.forward: audio must be [B, T_x, {self.audio_in_dim}], got {tuple(audio.shape)}')
        B, Tx = audio.shape[:2]
        if Tx % 8 or Tx == 0:
            raise ValueError(f'{name}.forward: T_x must be a positive multiple of 8 (the decoder rebuilds 4 * (T/4) frames; pad the features '
                             f'as get_hubert does), got {Tx}')
        if f0.dim() != 2 or tuple(f0.shape) != (B, Tx):
            raise ValueError(f'{name}.forward: f0 must be [B, T_x] = [{B}, {Tx}] like audio, got {tuple(f0.shape)}')
        T = Tx // 2
        if tuple(mask.shape) != (B, T):
            raise ValueError(f'{name}.forward: y_mask must be [B, T_x/2] = [{B}, {T}], got {tuple(mask.shape)}')
        if z is not None and tuple(z.shape) != (B, LATENT, Tx // 8):
            raise ValueError(f'{name}.forward: z must be [B, 16, T_x/8] = [{B}, 16, {Tx // 8}], got {tuple(z.shape)}')
        for key, t in batch.items():
            if isinstance(t, torch.Tensor) and key in ('audio', 'f0', 'y_mask', 'blink', 'mouth_amp', 'eye_amp') and not t.is_cuda:
                raise RuntimeError(f'real3dportrait_b200 runs on CUDA tensors only (no CPU fallback); batch[{key!r}] is on the CPU')
        return B, Tx

    # ---- public interface ----------------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, batch, ret, train=False, return_latent=False, temperature=1., z: Optional[torch.Tensor] = None,
                out: Optional[torch.Tensor] = None):
        """The reference's forward at inference (train=False): batch['audio'] [B, T_x, A], batch['f0'] [B, T_x], batch['y_mask'] [B, T_x/2],
        optional batch['blink'] [B, T_x, 1] int64 (default zeros), 'mouth_amp' / 'eye_amp' [B, 1] (default 0.4) -> the expression
        coefficients [B, T_x/2, 64] fp32 (also ret['pred']; ret['mask'] = y_mask).  The prior noise is drawn as the reference draws it
        (prior_dist.sample on the CPU generator) unless `z` [B, 16, T_x/8] is given.  `out`: an fp32 [B*T_x/2, 64] destination with unit
        column stride and any row stride (e.g. rows[:, 80:144] of the engine's [id | exp | t | T] rows); the return value is then its view."""
        name = type(self).__name__
        if train:
            raise NotImplementedError(f'{name}: only the inference path (train=False) is built')
        B, Tx = self._inputs(batch, z)
        T, T4 = Tx // 2, Tx // 8
        dev = batch['audio'].device
        f0 = capi.f32(batch['f0'])
        blink = batch.get('blink')
        if blink is not None:
            if blink.numel() != B * Tx:
                raise ValueError(f'{name}.forward: blink must be [B, T_x, 1], got {tuple(blink.shape)}')
            blink = blink.reshape(B, Tx).to(torch.int64).contiguous()
        if self.pitch:
            # the one host sync: inputs on which the reference's f0_to_coarse asserts or its blink_embed lookup fails
            bad = torch.isnan(f0).any() | (f0 < -700).any()
            if blink is not None:
                bad = torch.stack([bad, ((blink != 0) & (blink != 1)).any()]).any()
            if bool(bad):
                raise ValueError(f'{name}.forward: f0 has NaN or values below -700 (f0_to_coarse asserts on them) or blink ids outside {{0, 1}}')
        if z is None:
            z = self.vae.prior_dist.sample([B, LATENT, T4])
        z = z.to(dev, torch.float32).contiguous()
        mask = capi.f32(batch['y_mask'])
        if out is None:
            out = torch.empty(B * T, 64, device=dev)
        elif (out.dim() != 2 or tuple(out.shape) != (B * T, 64) or out.dtype != torch.float32 or out.device != dev or out.stride(1) != 1
              or out.stride(0) < 64):
            raise ValueError(f'{name}.forward: out must be an fp32 [{B * T}, 64] tensor on {dev} with unit column stride')
        amps = []
        if self.pitch:
            for key, on in (('mouth_amp', 'use_mouth_amp_embed'), ('eye_amp', 'use_eye_amp_embed')):
                if not self.hparams.get(on, False):
                    amps.append(None)
                    continue
                a = batch.get(key)
                a = torch.full((B,), 0.4, device=dev) if a is None else capi.f32(a.reshape(B))
                amps.append(a)
        self._run(capi.f32(batch['audio']), f0, blink, amps, z, float(temperature), mask, out, B, Tx)
        pred = out.unflatten(0, (B, T))
        ret['pred'] = pred
        ret['mask'] = batch['y_mask']
        return pred

    # ---- the launch sequence -----------------------------------------------------------------------------------------------------------
    def _run(self, audio, f0, blink, amps, z, temperature, mask, out, B, Tx):
        Q, L, st, dev = self._prepared(), capi.lib(), capi.stream(), audio.device
        T, T4 = Tx // 2, Tx // 8
        A, Ap, gin = Q['A'], Q['Ap'], Q['gin']
        ptr = capi.ptr

        def at(t, halves=0):
            return ctypes.c_void_p(t.data_ptr() + 2 * halves)

        def wavenet(x, layers, cond, cs, hidden, k, rows, wn_out):
            """x fp32 [B*rows, hidden] (clobbered) -> wn_out split [B*rows, hi | lo]; cond fp32 rows (cs floats), layer i at 2 * hidden * i."""
            xb = torch.empty_like(x)
            skip = torch.empty_like(x)
            n = len(layers)
            for i, (w, b) in enumerate(layers):
                last = i == n - 1
                capi.check(L.r3dp_a2m_wn_layer(ptr(x), None if last else ptr(xb), ctypes.c_void_p(cond.data_ptr() + 4 * 2 * hidden * i), cs,
                                               ptr(w, F16), ptr(b), ptr(skip), ptr(wn_out, F16) if last else None, B, rows, hidden, k,
                                               int(i == 0), int(last), st))
                x, xb = xb, x

        with capi.region('audio2motion'):
            # front end: xin = [audio Ap | pitch 128] split rows; the pitch model's cond_proj input gcat = [mel 128 | pitch 128 | blink /
            # amplitude 32] split rows, the last block written by the input pack, the first two by the encoders' last convs
            C = Ap + (128 if self.pitch else 0)
            xin = torch.empty(B * T, 2 * C, device=dev, dtype=F16)
            gcat = torch.empty(B * T, 576, device=dev, dtype=F16) if self.pitch else None
            capi.check(L.r3dp_a2m_input(ptr(audio), B, Tx, A, Ap, int(not self.pitch), ptr(f0) if self.pitch else None,
                                        ptr(blink, torch.int64) if self.pitch and blink is not None else None,
                                        ptr(amps[0]) if self.pitch else None, ptr(amps[1]) if self.pitch else None,
                                        ptr(Q['pitch_table']) if self.pitch else None, float(F0_MEL_MIN), float(F0_MEL_MAX - F0_MEL_MIN),
                                        ptr(xin, F16), 2 * C, C, at(gcat, 256) if self.pitch else None, 576, 288, st))
            c1 = Q['enc1'][2]
            h1 = torch.empty(B * T, 2 * c1, device=dev, dtype=F16)
            gf = torch.empty(B * T, gin, device=dev)
            conv3d.launch(Q['enc1'], xin, 2 * C, C, Ap, (B, 1, 1, T), (1, 1, 3), h1, 2 * c1, ylo=c1, relu=2, stream=st)
            if self.pitch:
                conv3d.launch(Q['enc2'], h1, 256, 128, 128, (B, 1, 1, T), (1, 1, 3), gcat, 576, 0, 288, stream=st)
                conv3d.launch(Q['penc1'], at(xin, Ap), 2 * C, C, 128, (B, 1, 1, T), (1, 1, 3), h1, 256, 0, 128, relu=2, stream=st)
                conv3d.launch(Q['penc2'], h1, 256, 128, 128, (B, 1, 1, T), (1, 1, 3), gcat, 576, 128, 288, stream=st)
                del h1
                conv3d.launch(Q['cond_proj'], gcat, 576, 288, 288, (1, 1, 1, B * T), (1, 1, 1), gf, gin, stream=st)
                del gcat
            else:
                conv3d.launch(Q['enc2'], h1, 2 * c1, c1, c1, (B, 1, 1, T), (1, 1, 3), gf, gin, stream=st)
                del h1
            del xin
            g = torch.empty(B * T, 2 * gin, device=dev, dtype=F16)
            g4 = torch.empty(B * T4, 8 * gin, device=dev, dtype=F16)
            capi.check(L.r3dp_a2m_split(ptr(gf), B * T, gin, ptr(g, F16), ptr(g4, F16), st))
            del gf
            gs = torch.empty(B * T4, 2 * gin, device=dev, dtype=F16)
            conv3d.launch(Q['g_pre'], g4, 8 * gin, 4 * gin, 4 * gin, (B, 1, 1, T4), (1, 1, 3), gs, 2 * gin, 0, gin, stream=st)
            del g4
            # prior flow, reversed
            zb = torch.empty(B * T4, 64, device=dev, dtype=F16)
            capi.check(L.r3dp_a2m_latent(ptr(z), B, T4, temperature, ptr(zb, F16), st))
            if 'flows' in Q:
                cf = torch.empty(B * T4, 2048, device=dev)
                conv3d.launch(Q['flow_cond'], gs, 2 * gin, gin, gin, (1, 1, 1, B * T4), (1, 1, 1), cf, 2048, stream=st)
                h = torch.empty(B * T4, 64, device=dev)
                ho = torch.empty(B * T4, 128, device=dev, dtype=F16)
                for n, f in enumerate(Q['flows']):
                    conv3d.launch(f['pre'], zb, 64, 32, 32, (1, 1, 1, B * T4), (1, 1, 1), h, 64, stream=st)
                    wavenet(h, f['wn'], cf[:, 512 * n:], 2048, 64, 3, T4, ho)
                    conv3d.launch(f['post'], ho, 128, 64, 64, (1, 1, 1, B * T4), (1, 1, 1), zb, 64, f['yc0'], 32, res=zb, stream=st)
                del cf, h, ho
            del gs
            # decoder
            cd = torch.empty(B * T, 2048, device=dev)
            conv3d.launch(Q['dec_cond'], g, 2 * gin, gin, gin, (1, 1, 1, B * T), (1, 1, 1), cd, 2048, stream=st)
            del g
            x = torch.empty(B * T, 256, device=dev)
            conv3d.launch(Q['dec_pre'], zb, 64, 32, 32, (1, 1, 1, B * T4), (1, 1, 1), x, 1024, stream=st)
            del zb
            ho = torch.empty(B * T, 512, device=dev, dtype=F16)
            wavenet(x, Q['dec_wn'], cd, 2048, 256, 5, T, ho)
            del x, cd
            y = torch.empty(B * T, 64, device=dev)
            conv3d.launch(Q['out_proj'], ho, 512, 256, 256, (1, 1, 1, B * T), (1, 1, 1), y, 64, stream=st)
            del ho
            capi.check(L.r3dp_a2m_store(ptr(y), ptr(mask), B * T, 64, ctypes.c_void_p(out.data_ptr()), out.stride(0), st))
        return out


class PitchContourVAEModel(_Audio2Motion):
    """PitchContourVAEModel(hparams, in_out_dim=64, audio_in_dim=1024, sqz_prior=False, cond_drop=False, use_prior_flow=True) (vae.py:340-385).
    `hparams` is a plain dict; only use_mouth_amp_embed / use_eye_amp_embed are read."""
    pitch = True

    def __init__(self, hparams, in_out_dim=64, audio_in_dim=1024, sqz_prior=False, cond_drop=False, use_prior_flow=True):
        super().__init__()
        self._check_config(in_out_dim, audio_in_dim, sqz_prior)
        self.hparams = copy.deepcopy(dict(hparams or {}))
        feat = 128
        self.audio_in_dim = audio_in_dim
        self.blink_embed = nn.Embedding(2, feat)
        self.mel_encoder = _encoder(audio_in_dim, feat)
        self.pitch_embed = nn.Embedding(300, feat)
        self.pitch_encoder = _encoder(feat, feat)
        cond_dim = 3 * feat
        if self.hparams.get('use_mouth_amp_embed', False):
            self.mouth_amp_embed = nn.Parameter(torch.randn(feat))
            cond_dim += feat
        if self.hparams.get('use_eye_amp_embed', False):
            self.eye_amp_embed = nn.Parameter(torch.randn(feat))
            cond_dim += feat
        self.cond_proj = nn.Linear(cond_dim, feat, bias=True)
        self.cond_drop = cond_drop
        if cond_drop:
            self.dropout = nn.Dropout(0.5)
        self.in_dim = self.out_dim = in_out_dim
        self.sqz_prior, self.use_prior_flow = sqz_prior, use_prior_flow
        self.vae = FVAE(feat, use_prior_flow)


class VAEModel(_Audio2Motion):
    """VAEModel(in_out_dim=64, audio_in_dim=1024, sqz_prior=False, cond_drop=False, use_prior_flow=True) (vae.py:272-296)."""

    def __init__(self, in_out_dim=64, audio_in_dim=1024, sqz_prior=False, cond_drop=False, use_prior_flow=True):
        super().__init__()
        self._check_config(in_out_dim, audio_in_dim, sqz_prior)
        feat = 64
        self.blink_embed = nn.Embedding(2, feat)
        self.audio_in_dim = audio_in_dim
        self.mel_encoder = _encoder(audio_in_dim, feat)
        self.cond_drop = cond_drop
        if cond_drop:
            self.dropout = nn.Dropout(0.5)
        self.in_dim = self.out_dim = in_out_dim
        self.sqz_prior, self.use_prior_flow = sqz_prior, use_prior_flow
        self.vae = FVAE(feat, use_prior_flow)
