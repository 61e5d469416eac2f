"""Float64 restatements of the audio2secc VAE's inference path (modules/audio2motion/vae.py, PitchContourVAEModel / VAEModel with
train=False; flow_base.py WN / ResidualCouplingBlock), seeded parameters and inputs, and the reference classes behind an hparams shim.

  forward(sd, batch, z, temperature, pitch, hp)   the network as the reference writes it, on the state_dict (weight norm, BatchNorm,
                                                  Flips, the cond_proj concatenation), float64
  forward_folded(P, batch, z, temperature, pitch) the same network on fold_weights(model): the layouts the kernels run (paired gate rows,
                                                  absorbed Flips, the one-hot blink / amplitude block, g_pre_net over groups of four
                                                  frames, the transposed conv as a GEMM), float64; with `operands`, every GEMM and conv
                                                  operand rounded as the kernels read it (split fp16, or fp16 alone at one launch)
  launch_plan(kind, A, B, Tx, hp)                 every kernel launch of the module's forward, restated from the architecture
The pitch bins are computed by f0_to_coarse_ref (the reference's float32 formula) in both."""
import math
import os
import socket
import sys
import types
import zlib

import numpy as np
import torch
import torch.nn.functional as F

from launch_harness import launch_signature  # noqa: F401  (the launch tests call it through this module)

F0_BIN, F0_MIN, F0_MAX = 256, 50.0, 1100.0
F0_MEL_MIN = 1127 * np.log(1 + F0_MIN / 700)
F0_MEL_MAX = 1127 * np.log(1 + F0_MAX / 700)
HP_PITCH = {'use_mouth_amp_embed': True, 'use_eye_amp_embed': False}
#: the end-to-end bar of the CUDA forward: max |got - exp64| <= E2E_BAR max |exp64|.  Measured on an H100 80GB HBM3 (700 W power limit):
#: worst 1.43e-5 (VAEModel, A = 1024), 1.30e-5 for the released pitch config, 5.1e-6 at A = 13.  The fp32 accumulation of enc1's K = 3072
#: products dominates it (that launch alone is 1.1e-5 of its max |ref|); the float64 emulation of split operands sits near 2e-7 and
#: float32 eager near 7e-7.  One launch reading fp16 operands alone moves the emulation by 2.9e-5 or more
#: (tests/test_cpu_audio2motion_launches.py); the per-launch rows of tests/test_gpu_audio2motion_launches.py tell those apart with 4x
#: margin or more
E2E_BAR = 2e-5
SPLIT_WEIGHT_SCALE = 1024.0                 # split weights are stored as [hi | lo] of w * 2^10


def reference_checkout():
    root = os.environ.get('R3DP_REFERENCE')
    return root if root and os.path.isdir(os.path.join(root, 'modules', 'audio2motion')) else None


class NetworkBlocked(RuntimeError):
    pass


def reference_classes(root):
    """(PitchContourVAEModel, VAEModel) from the reference, with utils.commons.hparams shimmed by an empty dict (the WN reads
    hparams.get('use_adapters') from it; the models take their own hparams).  Every socket connection raises first."""
    def refuse(*a, **k):
        raise NetworkBlocked('network access is blocked while the reference class is built')
    socket.getaddrinfo = socket.create_connection = refuse
    socket.socket.connect = refuse
    if root not in sys.path:
        sys.path.insert(0, root)
    hpm = types.ModuleType('utils.commons.hparams')
    hpm.hparams = {}
    sys.modules['utils.commons.hparams'] = hpm
    from modules.audio2motion.vae import PitchContourVAEModel, VAEModel
    return PitchContourVAEModel, VAEModel


def make_params(shapes, seed=0):
    """{key: shape} -> {key: float32 tensor}, each from its own generator (seed, crc32(key)).  Scales keep the activations O(1) and the gates
    off saturation: weight_v normal with weight_g ~ 0.5 - 1 / sqrt(#layers); `post` (zero-initialised in the reference, an identity flow)
    gets a real weight; BatchNorm statistics near identity; embeddings N(0, 0.5)."""
    out = {}
    for k, shape in shapes.items():
        g = torch.Generator().manual_seed(seed * 1_000_003 + zlib.crc32(k.encode()))
        shape = tuple(shape)
        leaf = k.rsplit('.', 1)[-1]
        if leaf == 'num_batches_tracked':
            out[k] = torch.zeros((), dtype=torch.long)
        elif leaf == 'running_mean':
            out[k] = 0.05 * torch.randn(shape, generator=g)
        elif leaf == 'running_var':
            out[k] = 1.0 + 0.2 * torch.rand(shape, generator=g)
        elif leaf == 'weight_g':
            out[k] = 0.4 + 0.4 * torch.rand(shape, generator=g)
        elif leaf == 'weight_v':
            out[k] = torch.randn(shape, generator=g)
        elif leaf == 'bias':
            out[k] = 0.05 * torch.randn(shape, generator=g)
        elif len(shape) == 1 and k.endswith('.1.weight'):               # BatchNorm gamma
            out[k] = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif len(shape) == 1 or 'embed' in k:                           # mouth / eye amp embeds, blink / pitch embeddings
            out[k] = 0.5 * torch.randn(shape, generator=g)
        else:                                                           # ConvTranspose1d weights are [in, out, k]: fan-in = in
            fan_in = shape[0] if k.endswith('decoder.pre_net.0.weight') else int(np.prod(shape[1:]))
            out[k] = torch.randn(shape, generator=g) / math.sqrt(fan_in)
    return out


def make_batch(B, Tx, A, seed, pitch=True, mouth_amp=0.45, masked=True):
    """Seeded inputs: audio ~ N(0, 1), f0 in Hz (a third unvoiced zeros, the rest 80-400 Hz), blink ids with runs of ones, y_mask ones
    (the last eighth of item 1 zero when masked and B > 1)."""
    g = torch.Generator().manual_seed(seed)
    T = Tx // 2
    batch = {'audio': torch.randn(B, Tx, A, generator=g), 'y_mask': torch.ones(B, T)}
    f0 = 80.0 + 320.0 * torch.rand(B, Tx, generator=g)
    f0[torch.rand(B, Tx, generator=g) < 0.33] = 0.0
    batch['f0'] = f0
    if masked and B > 1:
        batch['y_mask'][1, T - T // 8:] = 0.0
    if pitch:
        blink = torch.zeros(B, Tx, 1, dtype=torch.long)
        for b in range(B):
            for s in range(3 + 5 * b, Tx, 23):
                blink[b, s:s + 6] = 1
        batch['blink'] = blink
        batch['mouth_amp'] = torch.full((B, 1), mouth_amp)
    return batch


def f0_to_coarse_ref(f0):
    """utils/commons/pitch_utils.py:17-26 on a float32 CPU tensor (same ops, same order)."""
    f0_mel = 1127 * (1 + f0 / 700).log()
    f0_mel[f0_mel > 0] = (f0_mel[f0_mel > 0] - F0_MEL_MIN) * (F0_BIN - 2) / (F0_MEL_MAX - F0_MEL_MIN) + 1
    f0_mel[f0_mel <= 1] = 1
    f0_mel[f0_mel > F0_BIN - 1] = F0_BIN - 1
    return (f0_mel + 0.5).long()


def f0_mel_scaled64(f0):
    """The value f0_to_coarse rounds (before the clamp), in float64: how close each frame sits to a bin edge."""
    mel = 1127 * torch.log1p(f0.double() / 700)
    return torch.where(mel > 0, (mel - F0_MEL_MIN) * (F0_BIN - 2) / (F0_MEL_MAX - F0_MEL_MIN) + 1, mel)


# ---- the reference's network, float64 ---------------------------------------------------------------------------------------------------
def _wn_w(sd, p, dt):
    g, v = sd[p + '.weight_g'].to(dt), sd[p + '.weight_v'].to(dt)
    return g * v / v.flatten(1).norm(dim=1).view(-1, *([1] * (v.dim() - 1)))


def _wavenet(sd, p, x, g, L, H, k, dt):
    gc = F.conv1d(g, _wn_w(sd, p + '.cond_layer', dt), sd[p + '.cond_layer.bias'].to(dt))
    out = torch.zeros_like(x)
    for i in range(L):
        xi = F.conv1d(x, _wn_w(sd, f'{p}.in_layers.{i}', dt), sd[f'{p}.in_layers.{i}.bias'].to(dt), padding=k // 2)
        a = xi + gc[:, 2 * H * i:2 * H * (i + 1)]
        acts = torch.tanh(a[:, :H]) * torch.sigmoid(a[:, H:])
        rs = F.conv1d(acts, _wn_w(sd, f'{p}.res_skip_layers.{i}', dt), sd[f'{p}.res_skip_layers.{i}.bias'].to(dt))
        if i < L - 1:
            x = x + rs[:, :H]
            out = out + rs[:, H:]
        else:
            out = out + rs
    return out


def _bn(sd, p, x, dt):
    return F.batch_norm(x, sd[p + '.running_mean'].to(dt), sd[p + '.running_var'].to(dt), sd[p + '.weight'].to(dt), sd[p + '.bias'].to(dt),
                        False, 0.0, 1e-5)


def _encoder(sd, p, x, dt):
    x = F.conv1d(x, sd[p + '.0.weight'].to(dt), padding=1)
    x = F.gelu(_bn(sd, p + '.1', x, dt))
    return F.conv1d(x, sd[p + '.3.weight'].to(dt), padding=1)


def forward(sd, batch, z, temperature, pitch=True, hp=HP_PITCH, dt=torch.float64):
    """The reference's forward(batch, ret, train=False, temperature) on state_dict `sd` with the prior draw z [B,16,T/4] given, in float64
    (dt: the same eager network in another dtype, e.g. float32 on cuDNN as a timing baseline)."""
    audio = batch['audio'].to(dt)
    B, Tx, _ = audio.shape
    if pitch:
        mel = audio[:, ::2]
        f0 = batch['f0'].float()[:, ::2]
        emb = sd['pitch_embed.weight'].to(dt)[f0_to_coarse_ref(f0)]
        cond = _encoder(sd, 'mel_encoder', mel.transpose(1, 2), dt)
        pf = _encoder(sd, 'pitch_encoder', emb.transpose(1, 2), dt)
        blink = batch.get('blink', torch.zeros(B, Tx, 1, dtype=torch.long, device=audio.device))[:, ::2, 0]
        feats = [cond.transpose(1, 2), pf.transpose(1, 2), sd['blink_embed.weight'].to(dt)[blink]]
        T = mel.shape[1]
        for key, on, name in (('mouth_amp', 'use_mouth_amp_embed', 'mouth_amp_embed'), ('eye_amp', 'use_eye_amp_embed', 'eye_amp_embed')):
            if hp.get(on, False):
                amp = batch.get(key, torch.full((B, 1), 0.4, device=audio.device)).to(dt)
                feats.append((amp[:, :, None] * sd[name].to(dt)[None, None]).expand(B, T, -1))
        g = F.linear(torch.cat(feats, -1), sd['cond_proj.weight'].to(dt), sd['cond_proj.bias'].to(dt)).transpose(1, 2)
    else:
        mel = 0.5 * (audio[:, 0::2] + audio[:, 1::2])
        g = _encoder(sd, 'mel_encoder', mel.transpose(1, 2), dt)
    gs = F.conv1d(g, sd['vae.g_pre_net.0.weight'].to(dt), sd['vae.g_pre_net.0.bias'].to(dt), stride=4, padding=2)
    x = z.to(dt) * temperature
    if 'vae.prior_flow.flows.0.pre.weight' in sd:
        for i in reversed(range(4)):
            x = torch.flip(x, [1])
            p = f'vae.prior_flow.flows.{2 * i}'
            x0, x1 = x[:, :8], x[:, 8:]
            h = F.conv1d(x0, sd[p + '.pre.weight'].to(dt), sd[p + '.pre.bias'].to(dt))
            h = _wavenet(sd, p + '.enc', h, gs, 4, 64, 3, dt)
            m = F.conv1d(h, sd[p + '.post.weight'].to(dt), sd[p + '.post.bias'].to(dt))
            x = torch.cat([x0, x1 - m], 1)
    y = F.conv_transpose1d(x, sd['vae.decoder.pre_net.0.weight'].to(dt), sd['vae.decoder.pre_net.0.bias'].to(dt), stride=4)
    y = _wavenet(sd, 'vae.decoder.wn', y, g, 4, 256, 5, dt)
    y = F.conv1d(y, sd['vae.decoder.out_proj.weight'].to(dt), sd['vae.decoder.out_proj.bias'].to(dt))
    return y.transpose(1, 2) * batch['y_mask'].to(dt)[:, :, None]


# ---- the folded network (the kernels' layouts), float64 ---------------------------------------------------------------------------------
def _hi(v):
    return v.to(torch.float16).double()


class _Operands:
    """How forward_folded reads the operands of each GEMM / conv launch (tag as in launch_plan):
      'exact'  float64 as given;
      'split'  every operand as the kernels read it: activations hi + lo of their fp16 split, weights (hi + lo) / 2^10 of the split of w * 2^10;
      'hi'     fp16 hi halves alone (activations fp16(x), weights fp16(w * 2^10) / 2^10) at launch `site`, split everywhere else (site None:
               every launch hi-only)."""

    def __init__(self, mode='exact', site=None):
        assert mode in ('exact', 'split', 'hi'), mode
        self.mode, self.site, self.seen = mode, site, set()

    def _hi_only(self, tag):
        self.seen.add(tag)
        return self.mode == 'hi' and (self.site is None or self.site == tag)

    def x(self, tag, v):
        if self.mode == 'exact':
            return v
        h = _hi(v)
        return h if self._hi_only(tag) else h + _hi(v - h)

    def w(self, tag, v):
        if self.mode == 'exact':
            return v
        s = v * SPLIT_WEIGHT_SCALE
        h = _hi(s)
        return (h if self._hi_only(tag) else h + _hi(s - h)) / SPLIT_WEIGHT_SCALE


def _conv_cl(x, w, b, k, ops=None, tag=None):
    """channels-last [B, T, I] conv with w [O, I, k] (same padding) -> [B, T, O]"""
    if ops is not None:
        x, w = ops.x(tag, x), ops.w(tag, w)
    return F.conv1d(x.transpose(1, 2), w, b, padding=k // 2).transpose(1, 2)


def _gemm(x, w, b, ops, tag):
    """rows x [..., I] @ w [O, I]^T + b"""
    return ops.x(tag, x) @ ops.w(tag, w).t() + b


def _wavenet_folded(x, layers, cond, H, ops=None, prefix='wn'):
    """x [B, T, H]; layers [(w_in [2H, H, k], w_rs [NO, H], b_rs)]; cond [B, T, L*2H] paired rows with the in_layer bias added.
    Layer i is launch `{prefix}{i}`: its in_layer conv and res_skip GEMM read their operands through `ops`."""
    ops = ops or _Operands()
    skip = None
    for i, (wi, wr, br) in enumerate(layers):
        tag = f'{prefix}{i}'
        wi = wi[torch.stack([torch.arange(H), torch.arange(H) + H], 1).reshape(-1)]
        a = _conv_cl(x, wi, None, wi.shape[2], ops, tag) + cond[:, :, 2 * H * i:2 * H * (i + 1)]
        gated = torch.tanh(a[:, :, 0::2]) * torch.sigmoid(a[:, :, 1::2])
        rs = _gemm(gated, wr, br, ops, tag)
        if i < len(layers) - 1:
            x = x + rs[:, :, :H]
            skip = rs[:, :, H:] if skip is None else skip + rs[:, :, H:]
        else:
            skip = skip + rs
    return skip


def forward_folded(P, batch, z, temperature, pitch=True, hp=HP_PITCH, operands='exact', site=None):
    """The forward on fold_weights(model) in float64.  operands / site: how each launch reads its GEMM / conv operands (_Operands)."""
    ops = _Operands(operands, site)
    audio = batch['audio'].double()
    B, Tx, A = audio.shape
    T, T4 = Tx // 2, Tx // 8
    Ap = (A + 31) // 32 * 32
    mel = audio[:, ::2] if pitch else 0.5 * (audio[:, 0::2] + audio[:, 1::2])
    xin = torch.zeros(B, T, Ap, dtype=torch.float64)
    xin[:, :, :A] = mel
    (w1, b1), w2 = P['enc1'], P['enc2']
    w1p = torch.zeros(w1.shape[0], Ap, 3, dtype=torch.float64)
    w1p[:, :A] = w1
    h = F.gelu(_conv_cl(xin, w1p, b1, 3, ops, 'enc1'))
    if pitch:
        gcat = torch.zeros(B, T, 288, dtype=torch.float64)
        gcat[:, :, :128] = _conv_cl(h, w2, None, 3, ops, 'enc2')
        emb = P['pitch_table'][f0_to_coarse_ref(batch['f0'].float()[:, ::2])]
        (p1, pb1), p2 = P['penc1'], P['penc2']
        gcat[:, :, 128:256] = _conv_cl(F.gelu(_conv_cl(emb, p1, pb1, 3, ops, 'penc1')), p2, None, 3, ops, 'penc2')
        blink = batch.get('blink', torch.zeros(B, Tx, 1, dtype=torch.long))[:, ::2, 0]
        gcat[:, :, 256] = (blink == 0).double()
        gcat[:, :, 257] = (blink == 1).double()
        if hp.get('use_mouth_amp_embed', False):
            gcat[:, :, 258] = batch.get('mouth_amp', torch.full((B, 1), 0.4)).double()
        if hp.get('use_eye_amp_embed', False):
            gcat[:, :, 259] = batch.get('eye_amp', torch.full((B, 1), 0.4)).double()
        wc, bc = P['cond_proj']
        g = _gemm(gcat, wc, bc, ops, 'cond_proj')
    else:
        g = _conv_cl(h, w2, None, 3, ops, 'enc2')
    gin = g.shape[2]
    wq, bq = P['g_pre']
    gs = _conv_cl(g.reshape(B, T4, 4 * gin), wq, bq, 3, ops, 'g_pre')
    zs = torch.zeros(B, T4, 32, dtype=torch.float64)
    zs[:, :, :16] = z.double().transpose(1, 2) * temperature
    if 'flows' in P:
        wcf, bcf = P['flow_cond']
        cf = _gemm(gs, wcf, bcf, ops, 'flow_cond')
        for n, f in enumerate(P['flows']):
            wp, bp = f['pre']
            hh = _gemm(zs, wp, bp, ops, f'flow{n}.pre')
            out = _wavenet_folded(hh, f['wn'], cf[:, :, 512 * n:512 * (n + 1)], 64, ops, f'flow{n}.wn')
            wpo, bpo = f['post']
            zs[:, :, f['yc0']:f['yc0'] + 8] += _gemm(out, wpo, bpo, ops, f'flow{n}.post')
    wd, bd = P['dec_pre']
    x = _gemm(zs, wd, bd, ops, 'dec_pre').reshape(B, T, 256)
    wcd, bcd = P['dec_cond']
    y = _wavenet_folded(x, P['dec_wn'], _gemm(g, wcd, bcd, ops, 'dec_cond'), 256, ops, 'dec.wn')
    wo, bo = P['out_proj']
    out = _gemm(y, wo, bo, ops, 'out_proj') * batch['y_mask'].double()[:, :, None]
    assert site is None or site in ops.seen, f'no launch {site!r} reads GEMM operands'
    return out


# ---- the library's launch sequence, restated from the architecture ----------------------------------------------------------------------
def cop_of(cout):
    """Packed couts of an r3dp_mf_conv3d launch: cout rounded up to its cout tile (16, 32, 64 or 128)."""
    bn = 16 if cout <= 16 else 32 if cout <= 32 else 64 if cout <= 64 else 128
    return -(-cout // bn) * bn


#: launches that are not GEMMs or convolutions: no operand rounding to emulate
PACK_LAUNCHES = ('r3dp_a2m_input', 'r3dp_a2m_split', 'r3dp_a2m_latent', 'r3dp_a2m_store')


def launch_plan(kind, A, B, Tx, hp=HP_PITCH, temperature=1.0, ld=64):
    """Every kernel launch of PitchContourVAEModel (kind 'pitch') / VAEModel ('vae') forward on [B, T_x, A] features, as (tag, C entry
    point, the non-pointer arguments in C order), written from the architecture (vae.py, flow_base.py) and DESIGN.md's layouts rather than
    from the module's code.  T = T_x / 2 frames, T4 = T / 4 latent frames; every operand split fp16 ([hi | lo], lo at half the row).
    The blink / amplitude inputs (hp, batch['blink']) change pointers only, not a launch; temperature and the destination's row stride `ld`
    are arguments of r3dp_a2m_latent and r3dp_a2m_store.
      input                          audio (+ pitch row) -> xin [B*T, hi C | lo C], C = Ap (+ 128); the blink / amplitude block into gcat
      enc1, enc2 / penc1, penc2      k3 convs over B sequences of T frames (enc1 / penc1 with the GELU epilogue); the pitch model's second
                                     convs write column slices [0, 128) / [128, 256) of gcat [B*T, hi 288 | lo 288]
      cond_proj                      GEMM over gcat (K = 288) -> fp32 g [B*T, 128]   (VAEModel: enc2 writes g directly)
      split                          g -> split rows per frame and per group of four frames
      g_pre                          k3 conv over B sequences of T4 groups of four frames (K = 3 * 4 C_g)
      latent                         the draw x temperature -> zb [B*T4, hi 32 | lo 32]
      flow_cond                      the four coupling layers' cond_layers as one GEMM -> fp32 [B*T4, 2048]
      flow{n}.pre / .wn{i} / .post   per coupling layer (reversed order): pre GEMM (32 -> 64, fp32), four WaveNet layers (hidden 64, k 3), post
                                     GEMM (64 -> 8, cop 16) added in place into zb's channels [yc0, yc0 + 8), yc0 = 0 for flows 0, 2 (flipped)
      dec_cond, dec_pre              the decoder's cond GEMM -> fp32 [B*T, 2048]; the transposed conv as a GEMM 32 -> 1024 = 4 frames x 256
      dec.wn{i}, out_proj, store     four WaveNet layers (hidden 256, k 5), out_proj 256 -> 64 fp32, x y_mask into the destination"""
    assert kind in ('pitch', 'vae') and A in (1024, 13) and Tx % 8 == 0 and Tx > 0 and B > 0
    pitch = kind == 'pitch'
    T, T4 = Tx // 2, Tx // 8
    Ap = (A + 31) // 32 * 32
    C = Ap + (128 if pitch else 0)
    gin = 128 if pitch else 64
    c1 = gin
    plan = []

    def add(tag, fn, *args):
        plan.append((tag, fn, tuple(args)))

    def conv(tag, xs, xlo, cin, N, W, k, O, relu, ys, yc0, ylo, f32):
        add(tag, 'r3dp_mf_conv3d', xs, xlo, cin, N, 1, 1, W, 1, 1, k, 0, O, cop_of(O), relu, ys, yc0, ylo, int(f32), 1)

    def gemm(tag, K, R, O, ys, yc0=0, ylo=0, f32=True):
        conv(tag, 2 * K, K, K, 1, R, 1, O, 0, ys, yc0, ylo, f32)

    def wavenet(prefix, T_, hidden, k):
        for i in range(4):
            add(f'{prefix}{i}', 'r3dp_a2m_wn_layer', 2048, B, T_, hidden, k, int(i == 0), int(i == 3))

    add('input', 'r3dp_a2m_input', B, Tx, A, Ap, int(not pitch), float(F0_MEL_MIN), float(F0_MEL_MAX - F0_MEL_MIN), 2 * C, C, 576, 288)
    conv('enc1', 2 * C, C, Ap, B, T, 3, c1, 2, 2 * c1, 0, c1, False)
    if pitch:
        conv('enc2', 256, 128, 128, B, T, 3, 128, 0, 576, 0, 288, False)
        conv('penc1', 2 * C, C, 128, B, T, 3, 128, 2, 256, 0, 128, False)
        conv('penc2', 256, 128, 128, B, T, 3, 128, 0, 576, 128, 288, False)
        gemm('cond_proj', 288, B * T, gin, gin)
    else:
        conv('enc2', 2 * c1, c1, c1, B, T, 3, gin, 0, gin, 0, 0, True)
    add('split', 'r3dp_a2m_split', B * T, gin)
    conv('g_pre', 8 * gin, 4 * gin, 4 * gin, B, T4, 3, gin, 0, 2 * gin, 0, gin, False)
    add('latent', 'r3dp_a2m_latent', B, T4, float(temperature))
    gemm('flow_cond', gin, B * T4, 2048, 2048)
    for n in range(4):
        gemm(f'flow{n}.pre', 32, B * T4, 64, 64)
        wavenet(f'flow{n}.wn', T4, 64, 3)
        gemm(f'flow{n}.post', 64, B * T4, 8, 64, yc0=0 if n % 2 == 0 else 8, ylo=32, f32=False)
    gemm('dec_cond', gin, B * T, 2048, 2048)
    gemm('dec_pre', 32, B * T4, 1024, 1024)
    wavenet('dec.wn', T, 256, 5)
    gemm('out_proj', 256, B * T, 64, 64)
    add('store', 'r3dp_a2m_store', B * T, 64, ld)
    return plan
