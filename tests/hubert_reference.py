"""Float64 restatements of HuBERT (transformers' HubertModel, hubert-large architecture) and of extract_hubert.py's chunking, written from
the architecture: `forward_unfolded` as transformers writes it (from a state_dict), `forward_folded` on real3dportrait_b200.hubert's folded
weights in the kernels' layouts (GEMM rows, the conv windows' K order, the pos conv's tap-major K order), exact or with every GEMM,
attention and positional-conv operand rounded as the kernels read it (split fp16, or fp16 hi halves alone at one launch), and
`launch_plan`, every kernel launch of the module restated from the architecture."""
import math

import torch
import torch.nn.functional as Fn

from launch_harness import launch_signature  # noqa: F401  (the launch tests call it through this module)

KERNELS, STRIDES = (10, 3, 3, 3, 3, 2, 2), (5, 2, 2, 2, 2, 2, 2)
#: the end-to-end bar of get_hubert_from_16k_speech: max |got - exp64| <= E2E_BAR max |exp64|.  Measured on an H100 80GB HBM3 (700 W power
#: limit): hubert-large worst 4.4e-6 (T = 1 ... 9000), the small config worst 6.9e-6 (L up to 9 600 400).  The float64 emulation of split
#: operands sits at 1.6e-8 (hubert-large, T = 49) and with every operand fp16 hi alone at 6.3e-5, 3.1x this bar
#: (tests/test_cpu_hubert_launches.py); one launch that loses its lo halves moves it by only 4e-7 ... 2.5e-5, so the per-launch rows of
#: tests/test_gpu_hubert_launches.py are the tests that name such a launch
E2E_BAR = 2e-5


def gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def ln(x, g=None, b=None, eps=1e-5):
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    y = (x - mu) / torch.sqrt(var + eps)
    return y if g is None else y * g + b


def normalise(speech):
    x = torch.as_tensor(speech).double()
    return (x - x.mean()) / torch.sqrt(x.var(unbiased=False) + 1e-7)


def pos_weight(sd, p='encoder.pos_conv_embed.conv.'):
    g = sd.get(p + 'parametrizations.weight.original0', sd.get(p + 'weight_g')).double()
    v = sd.get(p + 'parametrizations.weight.original1', sd.get(p + 'weight_v')).double()
    return g * v / v.pow(2).sum(dim=(0, 1), keepdim=True).sqrt()


def forward_unfolded(sd, cfg, x):
    """x [L] float64 (normalised) -> last_hidden_state [T, H] float64."""
    sd = {k: v.double() for k, v in sd.items()}
    H, heads, eps = cfg['hidden_size'], cfg['num_attention_heads'], cfg.get('layer_norm_eps', 1e-5)
    h = x[None, None]
    for i in range(7):
        p = f'feature_extractor.conv_layers.{i}.'
        h = Fn.conv1d(h, sd[p + 'conv.weight'], sd.get(p + 'conv.bias'), stride=STRIDES[i])
        h = gelu(ln(h.transpose(1, 2), sd[p + 'layer_norm.weight'], sd[p + 'layer_norm.bias']).transpose(1, 2))
    h = h[0].t()
    if 'feature_projection.layer_norm.weight' in sd:
        h = ln(h, sd['feature_projection.layer_norm.weight'], sd['feature_projection.layer_norm.bias'], eps)
    h = h @ sd['feature_projection.projection.weight'].t() + sd['feature_projection.projection.bias']
    K, G = cfg.get('num_conv_pos_embeddings', 128), cfg['num_conv_pos_embedding_groups']
    pc = Fn.conv1d(h.t()[None], pos_weight(sd), sd['encoder.pos_conv_embed.conv.bias'], padding=K // 2, groups=G)[0, :, :-1]
    h = h + gelu(pc.t())
    T = h.shape[0]
    for li in range(cfg['num_hidden_layers']):
        p = f'encoder.layers.{li}.'
        a = ln(h, sd[p + 'layer_norm.weight'], sd[p + 'layer_norm.bias'], eps)
        lin = lambda n, z: z @ sd[p + n + '.weight'].t() + sd[p + n + '.bias']   # noqa: E731
        q = lin('attention.q_proj', a).view(T, heads, 64).transpose(0, 1) * 0.125
        k = lin('attention.k_proj', a).view(T, heads, 64).transpose(0, 1)
        v = lin('attention.v_proj', a).view(T, heads, 64).transpose(0, 1)
        o = torch.softmax(q @ k.transpose(1, 2), -1) @ v
        h = h + lin('attention.out_proj', o.transpose(0, 1).reshape(T, H))
        f = ln(h, sd[p + 'final_layer_norm.weight'], sd[p + 'final_layer_norm.bias'], eps)
        h = h + lin('feed_forward.output_dense', gelu(lin('feed_forward.intermediate_dense', f)))
    return ln(h, sd['encoder.layer_norm.weight'], sd['encoder.layer_norm.bias'], eps)


SPLIT_WEIGHT_SCALE = 1024.0                 # split weights are stored as [hi | lo] of w * 2^10
P_SCALE = 1024.0                            # attention splits P = exp(s - m) after scaling it by 2^10


def _round(v, scale, hi_only):
    """v as the kernels read a split operand of v * scale: (hi + lo) / scale, or hi / scale alone."""
    s = v * scale
    h = s.to(torch.float16).double()
    return (h if hi_only else h + (s - h).to(torch.float16).double()) / scale


class _Operands:
    """How forward_folded reads the operands of each GEMM, attention and positional-conv launch (site names as folded_sites lists them):
      'exact'  float64 as given;
      'split'  every operand as the kernels read it: activations hi + lo of their fp16 split, weights (hi + lo) / 2^10 of the split of
               w * 2^10, attention's P (hi + lo) / 2^10 of the split of P * 2^10;
      'hi'     fp16 hi halves alone at launch `site`, split everywhere else (site None: every launch hi-only).
    Rounded weights are cached in `cache` (a dict kept with the weights), so a sweep over sites rounds each weight twice."""

    def __init__(self, mode, site, cache):
        if mode not in ('exact', 'split', 'hi'):
            raise ValueError(f'operands must be exact, split or hi, not {mode!r}')
        self.mode, self.site, self.cache = mode, site, cache

    def _hi_only(self, tag):
        return self.mode == 'hi' and (self.site is None or self.site == tag)

    def x(self, tag, v, scale=1.0):
        return v if self.mode == 'exact' else _round(v, scale, self._hi_only(tag))

    def w(self, tag, key, make):
        """The weight `key` (built by make() in float64) as launch `tag` reads it."""
        form = 'exact' if self.mode == 'exact' else 'hi' if self._hi_only(tag) else 'split'
        if (key, form) not in self.cache:
            w = self.cache[(key, 'exact')] if (key, 'exact') in self.cache else make()
            self.cache[(key, 'exact')] = w
            if form != 'exact':
                self.cache[(key, form)] = _round(w, SPLIT_WEIGHT_SCALE, form == 'hi')
        return self.cache[(key, form)]


def folded_sites(cfg):
    """The launches whose operands forward_folded rounds, by the tag launch_plan gives them without its group prefix: the six conv GEMMs,
    the projection, the positional conv and per layer the QKV GEMM, attention, out_proj, FFN in and FFN out."""
    layers = [f'l{j}.{n}' for j in range(cfg['num_hidden_layers']) for n in ('qkv', 'attn', 'out', 'ffn1', 'ffn2')]
    return [f'conv{i}' for i in range(1, 7)] + ['proj', 'pos'] + layers


def _attention(qkv, L, H, heads, ops, tag):
    """softmax(q k^T) v per head as the kernel computes it: P = exp(s - max) split after scaling by 2^10, P v divided by the row sum."""
    qkv = ops.x(tag, qkv)
    q, k, v = (qkv[:, j * H:(j + 1) * H].view(L, heads, 64).transpose(0, 1) for j in range(3))
    s = q @ k.transpose(1, 2)
    p = torch.exp(s - s.amax(-1, keepdim=True))
    o = (ops.x(tag, p, P_SCALE) @ v) / p.sum(-1, keepdim=True)
    return o.transpose(0, 1).reshape(L, H)


def forward_folded(P, cfg, x, segs=None, operands='exact', site=None):
    """The same network on real3dportrait_b200.hubert.fold_weights(model) (float64), in the kernels' order: conv windows as GEMMs over K
    channel j Cp + i, LayerNorms that only standardise where their gamma / beta were folded, the pos conv as a GEMM over tap-major K on each
    segment with its own zero padding, one QKV GEMM.  segs: encoder segment lengths (default: one segment).
    operands / site: how each GEMM, attention and positional-conv launch reads its operands (_Operands); an unknown site raises."""
    from real3dportrait_b200.hubert import conv_gemm_weight, pos_gemm_weight
    if site is not None and site not in folded_sites(cfg):
        raise ValueError(f'no launch {site!r} reads GEMM, attention or positional-conv operands')
    ops = _Operands(operands, site, P.setdefault('_rounded', {}))
    H, heads, eps = cfg['hidden_size'], cfg['num_attention_heads'], cfg.get('layer_norm_eps', 1e-5)
    w0, b0, l0 = P['conv'][0]
    n = (x.shape[0] - 10) // 5 + 1
    win = torch.stack([x[5 * f:5 * f + 10] for f in range(n)]) if n < 4096 else x.unfold(0, 10, 5)
    h = win @ w0[:, 0, :].t() + (0 if b0 is None else b0)
    h = gelu(ln(h, l0.weight.detach().double(), l0.bias.detach().double(), l0.eps))
    C = h.shape[1]
    Cp = (C + 63) // 64 * 64
    for i in range(1, 7):
        w, b, l = P['conv'][i]
        k, s = KERNELS[i], STRIDES[i]
        hp = torch.zeros(h.shape[0], Cp, dtype=torch.float64)
        hp[:, :C] = h
        rows = hp.unfold(0, k, s).permute(0, 2, 1).reshape(-1, k * Cp)
        tag = f'conv{i}'
        h = ops.x(tag, rows) @ ops.w(tag, tag, lambda: conv_gemm_weight(w, Cp)).t() + (0 if b is None else b)
        h = gelu(ln(h, l.weight.detach().double(), l.bias.detach().double(), l.eps))
    if cfg.get('feat_proj_layer_norm', True):
        h = ln(h, eps=eps)
    h = ops.x('proj', h) @ ops.w('proj', 'proj', lambda: P['proj'][0]).t() + P['proj'][1]
    T = h.shape[0]
    segs = segs or [T]
    wp = ops.w('pos', 'pos', lambda: pos_gemm_weight(P['pos'][0]))
    G = H // 64
    out = []
    s0 = 0
    for L in segs:
        hs = h[s0:s0 + L]
        pad = torch.zeros(L + 128, H, dtype=torch.float64)
        pad[64:64 + L] = ops.x('pos', hs)
        pc = torch.empty(L, H, dtype=torch.float64)
        for g in range(G):
            cols = pad[:, 64 * g:64 * g + 64].unfold(0, 128, 1)[:L]            # [L, 64, 128]: window t = frames t - 64 .. t + 63
            pc[:, 64 * g:64 * g + 64] = cols.permute(0, 2, 1).reshape(L, -1) @ wp[64 * g:64 * g + 64].t()
        hs = hs + gelu(pc + P['pos'][1])
        for j, (wq, bq, wo, bo, w1, b1, w2, b2) in enumerate(P['layers']):
            t = f'l{j}.'
            gemm = lambda site, a, w, b: ops.x(t + site, a) @ ops.w(t + site, t + site, lambda: w).t() + b   # noqa: E731
            qkv = gemm('qkv', ln(hs, eps=eps), wq, bq)
            hs = hs + gemm('out', _attention(qkv, L, H, heads, ops, t + 'attn'), wo, bo)
            hs = hs + gemm('ffn2', gelu(gemm('ffn1', ln(hs, eps=eps), w1, b1)), w2, b2)
        lf = P['ln_f']
        out.append(ln(hs, lf.weight.detach().double(), lf.bias.detach().double(), lf.eps))
        s0 += L
    return torch.cat(out)


#: the hubert-large-ls960-ft architecture (transformers' config keys)
LARGE = dict(conv_dim=(512,) * 7, hidden_size=1024, num_attention_heads=16, intermediate_size=4096, num_hidden_layers=24,
             num_conv_pos_embeddings=128, num_conv_pos_embedding_groups=16, feat_extract_norm='layer', do_stable_layer_norm=True,
             conv_bias=True)


def small_config():
    """The config of the fixture tests/golden/hubert_small.npz: conv_dim 32 (Cp 64), H 128 in 2 heads, I 256, 2 layers."""
    import os
    import numpy as np
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'hubert_small.npz'))
    return {k[7:]: (tuple(z[k].tolist()) if z[k].ndim else z[k].item()) for k in z.files if k.startswith('config.')}


def formula_model(cfg):
    """HubertModel(cfg) with formula_params weights (fp32, CPU) and those parameters in float64."""
    from real3dportrait_b200 import HubertModel
    m = HubertModel(cfg)
    sd = formula_params({k: tuple(v.shape) for k, v in m.state_dict().items()})
    m.load_state_dict({k: v.float() for k, v in sd.items()}, strict=True)
    return m, sd


def frames(L):
    return (L - 80) // 320


def segments(T):
    return [min(1000, T - s) for s in range(0, T, 1000)]


def get_hubert(sd, cfg, speech):
    """extract_hubert.py's chunk loop in float64: normalise the clip, encode 1000-frame chunks (320080 samples) one by one."""
    x = normalise(speech)
    L = x.shape[0]
    clip = 320 * 1000
    res = []
    for i in range(L // clip):
        res.append(forward_unfolded(sd, cfg, x[clip * i:clip * i + clip - 320 + 400]))
    rest = x[clip * (L // clip):]
    if rest.shape[0] >= 400:
        res.append(forward_unfolded(sd, cfg, rest))
    return torch.cat(res)[:frames(L)]


def formula_params(shapes):
    """Deterministic parameters from a formula (no RNG, nothing stored): LayerNorm gamma around 1 and beta != 0, positive weight-norm g,
    other tensors ~ 1/sqrt(fan_in).  shapes: {name: shape} -> {name: float64 tensor}."""
    out = {}
    for j, (k, shp) in enumerate(sorted(shapes.items())):
        n = int(torch.tensor(shp).prod()) if len(shp) else 1
        i = torch.arange(n, dtype=torch.float64)
        u = torch.sin(i * 0.7548776662 + 1.3 * j + 0.1) * torch.cos(i * 0.0137 + 0.37 * j)
        if k.endswith('layer_norm.weight'):
            t = 1 + 0.2 * u
        elif k.endswith('original0') or k.endswith('weight_g'):
            t = 0.5 + 0.5 * u.abs()
        else:
            fan = shp[1] * (shp[2] if len(shp) > 2 else 1) if len(shp) > 1 else 25
            t = 1.7 * u / math.sqrt(fan)
        out[k] = t.reshape(shp)
    return out


def wave(L):
    """The fixture's formula waveform (float32 numpy)."""
    import numpy as np
    t = np.arange(L, dtype=np.float64)
    return (0.3 * np.sin(2 * np.pi * 220 * t / 16000) + 0.2 * np.sin(2 * np.pi * 37.5 * t / 16000 + 0.4)
            + 0.05 * np.sin(t * t * 1e-7) + 0.01).astype(np.float32)


# ---- the library's launch sequence, restated from the architecture ----------------------------------------------------------------------
SEG, GROUP = 1000, 4                        # frames per encoder segment; segments per launch group (DESIGN.md "Audio features")


def groups(T):
    """[(first frame, segment lengths)] of the launch groups of a T-frame clip: GROUP consecutive SEG-frame segments each."""
    segs = segments(T)
    return [(g * SEG, segs[g:g + GROUP]) for g in range(0, len(segs), GROUP)]


def launch_plan(cfg, L, B=None, ldo=None):
    """Every kernel launch of get_hubert_from_16k_speech on an L-sample clip (B None) or of HubertModel.forward on [B, L] inputs, as
    (tag, C entry point, the non-pointer arguments in C order), written from the architecture and DESIGN.md's launch sequence rather than
    from the module's code.  ldo: the row stride of the output (default H, a contiguous [T, H]).  Tags: 'stats', then per group g (per item
    b of forward: 'b{b}.') 'g{g}.conv0', 'g{g}.conv{i}' and its LayerNorm 'g{g}.conv{i}.ln', 'g{g}.proj.ln', 'g{g}.proj', 'g{g}.split',
    'g{g}.pos', per layer j 'g{g}.l{j}.ln1 / qkv / attn / out / ln2 / ffn1 / ffn2' and 'g{g}.ln_f'.  Split rows are [hi | lo] with the lo
    half at Cp (conv_dim C rounded up to 64, the pad channels zero) or at the row's width; attention's segment lengths appear as a tuple.
      conv0            normalise, k10 s5 conv 1 -> C, LayerNorm + GELU -> split rows [F, 2 Cp]
      conv1..6         GEMM over the previous rows read in place as windows (k frames, stride s frames) -> fp32 [F', C] (epilogue 3), then
                       a LayerNorm + GELU -> split rows; conv6's LayerNorm runs in place in fp32 when feat_proj_layer_norm
      proj.ln, proj    the projection's LayerNorm (standardise only, gamma / beta folded) -> split rows; GEMM -> fp32 h [Fg, H]
      split, pos       h -> split rows of the segment-padded copy; the positional conv adds GELU(conv + b) into h (epilogue in the kernel)
      l{j}             LayerNorm -> split; QKV GEMM -> split [Fg, 6H] (lo at 3H); attention -> split; out_proj into h (epilogue 2);
                       LayerNorm; FFN in with GELU -> split [Fg, 2I]; FFN out into h
      ln_f             the encoder's LayerNorm -> fp32 rows of the output"""
    C, H, I = cfg['conv_dim'][0], cfg['hidden_size'], cfg['intermediate_size']
    Cp = (C + 63) // 64 * 64
    eps = float(cfg.get('layer_norm_eps', 1e-5))
    ceps = 1e-5                                                           # the conv layers' LayerNorms: nn.LayerNorm's default eps
    fpln = cfg.get('feat_proj_layer_norm', True)
    heads = cfg['num_attention_heads']
    ldo = ldo or H
    plan = []

    def add(tag, fn, *args):
        plan.append((tag, fn, tuple(args)))

    def gemm(tag, M, K, N, epi, ldy, ylo, window=1, stride=1, seg=None):
        seg = seg or K
        add(tag, 'r3dp_hb_gemm', M, window * 2 * seg, stride * 2 * seg, seg, N, window * seg if window > 1 else K, epi, ldy, ylo)

    def group(p, segs):
        Fg = sum(segs)
        F = (320 * (Fg - 1) + 400 - 10) // 5 + 1
        add(p + 'conv0', 'r3dp_hb_conv0', F, C, ceps, 2 * Cp, Cp)
        for i in range(1, 7):
            k, s = KERNELS[i], STRIDES[i]
            F = (F - k) // s + 1
            gemm(f'{p}conv{i}', F, Cp, C, 3, C, 0, window=k, stride=s)
            if i < 6 or not fpln:
                add(f'{p}conv{i}.ln', 'r3dp_hb_layernorm', F, C, ceps, 1, 0, 2 * Cp, Cp)
            else:
                add(f'{p}conv{i}.ln', 'r3dp_hb_layernorm', F, C, ceps, 1, C, 0, 0)
        assert F == Fg, (F, Fg)
        if fpln:
            add(p + 'proj.ln', 'r3dp_hb_layernorm', Fg, C, eps, 0, 0, 2 * Cp, Cp)
        gemm(p + 'proj', Fg, Cp, H, 3, H, 0)
        add(p + 'split', 'r3dp_a2m_split', Fg, H)
        add(p + 'pos', 'r3dp_hb_pos_conv', len(segs), max(segs), Fg, H)
        for j in range(cfg['num_hidden_layers']):
            t = f'{p}l{j}.'
            add(t + 'ln1', 'r3dp_hb_layernorm', Fg, H, eps, 0, 0, 2 * H, H)
            gemm(t + 'qkv', Fg, H, 3 * H, 0, 6 * H, 3 * H)
            add(t + 'attn', 'r3dp_hb_attention', Fg, 6 * H, 3 * H, heads, tuple(segs), len(segs), 2 * H, H)
            gemm(t + 'out', Fg, H, H, 2, H, 0)
            add(t + 'ln2', 'r3dp_hb_layernorm', Fg, H, eps, 0, 0, 2 * H, H)
            gemm(t + 'ffn1', Fg, H, I, 1, 2 * I, I)
            gemm(t + 'ffn2', Fg, I, H, 2, H, 0)
        add(p + 'ln_f', 'r3dp_hb_layernorm', Fg, H, eps, 0, ldo, 0, 0)

    if B is None:
        add('stats', 'r3dp_hb_stats', L)
        for g, (_, segs) in enumerate(groups(frames(L))):
            group(f'g{g}.', segs)
    else:
        T = (L - 400) // 320 + 1
        for b in range(B):
            group(f'b{b}.', [T])
    return plan


#: the launches that read rounded operands (forward_folded's sites)
SITE_LAUNCHES = ('r3dp_hb_gemm', 'r3dp_hb_attention', 'r3dp_hb_pos_conv')


def site_of(tag, fn):
    """The forward_folded site of a plan launch ('g1.l23.ffn2' -> 'l23.ffn2'), None for a launch without rounded operands."""
    return tag.split('.', 1)[1] if fn in SITE_LAUNCHES else None
