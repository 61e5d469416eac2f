"""Float64 restatements of HuBERT (transformers' HubertModel, hubert-large architecture) and of extract_hubert.py's chunking, written from
the architecture: `forward_unfolded` as transformers writes it (from a state_dict), `forward_folded` on real3dportrait_b200.hubert's folded
weights in the kernels' layouts (GEMM rows, the conv windows' K order, the pos conv's tap-major K order), without the fp16 split."""
import math

import torch
import torch.nn.functional as Fn

KERNELS, STRIDES = (10, 3, 3, 3, 3, 2, 2), (5, 2, 2, 2, 2, 2, 2)


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


def forward_folded(P, cfg, x, segs=None):
    """The same network on real3dportrait_b200.hubert.fold_weights(model) (float64), in the kernels' order: conv windows as GEMMs over K
    channel j Cp + i, LayerNorms that only standardise where their gamma / beta were folded, the pos conv as a GEMM over tap-major K on each
    segment with its own zero padding, one QKV GEMM.  segs: encoder segment lengths (default: one segment)."""
    from real3dportrait_b200.hubert import conv_gemm_weight, pos_gemm_weight
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
        h = rows @ conv_gemm_weight(w, Cp).t() + (0 if b is None else b)
        h = gelu(ln(h, l.weight.detach().double(), l.bias.detach().double(), l.eps))
    if cfg.get('feat_proj_layer_norm', True):
        h = ln(h, eps=eps)
    h = h @ P['proj'][0].t() + P['proj'][1]
    T = h.shape[0]
    segs = segs or [T]
    wp = pos_gemm_weight(P['pos'][0])
    G = H // 64
    out = []
    s0 = 0
    for L in segs:
        hs = h[s0:s0 + L]
        pad = torch.zeros(L + 128, H, dtype=torch.float64)
        pad[64:64 + L] = hs
        pc = torch.empty(L, H, dtype=torch.float64)
        for g in range(G):
            cols = pad[:, 64 * g:64 * g + 64].unfold(0, 128, 1)[:L]            # [L, 64, 128]: window t = frames t - 64 .. t + 63
            pc[:, 64 * g:64 * g + 64] = cols.permute(0, 2, 1).reshape(L, -1) @ wp[64 * g:64 * g + 64].t()
        hs = hs + gelu(pc + P['pos'][1])
        for wq, bq, wo, bo, w1, b1, w2, b2 in P['layers']:
            qkv = ln(hs, eps=eps) @ wq.t() + bq
            q, k, v = (qkv[:, j * H:(j + 1) * H].view(L, heads, 64).transpose(0, 1) for j in range(3))
            o = torch.softmax(q @ k.transpose(1, 2), -1) @ v
            hs = hs + o.transpose(0, 1).reshape(L, H) @ wo.t() + bo
            hs = hs + gelu(ln(hs, eps=eps) @ w1.t() + b1) @ w2.t() + b2
        lf = P['ln_f']
        out.append(ln(hs, lf.weight.detach().double(), lf.bias.detach().double(), lf.eps))
        s0 += L
    return torch.cat(out)


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
