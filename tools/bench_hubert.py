"""HuBERT feature extraction on the library against the reference's way of running it (transformers' HubertModel, 20 s chunks one by one,
fp32, torch's default TF32 flags; without transformers, the float32 restatement in eager PyTorch on the GPU, labelled as such).
hubert-large shapes, formula weights, synthetic 10 s / 1 min / 10 min clips; median of 3 alternating windows after a warm-up of every shape.
Also: r3dp_hb_gemm's and r3dp_hb_attention's algorithmic TFLOP/s (2MNK, not counting the split's three MMAs), the clip statistics' time and the peak extra memory
at 10 min.  `--weights DIR`: a local hubert-large snapshot, compared against transformers on a clip.
Usage: python tools/bench_hubert.py [--clips 10,60,600] [--weights DIR]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from real3dportrait_b200 import _capi as capi  # noqa: E402
from real3dportrait_b200 import hubert as hb  # noqa: E402
from real3dportrait_b200 import HubertModel, get_hubert_from_16k_speech  # noqa: E402
import hubert_reference as hr  # noqa: E402

LARGE = dict(conv_dim=(512,) * 7, hidden_size=1024, num_attention_heads=16, intermediate_size=4096, num_hidden_layers=24,
             num_conv_pos_embeddings=128, num_conv_pos_embedding_groups=16, feat_extract_norm='layer', do_stable_layer_norm=True,
             conv_bias=True)


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
        return q.stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def timed(fn, reps=1):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def eager_arm(sd):
    """transformers' HubertModel if importable, else the float32 restatement (eager PyTorch): the reference's chunk loop."""
    try:
        import transformers
        m = transformers.HubertModel(transformers.HubertConfig(**LARGE)).eval()
        m.load_state_dict({k: v.float() for k, v in sd.items()}, strict=True)
        m = m.cuda()
        label = f'transformers {transformers.__version__} HubertModel, fp32 eager, 20 s chunks'

        def enc(x):
            return m(x[None]).last_hidden_state[0]
    except ImportError:
        sdf = {k: v.float().cuda() for k, v in sd.items()}
        label = 'float32 restatement in eager PyTorch (transformers not importable), 20 s chunks'

        def enc(x):
            return _f32_forward(sdf, x)

    @torch.no_grad()
    def run(wave):
        x = wave.cuda().float()
        x = (x - x.mean()) / torch.sqrt(x.var(unbiased=False) + 1e-7)
        L, clip, res = x.shape[0], 320000, []
        for i in range(L // clip):
            res.append(enc(x[clip * i:clip * i + clip + 80]))
        if L - clip * (L // clip) >= 400:
            res.append(enc(x[clip * (L // clip):]))
        return torch.cat(res)[:(L - 80) // 320].cpu()
    return run, label


def _f32_forward(sd, x):
    # hubert_reference.forward_unfolded promotes to float64; this arm keeps the reference's fp32
    import torch.nn.functional as Fn
    H, heads, eps = 1024, 16, 1e-5
    h = x[None, None]
    for i in range(7):
        p = f'feature_extractor.conv_layers.{i}.'
        h = Fn.conv1d(h, sd[p + 'conv.weight'], sd.get(p + 'conv.bias'), stride=hr.STRIDES[i])
        h = Fn.gelu(Fn.layer_norm(h.transpose(1, 2), (h.shape[1],), sd[p + 'layer_norm.weight'], sd[p + 'layer_norm.bias']).transpose(1, 2))
    h = Fn.layer_norm(h[0].t(), (512,), sd['feature_projection.layer_norm.weight'], sd['feature_projection.layer_norm.bias'], eps)
    h = Fn.linear(h, sd['feature_projection.projection.weight'], sd['feature_projection.projection.bias'])
    pc = Fn.conv1d(h.t()[None], hr.pos_weight(sd).float(), sd['encoder.pos_conv_embed.conv.bias'], padding=64, groups=16)[0, :, :-1]
    h = h + Fn.gelu(pc.t())
    T = h.shape[0]
    for li in range(24):
        p = f'encoder.layers.{li}.'
        a = Fn.layer_norm(h, (H,), sd[p + 'layer_norm.weight'], sd[p + 'layer_norm.bias'], eps)
        lin = lambda n, z: Fn.linear(z, sd[p + n + '.weight'], sd[p + n + '.bias'])   # noqa: E731
        q, k, v = (lin(f'attention.{n}_proj', a).view(T, heads, 64).transpose(0, 1) for n in 'qkv')
        o = Fn.scaled_dot_product_attention(q[None], k[None], v[None])[0]
        h = h + lin('attention.out_proj', o.transpose(0, 1).reshape(T, H))
        f = Fn.layer_norm(h, (H,), sd[p + 'final_layer_norm.weight'], sd[p + 'final_layer_norm.bias'], eps)
        h = h + lin('feed_forward.output_dense', Fn.gelu(lin('feed_forward.intermediate_dense', f)))
    return Fn.layer_norm(h, (H,), sd['encoder.layer_norm.weight'], sd['encoder.layer_norm.bias'], eps)


def kernel_rates():
    L, st = capi.lib(), capi.stream()
    out = {}
    M = 4000
    for name, N, K, epi in (('ffn_in', 4096, 1024, 1), ('ffn_out', 1024, 4096, 2), ('qkv', 3072, 1024, 0), ('out_proj', 1024, 1024, 2)):
        A = torch.randn(M, 2 * K, device='cuda').half()
        wp = hb.pack_split(torch.randn(N, K, dtype=torch.float64) / K ** 0.5).cuda()
        b = torch.zeros(N, device='cuda')
        y = torch.zeros(M, 2 * N if epi < 2 else N, device='cuda', dtype=torch.float16 if epi < 2 else torch.float32)

        def f():
            capi.check(L.r3dp_hb_gemm(capi.ptr(A, torch.float16), M, 2 * K, 2 * K, K, capi.ptr(wp, torch.float16), N, K, capi.ptr(b), epi,
                                      ctypes.c_void_p(y.data_ptr()), y.shape[1], N if epi < 2 else 0, st))
        f()
        ms = timed(f, 50)
        out[f'gemm_{name}_M{M}'] = {'ms': round(ms, 4), 'tflops': round(2 * M * N * K / ms / 1e9, 1)}
    segs = [1000] * 4
    R = sum(segs)
    qkv = torch.randn(R, 6144, device='cuda').half()
    o = torch.empty(R, 2048, device='cuda', dtype=torch.float16)
    lens = (ctypes.c_int * 4)(*segs)

    def fa():
        capi.check(L.r3dp_hb_attention(capi.ptr(qkv, torch.float16), R, 6144, 3072, 16, lens, 4, capi.ptr(o, torch.float16), 2048, 1024, st))
    fa()
    ms = timed(fa, 50)
    out['attention_4x1000'] = {'ms': round(ms, 4), 'tflops': round(4 * 4 * 1000 * 1000 * 1024 / ms / 1e9, 1)}
    # the clip statistics: one CTA, two fp64 passes over a 10-minute clip
    x = torch.randn(16000 * 600, device='cuda')
    stats = torch.empty(2, dtype=torch.float64, device='cuda')

    def fs():
        capi.check(L.r3dp_hb_stats(capi.ptr(x), x.numel(), capi.ptr(stats, torch.float64), st))
    fs()
    out['stats_10min'] = {'ms': round(timed(fs, 20), 4)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--clips', default='10,60,600')
    ap.add_argument('--weights', default=None)
    args = ap.parse_args()
    torch.backends.cudnn.benchmark = False
    print(json.dumps({'card': card()}))
    m = HubertModel(LARGE)
    sd = hr.formula_params({k: tuple(v.shape) for k, v in m.state_dict().items()})
    m.load_state_dict({k: v.float() for k, v in sd.items()}, strict=True)
    m = m.cuda()
    eager, label = eager_arm(sd)
    res = {'eager_arm': label, 'clips': {}}
    for sec in [int(s) for s in args.clips.split(',')]:
        wave = torch.from_numpy(hr.wave(16000 * sec))
        lib = lambda: get_hubert_from_16k_speech(wave, m)    # noqa: E731
        ref = lambda: eager(wave)                            # noqa: E731
        a, b = lib(), ref()
        err = float((a.cpu() - b).abs().max()) / float(b.abs().max())
        tl, te = [], []
        for _ in range(3):
            tl.append(timed(lib))
            te.append(timed(ref))
        tl.sort(), te.sort()
        res['clips'][f'{sec}s'] = {'library_ms': round(tl[1], 2), 'eager_ms': round(te[1], 2), 'speedup': round(te[1] / tl[1], 2),
                                   'max_rel_diff_vs_eager': float(f'{err:.2e}')}
        if sec == max(int(s) for s in args.clips.split(',')):
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            lib()
            torch.cuda.synchronize()
            res['clips'][f'{sec}s']['library_peak_extra_MB'] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
        print(json.dumps({f'{sec}s': res['clips'][f'{sec}s']}), flush=True)
    res['kernels'] = kernel_rates()
    if args.weights:
        import transformers
        mt = transformers.HubertModel.from_pretrained(args.weights).cuda().eval()
        ml = HubertModel.from_pretrained(args.weights).cuda()
        x = torch.from_numpy(hr.wave(16000 * 30))
        xn = ((x - x.mean()) / torch.sqrt(x.var(unbiased=False) + 1e-7)).cuda()
        with torch.no_grad():
            r = mt(xn[None, :320080]).last_hidden_state[0]
        g = ml(xn[None, :320080]).last_hidden_state[0]
        res['weights_max_rel_diff'] = float((g - r).abs().max() / r.abs().max())
    print(json.dumps(res))


if __name__ == '__main__':
    main()
