"""Audio-to-motion (PitchContourVAEModel, the released audio2motion_vae config) on the H100: forward time against the same network in eager
PyTorch, launches per forward, and the fused WaveNet layer's rate on the decoder shape.

    python tools/bench_audio2motion.py [--out DIR]

Reports, with the card's name, power limit and clocks read in the same call:
  - forward at T_x = 500, 3000 and 30000 (10 s, 1 min, 10 min of 50 Hz features), B = 1, against the network run eagerly in PyTorch on
    cuDNN (tests/audio2motion_reference.py on fp32 CUDA tensors) at torch's default TF32 setting; the arms alternate, median of 3 windows;
  - CUDA kernels the library launches per forward (r3dp_launch_count);
  - r3dp_a2m_wn_layer alone on the decoder shape (hidden 256, k 5, a middle layer) at T = 15000: its time and algorithmic TFLOP/s,
    2 T (2H H k + 2H H) operations per layer (the split-fp16 form issues three MMAs per product; they are not counted).
Parameters are the seeded synthetic set of the tests; times do not depend on their values."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import audio2motion_reference as ref  # noqa: E402
import real3dportrait_b200 as r3  # noqa: E402
from real3dportrait_b200 import _capi as capi  # noqa: E402
from real3dportrait_b200.audio2motion import pack_wn_layer  # noqa: E402

DEV = 'cuda:0'


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    r = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader'], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else 'not read'


def timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_audio2motion: no CUDA device')
    torch.set_grad_enabled(False)
    torch.backends.cudnn.allow_tf32 = True                            # torch's defaults
    torch.backends.cuda.matmul.allow_tf32 = False
    m = r3.PitchContourVAEModel(ref.HP_PITCH)
    sd = ref.make_params({k: v.shape for k, v in m.state_dict().items()}, 11)
    m.load_state_dict(sd, strict=True)
    m = m.to(DEV).eval()
    sd32 = {k: v.to(DEV) for k, v in sd.items()}
    res = {'card': card(), 'forward': []}
    L = capi.lib()
    for Tx in (500, 3000, 30000):
        Tp = (Tx + 7) // 8 * 8                                          # get_hubert pads to a multiple of 8
        batch = {k: v.to(DEV) for k, v in ref.make_batch(1, Tp, 1024, seed=Tp).items()}
        z = torch.randn(1, 16, Tp // 8, generator=torch.Generator().manual_seed(1)).to(DEV)
        ours = lambda: m(batch, {}, temperature=0.2, z=z)                                           # noqa: E731
        eager = lambda: ref.forward(sd32, batch, z, 0.2, dt=torch.float32)                          # noqa: E731
        reps = 20 if Tp <= 3000 else 3
        for f in (ours, eager):
            f()
        n0 = L.r3dp_launch_count()
        ours()
        launches = int(L.r3dp_launch_count() - n0)
        t_ours, t_eager = [], []
        for _ in range(3):
            t_ours.append(timed(ours, reps))
            t_eager.append(timed(eager, reps))
        err = float((ours() - eager()).abs().max())
        row = {'T_x': Tp, 'ms_library': statistics.median(t_ours), 'ms_eager_pytorch': statistics.median(t_eager),
               'speedup': statistics.median(t_eager) / statistics.median(t_ours), 'launches_per_forward': launches,
               'max_abs_diff_vs_eager_fp32': err}
        res['forward'].append(row)
        print(json.dumps(row), flush=True)
    # the fused WaveNet layer on the decoder shape
    H, k, T = 256, 5, 15000
    g = torch.Generator().manual_seed(0)
    x = torch.randn(T, H, generator=g).to(DEV)
    xo, skip = torch.empty_like(x), torch.randn(T, H, generator=g).to(DEV)
    cond = torch.randn(T, 2048, generator=g).to(DEV)
    w = pack_wn_layer(torch.randn(2 * H, H, k, dtype=torch.float64) * 0.03, torch.randn(2 * H, H, dtype=torch.float64) * 0.05).to(DEV)
    bias = torch.zeros(2 * H, device=DEV)

    def layer():
        capi.check(L.r3dp_a2m_wn_layer(capi.ptr(x), capi.ptr(xo), capi.ptr(cond), 2048, capi.ptr(w, torch.float16), capi.ptr(bias), capi.ptr(skip),
                                       None, 1, T, H, k, 0, 0, capi.stream()))
    layer()
    t = statistics.median(timed(layer, 50) for _ in range(3))
    flops = 2.0 * T * (2 * H * H * k + 2 * H * H)
    res['wn_layer_decoder'] = {'T': T, 'ms': t, 'tflops_algorithmic': flops / (t * 1e-3) / 1e12}
    print(json.dumps(res['wn_layer_decoder']), flush=True)
    print(json.dumps({'card': res['card']}))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_audio2motion.json'), 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
