"""Canonical plane backbone (Img2PlaneModel) on the H100: time, per-stage split, the attention kernel, and time to a clip's first frame.

    python tools/bench_img2plane.py [--out DIR]

Reports, with the card's name, power limit and clocks read in the same call:
  - forward at 512^2, B = 1 (the engine's case) and B = 4, against the same network in PyTorch (tests/img2plane_reference.py on fp32
    CUDA tensors) at torch's default TF32 setting (cuDNN convolutions TF32, matmuls fp32) and with TF32 off; the arms alternate, median of 3;
  - a per-stage split from CUDA events around the library's regions (a separate, profiled run), and r3dp_ip_attention alone at
    (Tq, Tk) = (16384, 4096) with its algorithmic TFLOP/s (4 * B * heads * Tq * Tk * 256 operations);
  - begin_planes(img=...) + the first step of a warm engine, against the PyTorch backbone + canonical_planes_cl + begin_planes(cano_planes)
    + the same step.
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

import img2plane_reference as iref  # noqa: E402
import secc2plane_reference as sref  # noqa: E402
import real3dportrait_b200 as r3  # noqa: E402
from real3dportrait_b200 import _capi as capi, engine, synthetic as syn  # noqa: E402

DEV = 'cuda:0'


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    r = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader'], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else 'not read'


def timed(fn, reps=1):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def tf32(on):
    torch.backends.cudnn.allow_tf32 = on
    torch.backends.cuda.matmul.allow_tf32 = False                    # torch's default either way


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    res = {'card': card()}
    m = r3.Img2PlaneModel()
    sd = iref.make_params({k: v.shape for k, v in m.state_dict().items()}, 5)
    m.load_state_dict(sd, strict=True)
    m = m.to(DEV).eval()
    sd32 = {k: v.to(DEV) for k, v in sd.items()}

    for B in (1, 4):
        x = iref.make_inputs(B, 512, 11).to(DEV)
        arms = {'cuda': lambda: m(x), 'torch_tf32_default': lambda: iref.forward(sd32, x), 'torch_tf32_off': lambda: iref.forward(sd32, x)}
        times = {k: [] for k in arms}
        for k, f in arms.items():                                    # warm-up: module loads, cuDNN algorithm choice
            tf32(k != 'torch_tf32_off')
            f()
        for _ in range(3):
            for k, f in arms.items():
                tf32(k != 'torch_tf32_off')
                times[k].append(timed(f))
        tf32(True)
        res[f'forward_B{B}_ms'] = {k: statistics.median(v) for k, v in times.items()}
        print(f'forward 512^2 B={B}: ' + ', '.join(f'{k} {statistics.median(v):.2f} ms' for k, v in times.items()), flush=True)

    # per-stage split (profiled run)
    x = iref.make_inputs(1, 512, 11).to(DEV)
    capi.PROF = capi.Profiler()
    m(x)
    split = capi.PROF.totals()
    capi.PROF = None
    res['stages_B1_ms'] = split
    print('stages (B=1): ' + ', '.join(f'{k} {v:.2f}' for k, v in sorted(split.items())), flush=True)

    # the attention kernel alone at the TriplanePredictorViT shape
    for B in (1, 4):
        Tq, Tk = 16384, 4096
        q = torch.randn(B, Tq, 1024, device=DEV).half()
        kv = torch.randn(B, Tk, 2048, device=DEV).half()
        o = torch.empty(B, Tq, 1024, device=DEV, dtype=torch.float16)
        call = lambda: capi.check(capi.lib().r3dp_ip_attention(capi.ptr(q, torch.float16), 1024, capi.ptr(kv, torch.float16), 2048, B, Tq, Tk,  # noqa: E731
                                                               4, 1.0 / 16.0, capi.ptr(o, torch.float16), 1024, capi.stream()))
        call()
        ms = timed(call, 20)
        tflops = 4.0 * B * 4 * Tq * Tk * 256 / (ms * 1e-3) / 1e12
        res[f'attention_B{B}'] = {'ms': ms, 'tflops': tflops}
        print(f'attention (16384, 4096) B={B}: {ms:.3f} ms, {tflops:.0f} TFLOP/s', flush=True)

    # time from begin_planes(img=...) to the first finished frame, warm engine
    eng = engine.FrameEngine(batch=4, sr_mode='tc', hp={'num_samples_fine': 0}, out_uint8=True,
                             secc2plane=r3.SegFormerSECC2PlaneBackbone(), img2plane=m)
    eng.secc.load_state_dict(sref.make_params({k: v.shape for k, v in eng.secc.state_dict().items()}, 7), strict=True)
    eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_params(seed=5))
    cano, src, tgt = (t.to(DEV) for t in sref.make_inputs(4, 512, 3))
    cams = syn.make_cameras(4, seed=1).to(DEV)
    u_c = syn.make_jitter(4, 4096, 48, 0, seed=2)[0].to(DEV)
    img = iref.make_inputs(1, 512, 21).to(DEV)

    def start_cuda():
        eng.begin_planes(img=img, cond_cano=cano, cond_src=src)
        eng.step(None, cams, u_c, cond_tgt=tgt)

    def start_torch():
        tf32(True)
        planes = iref.forward(sd32, img)
        eng.begin_planes(planes, cano, src)                          # canonical_planes_cl inside
        eng.step(None, cams, u_c, cond_tgt=tgt)

    start_cuda()
    start_torch()
    t = {'cuda': [], 'torch': []}
    for _ in range(3):
        t['cuda'].append(timed(start_cuda))
        t['torch'].append(timed(start_torch))
    res['first_frame_ms'] = {k: statistics.median(v) for k, v in t.items()}
    print('begin_planes -> first frame: ' + ', '.join(f'{k} {statistics.median(v):.2f} ms' for k, v in t.items()), flush=True)
    print('card: ' + res['card'])
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_img2plane.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
