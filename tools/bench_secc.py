"""Time SegFormerSECC2PlaneBackbone (MiT-b0, 512^2 SECC input, batch 4) on one GPU: this library against PyTorch running the same module
(the float64-checked restatement tests/secc2plane_reference.py in fp32 nn ops), with torch's default TF32 setting and with TF32 off.
Arms alternate; each figure is the median of 3 windows of CUDA-event time.  Prints the card, its power limit and SM clock samples.
Also: per-launch times of the conv stack (a profiled pass of its own), and the clip step at batch 4 with uint8 frames in three arms:
  resident   FrameEngine fed resident planes (the headline workload's step; no backbone)
  torch      the PyTorch backbone, then FrameEngine on the (canonical, secc) pair (what a user pays without this library's backbone)
  engine     FrameEngine(secc2plane=...): backbone and render in one CUDA graph

    python tools/bench_secc.py [--batch 4] [--iters 20]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]
import secc2plane_reference as ref  # noqa: E402
import real3dportrait_b200 as r3  # noqa: E402
from real3dportrait_b200 import _capi as capi, engine, synthetic as syn  # noqa: E402


def gflop(H):
    """Algorithmic FLOPs of one frame (2 per MAC), counted from the shapes of SegFormerSECC2PlaneBackbone('b0') at H x H, unfolded head."""
    f, h = 0, H // 4
    f += 2 * 9 * 3 * H * H + 2 * 3 * 49 * 32 * h * h                      # prenet, patch_embed1
    cin = 3
    for s, (C, sr) in enumerate(zip(ref.EMBED, ref.SR)):
        if s > 0:
            h //= 2
            f += 2 * 9 * cin * C * h * h
        T, Tk = h * h, (h // sr) ** 2
        for _ in range(2):
            f += 2 * T * C * C * 2                                        # q, proj
            if sr > 1:
                f += 2 * Tk * sr * sr * C * C                             # sr conv
            f += 2 * Tk * C * 2 * C                                       # kv
            f += 2 * 2 * T * Tk * C                                       # QK^T, PV
            f += 2 * 2 * T * C * 4 * C + 2 * 9 * 4 * C * T                # fc1, fc2, dwconv
        cin = C
    h1 = H // 4
    f += sum(2 * (H // 2 ** (i + 2)) ** 2 * C * 256 for i, C in enumerate(ref.EMBED))   # linear_c*
    f += 2 * h1 * h1 * 1024 * 256                                          # linear_fuse
    f += 3 * 2 * 9 * 256 * 256 * h1 * h1 + 2 * 9 * 256 * 96 * (2 * h1) ** 2
    return f / 1e9


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=4)
    ap.add_argument('--iters', type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_secc needs a CUDA device')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    dev = 'cuda:0'
    B, H = args.batch, 512
    m = r3.SegFormerSECC2PlaneBackbone()
    m.load_state_dict(ref.make_params({k: v.shape for k, v in m.state_dict().items()}, 7), strict=True)
    m = m.to(dev).eval()
    sd = {k: (v.to(dev, torch.float32) if v.is_floating_point() else v.to(dev)) for k, v in m.state_dict().items()}
    cano, src, tgt = (t.to(dev) for t in ref.make_inputs(B, H, 3))
    x = torch.cat([cano.expand(B, -1, -1, -1), src.expand(B, -1, -1, -1), tgt], 1).contiguous()
    m.begin_clip(cano, src)
    default_tf32 = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32

    def torch_arm(tf32):
        def run():
            torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = (True, True) if tf32 else (False, False)
            ref.forward(sd, x)
        return run
    arms = {'ours_forward': lambda: m(x), 'ours_planes_cl': lambda: m.planes_cl(tgt),
            'torch_default_tf32': lambda: (setattr(torch.backends.cuda.matmul, 'allow_tf32', default_tf32[0]),
                                           setattr(torch.backends.cudnn, 'allow_tf32', default_tf32[1]), ref.forward(sd, x)),
            'torch_tf32_off': torch_arm(False)}
    with torch.no_grad():
        for fn in arms.values():
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        res = {k: [] for k in arms}
        clocks = []
        for _ in range(3):
            for k, fn in arms.items():
                res[k].append(timed(fn, args.iters))
            clocks.append(subprocess.run(['nvidia-smi', '--query-gpu=clocks.sm', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip())
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = default_tf32
    # per-launch times of the conv stack: one profiled pass of its own (CUDA events around each launch), averaged over `iters` calls
    with torch.no_grad():
        capi.PROF = capi.Profiler()
        try:
            for _ in range(args.iters):
                m.planes_cl(tgt)
            prof = {k: round(v / args.iters, 3) for k, v in capi.PROF.totals().items() if k.startswith('secc2plane')}
        finally:
            capi.PROF = None

    # the clip step, batch 4, uint8 frames
    def mk(**kw):
        e = engine.FrameEngine(batch=B, sr_mode='tc', hp={'num_samples_fine': 0}, out_uint8=True, **kw)
        e.load_params(syn.make_decoder_params(seed=4), syn.make_sr_params(seed=5))
        return e
    cano_planes = syn.make_planes(1, seed=0).to(dev)
    cams = syn.make_cameras(B, seed=1).to(dev)
    u_c = syn.make_jitter(B, 4096, 48, 0, seed=2)[0].to(dev)
    resident = syn.make_planes(B, seed=3).to(dev)
    e_res, e_torch, e_secc = mk(), mk(), mk(secc2plane=m)
    e_secc.begin_planes(cano_planes, cano, src)
    with torch.no_grad():
        e_res.prepare([(resident, cams, u_c)])
        e_secc.prepare([(tgt, cams, u_c)])
    with torch.no_grad():
        # cuDNN may hand back the last conv's output channels-last; the render then samples it in place ('hwpc'), and the canonical set must
        # be in the same layout
        cano_for_torch = r3.canonical_planes_cl(cano_planes) if r3.producer_view(ref.forward(sd, x)) is not None else cano_planes
    steps = {'resident': lambda: e_res.step(resident, cams, u_c),
             'torch': lambda: e_torch.step((cano_for_torch, ref.forward(sd, x)), cams, u_c),
             'engine': lambda: e_secc.step(None, cams, u_c, cond_tgt=tgt)}
    with torch.no_grad():
        for fn in steps.values():
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        step_res = {k: [] for k in steps}
        for _ in range(3):
            for k, fn in steps.items():
                step_res[k].append(timed(fn, args.iters))
            clocks.append(subprocess.run(['nvidia-smi', '--query-gpu=clocks.sm', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip())
    gf = gflop(H) * B
    out = {'gpu': q, 'sm_clock_samples': clocks, 'batch': B, 'size': H, 'gflop_per_call': round(gf, 2),
           'torch_default_tf32_flags': list(default_tf32)}
    for k, v in res.items():
        ms = statistics.median(v)
        out[k] = {'ms': round(ms, 3), 'tflops': round(gf / ms, 1), 'runs_ms': [round(t, 3) for t in v]}
    out['conv_stack_ms_per_launch'] = prof
    out['clip_step_uint8'] = {k: {'ms': round(statistics.median(v), 3), 'frames_per_s': round(B * 1e3 / statistics.median(v), 1),
                                  'runs_ms': [round(t, 3) for t in v]} for k, v in step_res.items()}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
