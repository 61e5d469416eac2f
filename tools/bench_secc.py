"""Time SegFormerSECC2PlaneBackbone (MiT-b0, 512^2 SECC input, batch 4) on one GPU: this library against PyTorch running the same module
(the float64-checked restatement tests/secc2plane_reference.py in fp32 nn ops), with torch's default TF32 setting and with TF32 off.
Arms alternate; each figure is the median of 3 windows of CUDA-event time.  Prints the card, its power limit and SM clock samples.
Also: per-launch times of the conv stack (a profiled pass of its own), and the clip step at batch 4 with uint8 frames in three arms:
  resident   FrameEngine fed resident planes (the headline workload's step; no backbone)
  torch      the PyTorch backbone, then FrameEngine on the (canonical, secc) pair (what a user pays without this library's backbone)
  engine     FrameEngine(secc2plane=...): backbone and render in one CUDA graph

The `render` section times SECC_Renderer (synthetic BFM at the real BFM's size, 512^2): per call at batch 4 and 50, per launch (with the vertex
pass's GB/s on its algorithmic bytes: basis + mean + coefficients + vertices out), the clip step fed coefficients (secc_renderer engine) against
the same engine fed resident SECC images, and the step_host loop with coefficients against SECC images.  There is no pytorch3d comparator.

The `blink` section times the SECC blink (SECC_Renderer.blink) at 512^2: one batch call with every frame blinking (p = 1 and p = 0.44) and with
no frame blinking (each call re-copies the rendered batch first; the copy alone is timed too), the coefficient clip step with blink=True
against blink=False (a step with no blinking frame, a step whose frames all blink, and 500 frames under a period_blink_schedule), and for
context the reference-semantics CPU cost of one frame through the numpy restatement (tests/blink_reference.py).

    python tools/bench_secc.py [--batch 4] [--iters 20] [--section all|backbone|render|blink]"""
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
    ap.add_argument('--section', choices=('all', 'backbone', 'render', 'blink'), default='all')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_secc needs a CUDA device')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    out = {'gpu': q}
    if args.section in ('all', 'backbone'):
        out.update(bench_backbone(args))
    if args.section in ('all', 'render'):
        out['render'] = bench_render(args)
    if args.section in ('all', 'blink'):
        out['blink'] = bench_blink(args)
    print(json.dumps(out))


def _clock():
    return subprocess.run(['nvidia-smi', '--query-gpu=clocks.sm', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()


def _alternate(arms, iters, clocks):
    """Warm every arm, then 3 rounds of the arms in turn; -> {arm: {'ms': median, 'runs_ms': [...]}}."""
    with torch.no_grad():
        for fn in arms.values():
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        res = {k: [] for k in arms}
        for _ in range(3):
            for k, fn in arms.items():
                res[k].append(timed(fn, iters))
            clocks.append(_clock())
    return {k: {'ms': round(statistics.median(v), 4), 'runs_ms': [round(t, 4) for t in v]} for k, v in res.items()}


def bench_render(args):
    import tempfile
    dev, B, S = 'cuda:0', args.batch, 512
    kw = syn.write_bfm_folder(tempfile.mkdtemp(prefix='r3dp_bfm_'), seed=0)
    r = r3.SECC_Renderer(S, device=dev, **kw)
    clocks = []
    calls = {}
    for n in (B, 50):
        c = {k: v.to(dev) for k, v in syn.make_coeffs(n, seed=1).items()}
        calls[n] = c
    call = _alternate({f'call_b{n}': (lambda c=c: r(c['id'], c['exp'], c['euler'], c['trans'])) for n, c in calls.items()}, args.iters, clocks)
    # per-launch times: a profiled pass of its own (CUDA events around each launch)
    per_launch = {}
    with torch.no_grad():
        for n, c in calls.items():
            capi.PROF = capi.Profiler()
            try:
                for _ in range(args.iters):
                    r(c['id'], c['exp'], c['euler'], c['trans'])
                t = {k.split('.', 1)[1]: v / args.iters for k, v in capi.PROF.totals().items() if k.startswith('secc_render.')}
            finally:
                capi.PROF = None
            nbytes = r.basis.numel() * 4 + r.mean_shape.numel() * 4 + n * (r.n_id + r.n_exp) * 4 + n * r.n_verts * 16
            per_launch[f'b{n}'] = {k: round(v * 1e3, 1) for k, v in t.items()}
            per_launch[f'b{n}']['unit'] = 'us'
            per_launch[f'b{n}']['vertices_GBps'] = round(nbytes / (t['vertices'] * 1e-3) / 1e9, 1)
            per_launch[f'b{n}']['vertices_bytes'] = nbytes
    # the clip step, batch B, uint8 frames, secc2plane engine: fed coefficients vs fed resident SECC images
    m = r3.SegFormerSECC2PlaneBackbone()
    m.load_state_dict(ref.make_params({k: v.shape for k, v in m.state_dict().items()}, 7), strict=True)
    m = m.to(dev).eval()

    def mk(**k):
        e = engine.FrameEngine(batch=B, sr_mode='tc', hp={'num_samples_fine': 0}, out_uint8=True, secc2plane=m, **k)
        e.load_params(syn.make_decoder_params(seed=4), syn.make_sr_params(seed=5))
        return e
    src = syn.make_coeffs(1, seed=2)
    coeff_src = torch.cat([src['id'], src['exp']], 1).to(dev)
    cano_c = coeff_src.clone()
    cano_c[:, r.n_id:] = 0
    cano_planes = syn.make_planes(1, seed=0).to(dev)
    e_coef, e_img = mk(secc_renderer=r), mk()
    with torch.no_grad():
        e_coef.begin_planes(cano_planes, coeff_src=coeff_src)
        e_img.begin_planes(cano_planes, r.render(cano_c)[1], r.render(coeff_src)[1])
    drv = syn.make_coeffs(B, seed=3)
    coeff = torch.cat([drv['id'], drv['exp']], 1).to(dev)
    with torch.no_grad():
        img = r.render(coeff)[1].clone()
    cams = syn.make_cameras(B, seed=1).to(dev)
    u_c = syn.make_jitter(B, 4096, 48, 0, seed=2)[0].to(dev)
    with torch.no_grad():
        e_coef.prepare([(coeff, cams, u_c)])
        e_img.prepare([(img, cams, u_c)])
    step = _alternate({'coeff': lambda: e_coef.step(None, cams, u_c, coeff=coeff),
                       'resident_image': lambda: e_img.step(None, cams, u_c, cond_tgt=img)}, args.iters, clocks)
    # the step_host loop: pinned host inputs -> pinned host frames, coefficients vs SECC images
    h_cams, h_u = cams.cpu().pin_memory(), u_c.cpu().pin_memory()
    h_coeff, h_img = coeff.cpu().pin_memory(), img.cpu().pin_memory()
    h_out = torch.empty(B, 512, 512, 3, dtype=torch.uint8).pin_memory()
    eh_coef, eh_img = mk(secc_renderer=r), mk()
    with torch.no_grad():
        eh_coef.begin_planes(cano_planes, coeff_src=coeff_src)
        eh_img.begin_planes(cano_planes, r.render(cano_c)[1], r.render(coeff_src)[1])

    def host_loop(e, h):
        def run():
            e.step_host(h, h_cams, h_u, h_out)
        return run
    host = _alternate({'coeff': host_loop(eh_coef, h_coeff), 'image': host_loop(eh_img, h_img)}, args.iters, clocks)
    for k, h in (('coeff', h_coeff), ('image', h_img)):
        host[k]['planes_slot_h2d_bytes_per_step'] = h.numel() * h.element_size()
    return {'size': S, 'batch': B, 'faces': r.n_faces, 'vertices': r.n_verts, 'sm_clock_samples': clocks, 'per_call_ms': call,
            'per_launch': per_launch, 'clip_step_uint8': step, 'step_host_loop': host,
            'comparator': 'none: no pytorch3d arm (no speed-up over the reference renderer is claimed)'}


def bench_blink(args):
    import random
    import tempfile
    import time
    import blink_reference as bref
    dev, B, S = 'cuda:0', args.batch, 512
    kw = syn.write_bfm_folder(tempfile.mkdtemp(prefix='r3dp_bfm_'), seed=0)
    r = r3.SECC_Renderer(S, device=dev, **kw)
    clocks = []
    drv = syn.make_coeffs(B, seed=3)
    coeff = torch.cat([drv['id'], drv['exp']], 1).to(dev)
    with torch.no_grad():
        src = r.render(coeff)[1].clone()
    work = src.clone()

    def call(p):
        def run():
            work.copy_(src)
            r.blink(work, p=p)
        return run
    p1, p44, none = (torch.full((B,), v, dtype=torch.float64, device=dev) for v in (1.0, 0.44, -1.0))
    calls = _alternate({'all_blink_p1': call(p1), 'all_blink_p044': call(p44), 'none_blink': call(none), 'copy_only': lambda: work.copy_(src)},
                       args.iters, clocks)
    assert r.blink_faults() == 0
    m = r3.SegFormerSECC2PlaneBackbone()
    m.load_state_dict(ref.make_params({k: v.shape for k, v in m.state_dict().items()}, 7), strict=True)
    m = m.to(dev).eval()

    def mk(**k):
        e = engine.FrameEngine(batch=B, sr_mode='tc', hp={'num_samples_fine': 0}, out_uint8=True, secc2plane=m, secc_renderer=r, **k)
        e.load_params(syn.make_decoder_params(seed=4), syn.make_sr_params(seed=5))
        return e
    s0 = syn.make_coeffs(1, seed=2)
    coeff_src = torch.cat([s0['id'], s0['exp']], 1).to(dev)
    cano_planes = syn.make_planes(1, seed=0).to(dev)
    e_blink, e_plain = mk(blink=True), mk()
    with torch.no_grad():
        e_blink.begin_planes(cano_planes, coeff_src=coeff_src)
        e_plain.begin_planes(cano_planes, coeff_src=coeff_src)
    cams = syn.make_cameras(B, seed=1).to(dev)
    u_c = syn.make_jitter(B, 4096, 48, 0, seed=2)[0].to(dev)

    def rows_of(tT):
        return torch.cat([coeff, torch.tensor(tT, dtype=torch.float32, device=dev)], 1).contiguous()
    r_none, r_all = rows_of([[0, 0]] * B), rows_of([[t, 10] for t in range(1, B + 1)])
    step = _alternate({'blink_none_blinking': lambda: e_blink.step(None, cams, u_c, coeff=r_none),
                       'blink_all_blinking': lambda: e_blink.step(None, cams, u_c, coeff=r_all),
                       'no_blink': lambda: e_plain.step(None, cams, u_c, coeff=coeff)}, args.iters, clocks)
    # 500 frames: steps of B frames with a period_blink_schedule (random.Random(0)), every step's rows resident
    N = 500
    sched = r3.period_blink_schedule(N, rng=random.Random(0)).float().to(dev)
    clip_rows = [torch.cat([coeff, sched[i:i + B]], 1).contiguous() for i in range(0, N - N % B, B)]

    def clip(e, wide):
        def run():
            for rw in clip_rows:
                e.step(None, cams, u_c, coeff=rw if wide else coeff)
        return run
    clip_ms = _alternate({'blink': clip(e_blink, True), 'no_blink': clip(e_plain, False)}, 1, clocks)
    assert e_blink.blink_faults() == 0
    # context: the reference semantics on the CPU, one frame (numpy restatement; the reference itself adds two k-d trees per frame)
    x = src[0].cpu().numpy()
    t0 = time.perf_counter()
    for _ in range(3):
        bref.blink(x, 0.44)
    cpu_ms = (time.perf_counter() - t0) / 3 * 1e3
    net = {k: round(calls[k]['ms'] - calls['copy_only']['ms'], 4) for k in ('all_blink_p1', 'all_blink_p044', 'none_blink')}
    return {'size': S, 'batch': B, 'sm_clock_samples': clocks, 'call_ms': calls, 'call_net_of_copy_ms': net, 'clip_step_uint8': step,
            'step_overhead_pct': {k: round(100 * (step[k]['ms'] / step['no_blink']['ms'] - 1), 2) for k in ('blink_none_blinking', 'blink_all_blinking')},
            'clip_500_frames_ms': clip_ms, 'blinking_frames_in_500': int((sched[:, 1] > 0).sum()),
            'cpu_restatement_ms_per_frame': round(cpu_ms, 1)}


def bench_backbone(args):
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
    out = {'sm_clock_samples': clocks, 'batch': B, 'size': H, 'gflop_per_call': round(gf, 2),
           'torch_default_tf32_flags': list(default_tf32)}
    for k, v in res.items():
        ms = statistics.median(v)
        out[k] = {'ms': round(ms, 3), 'tflops': round(gf / ms, 1), 'runs_ms': [round(t, 3) for t in v]}
    out['conv_stack_ms_per_launch'] = prof
    out['clip_step_uint8'] = {k: {'ms': round(statistics.median(v), 3), 'frames_per_s': round(B * 1e3 / statistics.median(v), 1),
                                  'runs_ms': [round(t, 3) for t in v]} for k, v in step_res.items()}
    return out


if __name__ == '__main__':
    main()
