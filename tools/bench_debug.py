"""Cost of the 'concat_debug' video frames: a clip through FrameEngine (secc2plane head, cond_tgt, batch 4, CUDA graphs) with
out_mode='final' and out_mode='concat_debug', alternating, median of 3; and the reference's host-side post-processing (real3d_infer.py:494-521,
as tests/debug_frames_reference.py restates it) on the same number of frames.

    python tools/bench_debug.py [--frames 512] [--host-frames 64]

Prints one JSON line: the card, its power limit and SM clock, frames/s of each mode, the added time per step, the close_clip() time, and the
host restatement's time per frame (measured on --host-frames frames and scaled to the clip)."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import real3dportrait_b200 as r3  # noqa: E402
from real3dportrait_b200 import engine, synthetic as syn  # noqa: E402
import secc2plane_reference as s2p_ref  # noqa: E402
from debug_frames_reference import concat_debug_reference  # noqa: E402

DEV = 'cuda:0'


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        out = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout
        name, pl, sm, smax = [x.strip() for x in out.splitlines()[0].split(',')]
        return {'gpu': name, 'power_limit': pl, 'sm_clock': sm, 'sm_clock_max': smax}
    except Exception as e:                                             # noqa: BLE001
        return {'gpu': torch.cuda.get_device_name(0), 'card_query_error': str(e)}


def make_engine(mode, B):
    bb = r3.SegFormerSECC2PlaneBackbone()
    bb.load_state_dict(s2p_ref.make_params({k: v.shape for k, v in bb.state_dict().items()}, 7), strict=True)
    eng = engine.FrameEngine(batch=B, sr_mode='tc', hp={'num_samples_fine': 0}, secc2plane=bb, out_uint8=True, out_mode=mode)
    eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_params(seed=5))
    cano_in = s2p_ref.make_inputs(1, 512, 1)
    eng.begin_planes(syn.make_planes(1, seed=1).to(DEV), cano_in[0].to(DEV), cano_in[1].to(DEV))
    return eng


@torch.no_grad()
def run_clip(eng, inputs, frames, B, ref_gt):
    """-> (ms for all steps, ms for close_clip)."""
    if eng.debug:
        eng.open_clip(frames, ref_gt_img=ref_gt)
    else:
        eng.open_clip(frames)
    torch.cuda.synchronize()
    a, b, c = (torch.cuda.Event(enable_timing=True) for _ in range(3))
    a.record()
    for s in range(frames // B):
        tgt, cams, u = inputs[s % len(inputs)]
        eng.step(None, cams, u, cond_tgt=tgt, frame_index=s * B)
    b.record()
    eng.close_clip()
    c.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), b.elapsed_time(c)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=512)
    ap.add_argument('--batch', type=int, default=4)
    ap.add_argument('--host-frames', type=int, default=64)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    B, F = args.batch, args.frames
    torch.cuda.set_device(0)
    info = card()
    inputs = []
    for s in range(4):
        _, _, tgt = s2p_ref.make_inputs(B, 512, 40 + s)
        u_c, _ = syn.make_jitter(B, 4096, 48, 0, seed=140 + s)
        inputs.append((tgt.to(DEV), syn.make_cameras(B, seed=240 + s).to(DEV), u_c.to(DEV)))
    ref_gt = ((torch.randint(0, 256, (1, 3, 512, 512), generator=torch.Generator().manual_seed(5)).float() - 127.5) / 127.5).to(DEV)
    engs = {m: make_engine(m, B) for m in ('final', 'concat_debug')}
    for m, e in engs.items():                                          # warm-up: graph capture, clip allocation
        run_clip(e, inputs, 4 * B, B, ref_gt)
    times = {m: [] for m in engs}
    for _ in range(args.reps):
        for m, e in engs.items():
            times[m].append(run_clip(e, inputs, F, B, ref_gt))
    med = {m: (statistics.median(t[0] for t in ts), statistics.median(t[1] for t in ts)) for m, ts in times.items()}
    steps = F // B
    # the reference's host post-processing on CPU copies of the clip's tensors (what this feature replaces)
    n = min(args.host_frames, F)
    g = torch.Generator().manual_seed(0)
    host = [torch.rand(1, 3, 512, 512, generator=g) * 2 - 1, torch.rand(n, 3, 512, 512, generator=g) * 2 - 1,
            torch.rand(n, 3, 64, 64, generator=g) * 2 - 1, torch.rand(n, 1, 64, 64, generator=g) + 2, torch.rand(n, 3, 512, 512, generator=g) * 2 - 1]
    ht = []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        concat_debug_reference(*host)
        ht.append((time.perf_counter() - t0) * 1e3)
    host_ms_per_frame = statistics.median(ht) / n
    res = dict(info, frames=F, batch=B, reps=args.reps,
               final_fps=F / med['final'][0] * 1e3, concat_debug_fps=F / med['concat_debug'][0] * 1e3,
               added_ms_per_step=(med['concat_debug'][0] - med['final'][0]) / steps,
               close_clip_ms_final=med['final'][1], close_clip_ms_concat_debug=med['concat_debug'][1],
               host_postprocess_ms_per_frame=host_ms_per_frame, host_postprocess_ms_clip=host_ms_per_frame * F,
               host_threads=torch.get_num_threads(), host_frames_measured=n)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
