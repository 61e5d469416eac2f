"""Per-launch timing of the tensor-core SR of the bench step: batch of 4, 32-channel 128x128 features -> 512x512 image, shared styles.

    python tools/bench_sr.py [--modes tc tc_exact] [--batch 4] [--iters 30] [--warmup 5] [--dump DIR]

The SR runs layer by layer through the library's C entry points, in the order sr_tc.forward uses for the standard SR with prepared
(static) styles, so that every intermediate can be kept.  Kernel times are the device durations of torch.profiler's CUDA activity
records, median over the iterations: the transposed conv, its edge column and its FIR pass are launched by one library call, so CUDA
events around the calls could not split them.  The whole SR is also timed with CUDA events (median), in a run without the profiler.
Per conv launch the script prints the MMA GFLOP issued for the valid output rows (input channels padded to 64, 32 for block0.conv0, three products per
multiply-add in tc_exact) and the TFLOP/s this gives.

--dump DIR writes every layer's output of the last iteration as DIR/<mode>/<name>.npy.  R3DP_LIB selects the library file, so two
builds run through this script on the same seeds give dumps that compare byte for byte."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import real3dportrait_b200 as r3                                          # noqa: E402
from real3dportrait_b200 import _capi as capi, sr_tc, synthetic as syn   # noqa: E402

CONV_LAUNCHES = ('block0.conv0', 'block0.conv1+torgb', 'block1.conv0', 'block1.conv1+torgb')


def conv_gflop(B, split):
    """MMA GFLOP of the four conv launches for the valid output rows (Cin padded to 64 as issued; block0.conv0 runs 32-channel K chunks)."""
    f = [4 * 9 * 128 * 128 * 256 * 32,                     # block0.conv0: 4 output parities x 9 FIR-composed taps on the 128^2 grid, Cin 32
         9 * 256 * 256 * 256 * 256,                        # block0.conv1
         (6 * 257 + 3 * 256) * 256 * 128 * 256,            # block1.conv0: 4 + 2 taps on 257 rows, 2 + 1 taps on 256 rows, 256 columns
         9 * 512 * 512 * 128 * 128]                        # block1.conv1
    return [2 * x * B * (3 if split else 1) / 1e9 for x in f]


def build_sr(mode, dev):
    sr = r3.SuperresolutionHybrid8XDC(channels=32, img_resolution=512, sr_num_fp16_res=0, sr_antialias=True, sr_mode=mode)
    sr.load_state_dict(syn.make_sr_params(seed=5), strict=True)
    sr = sr.to(dev).eval()
    split = mode == 'tc_exact'
    prep = sr_tc.Prepared(sr, torch.ones(1, 3, 512, device=dev), split)
    return sr, prep, split


def make_step(sr, prep, split, fimg):
    """Returns run() -> dict of every layer output (fresh buffers each call, allocated before the first launch)."""
    L = capi.lib()
    (b0, b1), Nw, wp = sr_tc._sblocks(sr), prep.Nw, prep.wp
    N, dev, wide = fimg.shape[0], fimg.device, 2 if split else 1
    rgb0 = fimg[:, :3].contiguous()
    fn = lambda name: sr_tc._fn(name, split)                           # noqa: E731
    f16 = lambda t: capi.ptr(t, torch.float16)                          # noqa: E731
    bias = [capi.f32(b.bias) for b in (b0.conv0, b0.conv1, b1.conv0, b1.conv1, b0.torgb, b1.torgb)]

    def run():
        o = {'x0': torch.empty(N, 128, 128, 64 * wide, device=dev, dtype=torch.float16),
             'block0.conv0': torch.empty(N, 256, 256, 256 * wide, device=dev, dtype=torch.float16),
             'block0.conv1': torch.empty(N, 256, 256, 256 * wide, device=dev, dtype=torch.float16),
             'img1': torch.empty(N, 3, 256, 256, device=dev),
             'block1.conv0.raw': torch.empty(fn('scratch_bytes')(N, 128, 256, 256) // 2, device=dev, dtype=torch.float16),
             'block1.conv0': torch.empty(N, 512, 512, 128 * wide, device=dev, dtype=torch.float16),
             'image': torch.empty(N, 3, 512, 512, device=dev)}
        capi.check(fn('input')(capi.ptr(fimg), N, 32, 128, 128, 128, f16(o['x0']), capi.stream()))
        capi.check(fn('layer_up_composed')(f16(o['x0']), f16(wp[0]), capi.ptr(bias[0]), N, Nw, 32, 256, 128, 128, f16(o['block0.conv0']),
                                           capi.stream()))
        capi.check(fn('layer_torgb')(f16(o['block0.conv0']), f16(wp[1]), capi.ptr(bias[1]), capi.ptr(prep.wrgb0), capi.ptr(bias[4]), capi.ptr(rgb0),
                                     N, Nw, 256, 256, 256, 256, f16(o['block0.conv1']), capi.ptr(o['img1']), capi.stream()))
        capi.check(fn('layer')(f16(o['block0.conv1']), f16(wp[2]), capi.ptr(bias[2]), N, Nw, 256, 128, 256, 256, 2, f16(o['block1.conv0']),
                               capi.ptr(o['block1.conv0.raw'], torch.float16), capi.stream()))
        last = L.r3dp_sr_tcx_last_layer if split else L.r3dp_sr_tc_last_layer_ex
        capi.check(last(f16(o['block1.conv0']), f16(wp[3]), capi.ptr(bias[3]), capi.ptr(prep.wrgb1), capi.ptr(bias[5]), capi.ptr(o['img1']), N, Nw,
                        128, 512, 512, capi.ptr(o['image']), None, 0, capi.stream()))
        return o

    return run


def short_name(name):
    s = name.split('(')[0]
    s = s.replace('void ', '').replace('r3dp::tc::', '').replace('r3dp::', '')
    return s.strip()


def profile_launches(run, iters, min_iters=20):
    """Kernel names of one SR pass and, per launch, its device times over the iterations.  The iterations are separated by a host sleep, so
    the kernel records split at the idle gaps; an iteration whose record list is incomplete (the activity buffer can drop a record) is skipped."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    gap_us = 2000.0
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            run()
            torch.cuda.synchronize()
            time.sleep(gap_us / 1e6)
    ev = sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA and 'memset' not in e.name.lower() and 'memcpy' not in e.name.lower()),
                key=lambda e: e.time_range.start)
    groups, cur = [], []
    for e in ev:
        if cur and e.time_range.start - cur[-1].time_range.end > gap_us / 2:
            groups.append(cur); cur = []
        cur.append(e)
    groups.append(cur)
    seqs = [tuple(short_name(e.name) for e in g) for g in groups]
    names = max(set(seqs), key=seqs.count)
    full = [g for g, s in zip(groups, seqs) if s == names]
    assert len(full) >= min_iters, f'only {len(full)} complete iterations of {iters}'
    return list(names), [[g[j].time_range.elapsed_us() / 1e3 for g in full] for j in range(len(names))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--modes', nargs='+', default=['tc', 'tc_exact'], choices=['tc', 'tc_exact'])
    ap.add_argument('--batch', type=int, default=4)
    ap.add_argument('--iters', type=int, default=30)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--seed', type=int, default=11)
    ap.add_argument('--dump', metavar='DIR', default=None)
    args = ap.parse_args()
    assert args.iters >= 20, 'medians need at least 20 runs'
    dev = torch.device('cuda')
    g = torch.Generator().manual_seed(args.seed)
    fimg = (torch.rand(args.batch, 32, 128, 128, generator=g) * 2 - 1).to(dev)
    with torch.no_grad():
        for mode in args.modes:
            sr, prep, split = build_sr(mode, dev)
            run = make_step(sr, prep, split, fimg)
            for _ in range(args.warmup):
                run()
            torch.cuda.synchronize()
            whole = []
            for _ in range(args.iters):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(); out = run(); b.record()
                b.synchronize()
                whole.append(a.elapsed_time(b))
            names, times = profile_launches(run, args.iters)
            gf = iter(conv_gflop(args.batch, split))
            conv_i = 0
            rows = []
            for name, t in zip(names, times):
                row = {'kernel': name, 'ms': round(statistics.median(t), 4), 'spread_ms': round(max(t) - min(t), 4)}
                if name.startswith('conv_tc3_kernel'):
                    row['layer'] = CONV_LAUNCHES[conv_i]; conv_i += 1
                    row['gflop'] = round(next(gf), 2)
                    row['tflops'] = round(row['gflop'] / row['ms'], 1)
                rows.append(row)
            conv_ms = sum(r['ms'] for r in rows if 'gflop' in r)
            print(json.dumps({'sr_mode': mode, 'batch': args.batch, 'iters': args.iters, 'lib': capi.LIB_PATH,
                              'device': torch.cuda.get_device_name(), 'sr_ms_events': round(statistics.median(whole), 4),
                              'conv_ms': round(conv_ms, 4), 'conv_tflops': round(sum(conv_gflop(args.batch, split)) / conv_ms, 1), 'launches': rows}))
            if args.dump:
                d = os.path.join(args.dump, mode)
                os.makedirs(d, exist_ok=True)
                torch.cuda.synchronize()
                for k, v in out.items():
                    np.save(os.path.join(d, k + '.npy'), v.cpu().numpy())


if __name__ == '__main__':
    main()
