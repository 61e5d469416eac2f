"""Timing of the fused render on one GPU (BASELINE configs[1]: batch of 4 frames, 64x64 rays x 48 samples, render only).

    python tools/bench_render.py [--frames 4] [--pool 32] [--iters 30] [--fine 0 | 48]

Prints one JSON line per plane layout: CUDA-event time per call of r3dp_render_ex (limits + decoder image + render + clamp kernels) over
a pool of resident frames larger than L2, for channels-last planes, the producer's channels_last view ('hwpc') and the two-plane-set
(cano + secc) mode.  --fine 0 times single-pass renders (the streaming kernel), --fine 48 importance renders (the CTA-per-ray-tile
kernel).  Also checks that every layout returns the same image as the first.  Comparing two builds: run once per library (R3DP_LIB)."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import real3dportrait_b200 as r3                                          # noqa: E402
from real3dportrait_b200 import _capi, renderer as ren, synthetic as syn   # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=4)
    ap.add_argument('--pool', type=int, default=32)
    ap.add_argument('--iters', type=int, default=30)
    ap.add_argument('--fine', type=int, default=0)
    ap.add_argument('--only', default='', help='comma-separated variant names')
    args = ap.parse_args()
    dev = 'cuda'
    B, P = args.frames, args.pool
    planes = syn.make_planes(P, seed=100).to(dev)
    cams = syn.make_cameras(P, seed=200).to(dev)
    u_c, u_f = syn.make_jitter(P, 4096, 48, args.fine, seed=300)
    u_c = u_c.to(dev)
    u_f = None if u_f is None else u_f.to(dev)
    dec = r3.OSGDecoder(32, {'decoder_lr_mul': 1, 'decoder_output_dim': 32})
    dec.load_state_dict(syn.make_decoder_params(seed=4), strict=True)
    dec = dec.to(dev).eval()
    R = r3.ImportanceRenderer()
    nb = P // B
    cl = [ren.planes_to_channels_last(planes[i * B:(i + 1) * B]) for i in range(nb)]
    hw = [ren.PlanesCL(c.data.permute(0, 2, 3, 1, 4).contiguous(), 'hwpc') for c in cl]
    half = [ren.PlanesCL(c.data * 0.5) for c in cl]
    rays = [r3.RaySampler()(cams[i * B:(i + 1) * B, :16].reshape(-1, 4, 4), cams[i * B:(i + 1) * B, 16:25].reshape(-1, 3, 3), 64) for i in range(nb)]

    def opts(i):
        o = dict(syn.RENDERING_OPTIONS, depth_resolution=48, depth_resolution_importance=args.fine, u_coarse=u_c[i * B:(i + 1) * B])
        if u_f is not None:
            o['u_fine'] = u_f[i * B * 4096:(i + 1) * B * 4096]
        return o

    def run(pl, i):
        return R(pl[i % nb], dec, rays[i % nb][0], rays[i % nb][1], opts(i % nb))

    def timed(pl):
        for i in range(3):
            run(pl, i)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for i in range(args.iters):
            run(pl, i)
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / args.iters

    variants = [('cl', cl), ('hwpc', hw), ('two_sets', [(h, h) for h in half])]      # two sets: x/2 + x/2, same image, twice the gather
    if args.only:
        variants = [v for v in variants if v[0] in args.only.split(',')]
    ref = None
    for name, pl in variants:
        out = run(pl, 0)[0]
        if ref is None:
            ref, first = out.clone(), name
        diff = float((out - ref).abs().max())
        ms = timed(pl)
        print(json.dumps({'variant': name, 'ms_per_call': round(ms, 4), 'us_per_frame': round(1e3 * ms / B, 2), 'frames': B,
                          'samples_per_ray': 48 + args.fine, 'max_abs_diff_vs_' + first: diff, 'lib': _capi.LIB_PATH}))


if __name__ == '__main__':
    main()
