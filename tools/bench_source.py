"""Time the source images at 512^2 with CUDA events: prepare_source on one image (ref_head_img, ref_torso_img and bg_img, including the
geometry check's host sync), prepare_source with bg_img= given (the torso and head images alone), and extract_background over 100 and 1 000
frames (5 and 50 selected).  Warm-up, then the median of 10 calls.  Prints the card, its power limit and SM clock with the numbers.

    python tools/bench_source.py [--frames 100 1000] [--reps 10]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm,clocks.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=20)
        return q.stdout.strip() or 'unknown'
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, nargs='+', default=[100, 1000])
    ap.add_argument('--reps', type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_source needs a GPU'
    import real3dportrait_b200 as r3
    from real3dportrait_b200 import source, synthetic as syn
    dev = 'cuda:0'
    H = W = 512
    img = torch.from_numpy(syn.make_source_image(H, W, 0)).to(dev)
    seg = torch.from_numpy(syn.make_segmap(H, W, 0)).to(dev)
    out = {k: torch.empty(1, 3, H, W, device=dev) for k in source.OUTPUTS}
    res = {'card (name, power limit, max SM clock, SM clock)': card(), 'size': [H, W], 'ms': {}}
    res['ms']['prepare_source'] = timed(lambda: r3.prepare_source(img, seg, out=out), args.reps)
    res['ms']['prepare_source(bg_img=)'] = timed(lambda: r3.prepare_source(img, seg, bg_img=out['bg_img'], out=out), args.reps)
    for n in args.frames:
        frames = torch.stack([torch.from_numpy(syn.make_source_image(H, W, 100 + i)) for i in range(n)]).to(dev)
        segs = torch.stack([torch.from_numpy(syn.make_segmap(H, W, 7, center=0.5 + 0.2 * np.sin(0.7 * i))) for i in range(n)]).to(dev)
        bg = torch.empty(H, W, 3, dtype=torch.uint8, device=dev)
        res['ms'][f'extract_background N={n} ({len(source.selected_frames(n))} used)'] = timed(
            lambda: r3.extract_background(frames, segs, out=bg), args.reps)
        del frames, segs
    res['card after (name, power limit, max SM clock, SM clock)'] = card()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
