"""Time ClipMotion.clip (a clip's cameras and torso key points) for 1 500 and 15 000 frames (one and ten minutes at 25 fps) with CUDA events:
warm-up, then the median of 3.  The float64 host restatement (tests/motion_reference.py, numpy / scipy with one Rotation.mean per frame as the
reference's smooth_camera_sequence does) is timed beside it; it is a restatement, not the reference.  Prints the card and its power limit.

    python tools/bench_motion.py [--frames 1500 15000] [--no-host]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True, text=True,
                           timeout=20)
        power = q.stdout.strip() or 'unknown'
    except (OSError, subprocess.SubprocessError):
        power = 'unknown'
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, nargs='+', default=[1500, 15000])
    ap.add_argument('--no-host', action='store_true')
    a = ap.parse_args()
    import motion_reference as mref
    import real3dportrait_b200 as r3
    from real3dportrait_b200 import synthetic as syn
    name, power = card()
    out = {'gpu': name, 'power_limit': power, 'runs': []}
    with tempfile.TemporaryDirectory() as d:
        kw = syn.write_bfm_folder(d, seed=0, keypoints=True)
        cm = r3.ClipMotion(kw['bfm_folder'], device='cuda:0')
        model = mref.load(kw['bfm_folder'])
    for T in a.frames:
        c = mref.make_case(T, 300, seed=1)
        dv = {k: torch.from_numpy(np.ascontiguousarray(c[k])).cuda() for k in ('id', 'exp', 'src_euler', 'src_trans', 'src_exp')}
        pose = tuple(torch.from_numpy(x).cuda() for x in c['pose'])
        res = (torch.empty(T, 25, device='cuda'), torch.empty(1, 68, 3, device='cuda'), torch.empty(T, 68, 3, device='cuda'))

        def run():
            cm.clip(dv['id'], dv['exp'], dv['src_euler'], dv['src_trans'], dv['src_exp'], pose=pose, out=res)
        for _ in range(3):
            run()
        torch.cuda.synchronize()
        ms = []
        for _ in range(3):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run()
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        # the launches alone, without the host-side validation: a CUDA graph of the call
        g = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            run()
        torch.cuda.current_stream().wait_stream(s)
        with torch.cuda.graph(g):
            run()
        gm = []
        for _ in range(3):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            g.replay()
            e1.record()
            e1.synchronize()
            gm.append(e0.elapsed_time(e1))
        row = {'frames': T, 'clip_ms_median': float(np.median(ms)), 'clip_graph_ms_median': float(np.median(gm))}
        if not a.no_host:
            hs = []
            for _ in range(3):
                t0 = time.perf_counter()
                mref.clip(model, c['id'], c['exp'], c['src_euler'], c['src_trans'], c['src_exp'], c['pose'], True)
                hs.append((time.perf_counter() - t0) * 1e3)
            row['host_float64_restatement_ms_median'] = float(np.median(hs))
        out['runs'].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
