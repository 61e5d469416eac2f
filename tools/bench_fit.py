"""Time Fit3DMM.fit_image and Fit3DMM.fit_video (T = 125, the 5 s example; 1 500; 15 000 frames) with CUDA events: eagerly and as a
replayed CUDA graph, after a warm-up, the median of 3 runs alternating between the two.  Beside them, a PyTorch restatement of the
reference's loop on the same GPU in float32 (tests/fit_reference.py: autograd, torch.optim.Adam), without the fine stage and with it as the
reference runs it (50-iteration batches, whose results the reference discards); the fine stage is timed up to --fine-max frames.  It is a
restatement, not the reference.  Prints the card, its power limit and the stage-2 FLOP rate (2 x 2 x 1404 x 144 per frame-iteration).

    python tools/bench_fit.py [--frames 125 1500 15000] [--fine-max 1500]"""
import argparse
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'], capture_output=True,
                           text=True, timeout=20)
        power = q.stdout.strip() or 'unknown'
    except (OSError, subprocess.SubprocessError):
        power = 'unknown'
    return name, power


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, nargs='+', default=[125, 1500, 15000])
    ap.add_argument('--fine-max', type=int, default=1500)
    a = ap.parse_args()
    import fit_reference as fref
    import real3dportrait_b200 as r3
    from real3dportrait_b200 import synthetic as syn
    assert torch.cuda.is_available(), 'bench_fit needs a CUDA device'
    name, power = card()
    print(f'card: {name}, power limit / max SM clock: {power}')
    with tempfile.TemporaryDirectory() as d:
        bfm = syn.write_bfm_folder(d, seed=0, mp468=True)['bfm_folder']
        model = fref.load(bfm)
        f = r3.Fit3DMM(bfm)
    for T in [1] + a.frames:
        video = T > 1
        lms, _ = fref.make_landmarks(model, T, seed=T)
        x = torch.from_numpy(lms).cuda()
        call = (lambda: f.fit_video(x, out=out)) if video else (lambda: f.fit_image(x[0], out=out))
        out = {k: v.clone() for k, v in (f.fit_video(x) if video else f.fit_image(x[0])).items()}
        call()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            call()
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            call()
        g.replay()
        eager, graph = [], []
        for _ in range(3):
            eager.append(timed(call))
            graph.append(timed(g.replay))
        ref = lambda fine: fref.fit(model, lms, 512, video=video, dtype=torch.float32, device='cuda', fine=fine)  # noqa: E731
        ref(False)
        torch_plain = [timed(lambda: ref(False)) for _ in range(3)]
        torch_fine = [timed(lambda: ref(True)) for _ in range(1 if T > 150 else 3)] if T <= a.fine_max else None
        flop = 400 * 2 * 2 * 1404 * 144 * T / 2       # stage 2 only (200 of the 400 iterations run the GEMMs)
        e, gr = float(np.median(eager)), float(np.median(graph))
        fine_s = f'{np.median(torch_fine):.1f} ms' if torch_fine else 'not measured'
        print(f'{"fit_image" if not video else f"fit_video T={T}"}: eager {e:.2f} ms, graph {gr:.2f} ms '
              f'({flop / gr * 1e-9:.2f} TFLOP/s stage-2 GEMM rate over the whole graph); PyTorch loop {np.median(torch_plain):.1f} ms, '
              f'with the fine stage {fine_s}', flush=True)
        del g


if __name__ == '__main__':
    main()
