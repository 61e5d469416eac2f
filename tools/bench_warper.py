"""Times the torso warper's stage 2 (Generator + occlusion_2_predictor, modules/real3d/facev2v_warp/network2.py:248-301, model2.py:212-219)
on this library's kernels against cuDNN running the reference's own modules, and the torso head as a FrameEngine clip with the reference-shaped
warper in three arms.  Weights are random (tests/torso_warper_ref.randomize); the reference modules are the ones build() staged under oracle/_ref.

    python tools/bench_warper.py [--batch 4] [--iters 20] [--reps 3] [--frames 64] [--no-engine]

stage 2, per launch of --batch images: 'tc' and 'tc_exact' (torso_stage2='cuda'), 'cudnn_tf32' (the reference modules under torch's defaults,
cudnn.allow_tf32 = True) and 'cudnn_fp32' (TF32 off).  engine, frames/s of a --frames clip at --batch: 'torch' (the warper as the caller's
PyTorch module), 'cuda_uncached' (stage 2 on the kernels, appearance features recomputed per frame), 'cuda_cached' (the per-clip cache).
Arms alternate inside every rep; each number is the median of --reps.  The JSON line carries the card's name and power limit and the SM clock
and throttle reasons sampled after every rep (a power-capped card lowers its clocks under load).  Nothing on the device is reconfigured."""
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
from real3dportrait_b200 import synthetic as syn, torso_warp as tw      # noqa: E402
import torso_warper_ref as twr                                          # noqa: E402


def stage2_gflop(N: int) -> float:
    """Multiply-adds x 2 of the Generator (standard: 6 res blocks, up 256 -> 128 -> 64) and the predictor, from the layer shapes."""
    def conv(ci, co, k, hw):
        return 2.0 * ci * co * k * k * hw * hw
    g = conv(512, 256, 3, 64) + conv(256, 256, 1, 64) + 12 * conv(256, 256, 3, 64) + conv(256, 128, 3, 128) + conv(128, 64, 3, 256)
    g += conv(64, 3, 7, 256) + conv(65, 32, 3, 256) + conv(32, 32, 3, 256) + conv(32, 1, 3, 256)
    return N * g / 1e9


def sample_clocks():
    q = 'name,power.limit,clocks.sm,clocks_throttle_reasons.active'
    try:
        return subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                              capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:                                                     # noqa: BLE001
        return f'unavailable ({type(e).__name__})'


def time_ms(fn, iters):
    fn(); torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def stage2_arms(args, clocks):
    dev = 'cuda'
    G, _ = twr.ref_classes()
    gen, pred = twr.randomize(G(), seed=31).to(dev), twr.randomize(twr.make_predictor(), seed=32).to(dev)
    fs, deformation, occ = [t.to(dev) for t in twr.make_stage2_inputs(args.batch, 64, seed=32)]
    fsn = fs.permute(0, 2, 3, 4, 1).contiguous()
    wts = {m: tw.Stage2Weights(gen, pred, split=m == 'tc_exact') for m in ('tc', 'tc_exact')}

    def cudnn(tf32):
        def f():
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            with torch.no_grad():
                twr.reference_stage2(gen, pred, fs, deformation, occ)
        return f
    tf32_default = torch.backends.cudnn.allow_tf32
    arms = {'tc': lambda: tw.stage2(wts['tc'], fsn, deformation, occ), 'tc_exact': lambda: tw.stage2(wts['tc_exact'], fsn, deformation, occ),
            'cudnn_tf32': cudnn(tf32_default), 'cudnn_fp32': cudnn(False)}
    reps = {k: [] for k in arms}
    for _ in range(args.reps):
        for k, f in arms.items():
            reps[k].append(time_ms(f, args.iters))
        clocks.append(sample_clocks())
    torch.backends.cudnn.allow_tf32 = tf32_default
    gf = stage2_gflop(args.batch)
    return {k: {'ms': statistics.median(v), 'reps_ms': v, 'gflop': gf, 'tflops': gf / statistics.median(v)} for k, v in reps.items()}


def engine_arms(args, clocks):
    from real3dportrait_b200 import engine
    dev = 'cuda'
    _, Warp = twr.ref_classes()
    warper = twr.randomize(Warp('standard'), seed=41)
    srp = syn.make_sr_warp_params(seed=6)
    srp.update({'torso_model.' + k: v for k, v in warper.state_dict().items()})
    mlp = syn.make_decoder_params(seed=4)
    inp = syn.make_warp_inputs(1, seed=8)
    B = args.batch
    planes, cam = syn.make_planes(B, seed=0).to(dev), syn.make_cameras(B, seed=1).to(dev)
    u_c, u_f = syn.make_jitter(B, 4096, 48, 48, seed=3)
    kp_d = (torch.rand(B, 68, 3, generator=torch.Generator().manual_seed(2)) * 2 - 1).to(dev)
    engines = {}
    for arm in ('torch', 'cuda_uncached', 'cuda_cached'):
        eng = engine.FrameEngine(batch=B, sr_mode='tc', hp=dict(syn.WARP_HPARAMS, num_samples_fine=48), torso_model=twr.randomize(Warp('standard'), 41),
                                 torso_stage2='torch' if arm == 'torch' else 'cuda', out_uint8=True)
        eng.load_params(mlp, srp)
        eng.begin_clip(*(inp[k].to(dev) for k in ('ref_torso_rgb', 'ref_bg_rgb', 'segmap', 'kp_s')))
        if arm == 'cuda_uncached':                   # drop the appearance part of the clip cache: stage 1 runs whole every frame
            eng.head.superresolution._clip_cache['torso_app'] = None
        engines[arm] = eng
    steps = max(1, args.frames // B)

    def clip(eng):
        def f():
            with torch.no_grad():
                for _ in range(steps):
                    eng.step(planes, cam, u_c.to(dev), u_f.to(dev), kp_d=kp_d)
        return f
    reps = {k: [] for k in engines}
    for _ in range(args.reps):
        for k, eng in engines.items():
            reps[k].append(steps * B / (time_ms(clip(eng), 1) / 1e3))
        clocks.append(sample_clocks())
    return {k: {'frames_per_s': statistics.median(v), 'reps': v} for k, v in reps.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=4)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--frames', type=int, default=64)
    ap.add_argument('--no-engine', dest='engine', action='store_false')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_warper.py times the GPU: no CUDA device')
    if twr.ref_classes() is None:
        raise SystemExit('the reference warper modules are not staged under oracle/_ref (build() stages them where the reference exists)')
    clocks = [sample_clocks()]
    out = {'batch': args.batch, 'stage2': stage2_arms(args, clocks)}
    if args.engine:
        out['engine'] = engine_arms(args, clocks)
    out['clocks'] = clocks
    print(json.dumps(out))


if __name__ == '__main__':
    main()
