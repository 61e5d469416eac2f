"""Times the torso warper's stage 2 (Generator + occlusion_2_predictor, modules/real3d/facev2v_warp/network2.py:248-301, model2.py:212-219)
on this library's kernels against cuDNN running the reference's own modules, and the torso head as a FrameEngine clip with the reference-shaped
warper in three arms.  Weights are random (tests/torso_warper_ref.randomize); the reference modules are the ones build() staged under oracle/_ref.

    python tools/bench_warper.py [--batch 4] [--iters 20] [--reps 3] [--frames 64] [--no-engine]

stage 2, per launch of --batch images: 'tc' and 'tc_exact' (torso_stage2='cuda'), 'cudnn_tf32' (the reference modules under torch's defaults,
cudnn.allow_tf32 = True) and 'cudnn_fp32' (TF32 off).  engine, frames/s of a --frames clip at --batch: 'torch' (the warper as the caller's
PyTorch module), 'cuda_uncached' (stage 2 on the kernels, appearance features recomputed per frame), 'cuda_cached' (the per-clip cache).
motion, per launch of --batch images: the motion-field estimator (network2.py:162-244, 208.57 GFLOP/frame) in 'tc' and 'tc_exact'
(torso_motion='cuda') against the reference module under 'cudnn_tf32' and 'cudnn_fp32', plus the per-launch times of its fuser and mask
3-D convs in 'tc' (CUDA events around one launch each, averaged over --iters).  engine arm 'cuda_motion': stage 2 and the estimator on the
kernels, with the per-clip cache.  Arms alternate inside every rep; each number is the median of --reps.  The JSON line carries the card's name and power limit and the SM clock
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


def motion_gflop(N: int) -> float:
    """Multiply-adds x 2 of MotionFieldEstimator('standard', 34, 4) per the layer shapes (the up convs counted at the upsampled size)."""
    def conv(ci, co, taps, vox):
        return 2.0 * ci * co * taps * vox
    D, g = 16, 0.0
    for i, (ci, co) in enumerate(zip([25, 64, 128, 256, 512], [64, 128, 256, 512, 1024])):
        g += conv(ci, co, 27, D * (64 >> i) ** 2)
    for i, (ci, co) in enumerate(zip([1024, 512, 256, 128, 64], [512, 256, 128, 64, 32])):
        g += conv(ci, co, 27, D * (4 << i) ** 2)
    g += conv(4, 32, 49, 128 * 128) + 6 * conv(32, 32, 9, 128 * 128)
    g += conv(89, 32, 343, D * 64 * 64) + conv(32, 5, 343, D * 64 * 64) + 2 * conv(512, 1, 49, 64 * 64)
    return N * (g + conv(34, 4, 1, D * 64 * 64)) / 1e9


def motion_arms(args, clocks):
    dev = 'cuda'
    from modules.real3d.facev2v_warp.network2 import MotionFieldEstimator
    mfe = twr.randomize(MotionFieldEstimator('standard', input_channels=34, num_keypoints=4), seed=51).to(dev)
    B = args.batch
    g = torch.Generator().manual_seed(52)
    motion_inp = torch.randn(1, 34, 16, 64, 64, generator=g).to(dev).expand(B, -1, -1, -1, -1).contiguous()
    kp_s, kp_d = [(0.8 * (2 * torch.rand(B, 4, 3, generator=g) - 1)).to(dev) for _ in range(2)]
    rgb, wt = (2 * torch.rand(B, 3, 256, 256, generator=g) - 1).to(dev), torch.rand(B, 1, 256, 256, generator=g).to(dev)
    eye = torch.eye(3, device=dev)[None].repeat(B, 1, 1)
    wts = {m: tw.MotionWeights(mfe, split=m == 'tc_exact') for m in ('tc', 'tc_exact')}
    fc = tw.compress_volume(wts['tc'], motion_inp[:1])

    def cudnn(tf32):
        def f():
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            with torch.no_grad():
                mfe(motion_inp, kp_s, kp_d, eye, eye, rgb, wt)
        return f
    tf32_default = torch.backends.cudnn.allow_tf32
    arms = {'tc': lambda: tw.motion(wts['tc'], fc, kp_s, kp_d, rgb, wt), 'tc_exact': lambda: tw.motion(wts['tc_exact'], fc, kp_s, kp_d, rgb, wt),
            'cudnn_tf32': cudnn(tf32_default), 'cudnn_fp32': cudnn(False)}
    reps = {k: [] for k in arms}
    for _ in range(args.reps):
        for k, f in arms.items():
            reps[k].append(time_ms(f, args.iters))
        clocks.append(sample_clocks())
    torch.backends.cudnn.allow_tf32 = tf32_default
    gf = motion_gflop(B)
    out = {k: {'ms': statistics.median(v), 'reps_ms': v, 'gflop': gf, 'tflops': gf / statistics.median(v)} for k, v in reps.items()}
    # per-launch times of the two 7^3 convs in tc: the fuser (96 -> 32) and the mask logits (32 -> 5)
    from real3dportrait_b200 import _capi as capi
    L, f16 = capi.lib(), torch.float16
    w = wts['tc']
    xf = torch.randn(B, 16, 64, 64, w.CF, device=dev).half()
    fx = torch.empty(B, 16, 64, 64, 32, device=dev, dtype=f16)
    logits = torch.empty(B, 16, 64, 64, 8, device=dev)

    def launch(x, cin, packed, y, ys, out_f32):
        wp, bias, O, cop = packed
        return lambda: capi.check(L.r3dp_mf_conv3d(capi.ptr(x, f16), x.shape[-1], x.shape[-1], cin, capi.ptr(wp, f16), capi.ptr(bias), None, B, 16, 64, 64,
                                                   7, 7, 7, 0, O, cop, 0, capi.ptr(y, torch.float32 if out_f32 else f16), ys, 0, 0, out_f32, 0,
                                                   capi.stream()))
    for name, fn, gflop, byts in (('fuser', launch(xf, w.CF, w.fuser, fx, 32, 0), 2.0 * 89 * 32 * 343 * B * 16 * 4096 / 1e9,
                                   B * 16 * 4096 * 343 * w.CF * 2),
                                  ('mask', launch(fx, 32, w.mask, logits, 8, 1), 2.0 * 32 * 5 * 343 * B * 16 * 4096 / 1e9, B * 16 * 4096 * 343 * 32 * 2)):
        ms = statistics.median([time_ms(fn, args.iters) for _ in range(args.reps)])
        out[f'launch_{name}'] = {'ms': ms, 'gflop': gflop, 'tflops': gflop / ms, 'l2_operand_gb': byts / 1e9, 'l2_operand_tb_s': byts / 1e9 / ms}
    return out


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
    for arm in ('torch', 'cuda_uncached', 'cuda_cached', 'cuda_motion'):
        eng = engine.FrameEngine(batch=B, sr_mode='tc', hp=dict(syn.WARP_HPARAMS, num_samples_fine=48), torso_model=twr.randomize(Warp('standard'), 41),
                                 torso_stage2='torch' if arm == 'torch' else 'cuda', out_uint8=True,
                                 torso_motion='cuda' if arm == 'cuda_motion' else 'torch')
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
    out = {'batch': args.batch, 'stage2': stage2_arms(args, clocks), 'motion': motion_arms(args, clocks)}
    if args.engine:
        out['engine'] = engine_arms(args, clocks)
    out['clocks'] = clocks
    print(json.dumps(out))


if __name__ == '__main__':
    main()
