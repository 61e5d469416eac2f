"""BASELINE configs[4] in both tensor-core SR modes: 48 + 48 samples/ray -> SuperresolutionHybrid8XDC_Warp (fuse mode v2, stub torso warper),
per-clip constants cached with begin_clip(), one CUDA graph per resident batch.

    python tools/bench_torso.py [--modes tc tc_exact] [--batch 4] [--steps 16] [--warmup 3] [--reps 3]

The modes are timed alternately, --reps times each; the JSON line carries every rep and the median frames/s per mode, with the card's name,
power limit and the SM clock sampled during the timed runs (a power-capped card lowers its clocks under this load).  The timing loop and the
graph pool are bench.py's, so the numbers are comparable with its roofline.extra.configs entry for configs[4] in 'tc'."""
import argparse
import importlib.util
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import real3dportrait_b200 as r3                                          # noqa: E402
from real3dportrait_b200 import synthetic as syn, renderer as ren          # noqa: E402


def _bench_module():
    spec = importlib.util.spec_from_file_location('r3dp_bench', os.path.join(ROOT, 'bench.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--modes', nargs='+', default=['tc', 'tc_exact'], choices=['tc', 'tc_exact'])
    ap.add_argument('--batch', type=int, default=4)
    ap.add_argument('--pool', type=int, default=16, help='distinct resident frames (cycled in batches)')
    ap.add_argument('--steps', type=int, default=16)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    bench = _bench_module()
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    B, P = args.batch, max(args.pool, args.batch)
    nb = P // B
    sl = lambda i: slice((i % nb) * B, (i % nb) * B + B)
    planes_cl = ren.planes_to_channels_last(syn.make_planes(P, seed=100).to(dev)).data
    cams = syn.make_cameras(P, seed=200).to(dev)
    u_c, u_f = (u.to(dev) for u in syn.make_jitter(P, 4096, 48, 48, seed=300))
    resident = [(ren.PlanesCL(planes_cl[sl(i)]), cams[sl(i)], u_c[sl(i)], u_f[sl(i).start * 4096:sl(i).stop * 4096]) for i in range(nb)]
    inp = {k: v.to(dev) for k, v in syn.make_warp_inputs(1, seed=7).items()}
    kp_d = (torch.rand(P, 68, 3, generator=torch.Generator().manual_seed(9)) * 2 - 1).to(dev)
    cond_static = {'ref_torso_img': inp['ref_torso_rgb'].expand(B, -1, -1, -1).contiguous(), 'bg_img': inp['ref_bg_rgb'].expand(B, -1, -1, -1).contiguous(),
                   'segmap': inp['segmap'].expand(B, -1, -1, -1).contiguous(), 'kp_s': inp['kp_s'].expand(B, -1, -1).contiguous()}
    sd = {'decoder.' + k: v for k, v in syn.make_decoder_params(seed=4).items()}
    sd.update({'superresolution.' + k: v for k, v in syn.make_sr_warp_params(seed=6).items()})

    pools = {}
    for mode in args.modes:
        head = r3.RenderHead(hp=dict(syn.WARP_HPARAMS, num_samples_fine=48), torso_model=syn.StubTorsoModel(), sr_mode=mode)
        head.load_state_dict(sd, strict=True)
        head = head.to(dev).eval()
        head.superresolution.assume_shared_styles = True
        head.superresolution.begin_clip(inp['ref_torso_rgb'], inp['ref_bg_rgb'])

        def step(i, head=head):
            pl, cm, uc, uf = resident[i % nb]
            return head.synthesis(pl, cm, cond=dict(cond_static, kp_d=kp_d[sl(i)]), u_coarse=uc, u_fine=uf)['image']
        pools[mode] = (head, bench.GraphPool(step, nb))

    sampler = bench.ClockSampler(0)
    sampler.start()
    ms = {m: [] for m in args.modes}
    for _ in range(args.reps):
        for mode in args.modes:
            t = bench.timed_loop(pools[mode][1], args.steps, args.warmup, torch.cuda.synchronize, None, dev)
            ms[mode].append(t / args.steps)
    clocks = sampler.summary()
    for head, _ in pools.values():
        head.superresolution.end_clip()
    props = torch.cuda.get_device_properties(dev)
    try:
        import subprocess
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True, text=True,
                               timeout=20).stdout.strip()
    except Exception as e:                                                    # noqa: BLE001
        power = f'unavailable ({type(e).__name__})'
    out = {'config': "configs[4]: 48+48 samples/ray + SuperresolutionHybrid8XDC_Warp (fuse v2, stub torso warper), begin_clip() cache, CUDA graphs",
           'batch': B, 'steps': args.steps, 'reps': args.reps, 'device': props.name, 'power_limit': power, 'clocks': clocks, 'modes': {}}
    for mode, v in ms.items():
        med = statistics.median(v)
        out['modes'][mode] = {'frames_per_s': B / (med / 1e3), 'ms_per_step': med, 'ms_per_step_reps': v}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
