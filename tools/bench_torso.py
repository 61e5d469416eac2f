"""BASELINE configs[4] in both tensor-core SR modes: 48 + 48 samples/ray -> SuperresolutionHybrid8XDC_Warp (fuse mode v2, stub torso warper),
per-clip constants cached with begin_clip(), one CUDA graph per resident batch.

    python tools/bench_torso.py [--modes tc tc_exact] [--batch 4] [--steps 16] [--warmup 3] [--reps 3] [--no-weight-fuse]

The modes are timed alternately, --reps times each; the JSON line carries every rep and the median frames/s per mode, with the card's name,
power limit and the SM clock sampled during the timed runs (a power-capped card lowers its clocks under this load).  The timing loop and the
graph pool are bench.py's, so the numbers are comparable with its roofline.extra.configs entry for configs[4] in 'tc'.

    python tools/bench_torso.py --engine [--frames 512] [--batch 4] [--reps 3]
    python -m torch.distributed.run --nproc-per-node 8 tools/bench_torso.py --engine --frames 512

--engine times configs[4] as a clip through FrameEngine(torso_model=...) in 'tc': --frames uint8 frames, sharded over the ranks, pushed into
the clip on rank 0 (exchange='p2p'), with the warper run eagerly between two graphs and with the warper inside one graph, alternating with
the GraphPool loop above (one GPU per rank, fp32 frames, no clip).  Each reports the median of --reps clips; frames/s counts the whole clip.

--no-weight-fuse times the head's weight_fuse=False configuration instead of fuse mode v2 (sr_with_ref.py:158-161)."""
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


def _card(dev):
    props = torch.cuda.get_device_properties(dev)
    try:
        import subprocess
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', str(dev.index)], capture_output=True, text=True,
                               timeout=20).stdout.strip()
    except Exception as e:                                                    # noqa: BLE001
        power = f'unavailable ({type(e).__name__})'
    return props.name, power


def _fuse(args) -> str:
    return 'fuse v2' if args.weight_fuse else 'weight_fuse=False'


def engine_main(args):
    """configs[4] as a clip through FrameEngine(torso_model=stub): uint8 frames, p2p clip exchange, both warper settings, alternating with
    the GraphPool loop of main()."""
    from real3dportrait_b200 import engine
    import torch.distributed as dist
    rank, world, local = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1)), int(os.environ.get('LOCAL_RANK', 0))
    dev = torch.device('cuda', local)
    torch.cuda.set_device(dev)
    if world > 1:
        dist.init_process_group('nccl', device_id=dev)
    barrier = (lambda: (torch.cuda.synchronize(), dist.barrier())) if world > 1 else torch.cuda.synchronize
    bench = _bench_module()
    B = args.batch
    fpr = args.frames // world
    steps = fpr // B
    assert steps >= 1 and fpr % B == 0, 'frames per rank must be a multiple of --batch'
    nb = max(args.pool // B, 1)
    P = nb * B
    sl = lambda i: slice((i % nb) * B, (i % nb) * B + B)
    planes_cl = ren.planes_to_channels_last(syn.make_planes(P, seed=100 + rank).to(dev)).data
    cams = syn.make_cameras(P, seed=200 + rank).to(dev)
    u_c, u_f = (u.to(dev) for u in syn.make_jitter(P, 4096, 48, 48, seed=300 + rank))
    kp_d = (torch.rand(P, 68, 3, generator=torch.Generator().manual_seed(9 + rank)) * 2 - 1).to(dev)
    resident = [(ren.PlanesCL(planes_cl[sl(i)]), cams[sl(i)], u_c[sl(i)], u_f[sl(i).start * 4096:sl(i).stop * 4096], kp_d[sl(i)]) for i in range(nb)]
    inp = {k: v.to(dev) for k, v in syn.make_warp_inputs(1, seed=7).items()}
    consts = (inp['ref_torso_rgb'], inp['ref_bg_rgb'], inp['segmap'], inp['kp_s'])
    dec, srp = syn.make_decoder_params(seed=4), syn.make_sr_warp_params(seed=6, weight_fuse=args.weight_fuse)
    hp = dict(syn.WARP_HPARAMS, num_samples_fine=48, weight_fuse=args.weight_fuse)

    runs = {}
    for name, in_graph in (('engine_split_graphs', False), ('engine_whole_graph', True)):
        eng = engine.FrameEngine(batch=B, sr_mode='tc', device=dev, world=world, rank=rank, dist=dist if world > 1 else None, hp=hp,
                                 torso_model=syn.StubTorsoModel(), out_uint8=True, exchange='p2p', warper_in_graph=in_graph)
        eng.load_params(dec, srp)
        eng.begin_clip(*consts)
        eng.prepare(resident)

        def clip(eng=eng):
            eng.open_clip(fpr)
            for s in range(steps):
                pl, cm, uc, uf, kd = resident[s % nb]
                eng.step(pl, cm, uc, uf, frame_index=s * B, kp_d=kd)
            eng.close_clip()
        runs[name] = clip

    head = r3.RenderHead(hp=hp, torso_model=syn.StubTorsoModel(), sr_mode='tc')
    head.load_state_dict({**{'decoder.' + k: v for k, v in dec.items()}, **{'superresolution.' + k: v for k, v in srp.items()}}, strict=True)
    head = head.to(dev).eval()
    head.superresolution.assume_shared_styles = True
    head.superresolution.begin_clip(inp['ref_torso_rgb'], inp['ref_bg_rgb'])
    cond_static = {'ref_torso_img': inp['ref_torso_rgb'].expand(B, -1, -1, -1).contiguous(), 'bg_img': inp['ref_bg_rgb'].expand(B, -1, -1, -1).contiguous(),
                   'segmap': inp['segmap'].expand(B, -1, -1, -1).contiguous(), 'kp_s': inp['kp_s'].expand(B, -1, -1).contiguous()}

    def step(i):
        pl, cm, uc, uf, kd = resident[i % nb]
        return head.synthesis(pl, cm, cond=dict(cond_static, kp_d=kd), u_coarse=uc, u_fine=uf)['image']
    pool = bench.GraphPool(step, nb)
    runs['graphpool'] = lambda: [pool(i) for i in range(steps)]

    for fn in runs.values():                                                  # warm-up: one clip each
        fn()
    barrier()
    sampler = bench.ClockSampler(local)
    sampler.start()
    ms = {k: [] for k in runs}
    for _ in range(args.reps):
        for name, fn in runs.items():
            barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            barrier()
            t = torch.tensor([e0.elapsed_time(e1)], device=dev, dtype=torch.float64)
            if world > 1:
                dist.all_reduce(t, op=dist.ReduceOp.MAX)
            ms[name].append(float(t.item()))
    clocks = sampler.summary()
    name_, power = _card(dev)
    if rank == 0:
        out = {'config': f'configs[4] clip: 48+48 samples/ray + SuperresolutionHybrid8XDC_Warp ({_fuse(args)}, stub torso warper), tc, uint8 frames, p2p clip',
               'frames': fpr * world, 'gpus': world, 'batch': B, 'reps': args.reps, 'device': name_, 'power_limit': power, 'clocks': clocks,
               'graphpool_note': 'GraphPool: the same frames per GPU without clip, exchange or uint8 frames', 'runs': {}}
        for name, v in ms.items():
            med = statistics.median(v)
            out['runs'][name] = {'frames_per_s': fpr * world / (med / 1e3), 'ms_per_clip': med, 'ms_per_clip_reps': v}
        print(json.dumps(out))
    if world > 1:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--engine', action='store_true', help='time configs[4] as a clip through FrameEngine (see the module docstring)')
    ap.add_argument('--frames', type=int, default=512, help='--engine: frames per clip (all ranks)')
    ap.add_argument('--modes', nargs='+', default=['tc', 'tc_exact'], choices=['tc', 'tc_exact'])
    ap.add_argument('--batch', type=int, default=4)
    ap.add_argument('--pool', type=int, default=16, help='distinct resident frames (cycled in batches)')
    ap.add_argument('--steps', type=int, default=16)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--no-weight-fuse', dest='weight_fuse', action='store_false', help='the weight_fuse=False head instead of fuse mode v2')
    args = ap.parse_args()
    if args.engine:
        return engine_main(args)
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
    sd.update({'superresolution.' + k: v for k, v in syn.make_sr_warp_params(seed=6, weight_fuse=args.weight_fuse).items()})

    pools = {}
    for mode in args.modes:
        head = r3.RenderHead(hp=dict(syn.WARP_HPARAMS, num_samples_fine=48, weight_fuse=args.weight_fuse), torso_model=syn.StubTorsoModel(), sr_mode=mode)
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
    out = {'config': f"configs[4]: 48+48 samples/ray + SuperresolutionHybrid8XDC_Warp ({_fuse(args)}, stub torso warper), begin_clip() cache, CUDA graphs",
           'batch': B, 'steps': args.steps, 'reps': args.reps, 'device': props.name, 'power_limit': power, 'clocks': clocks, 'modes': {}}
    for mode, v in ms.items():
        med = statistics.median(v)
        out['modes'][mode] = {'frames_per_s': B / (med / 1e3), 'ms_per_step': med, 'ms_per_step_reps': v}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
