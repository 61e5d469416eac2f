"""Multi-GPU check of the clip exchange paths (run under torchrun, one rank per GPU):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 tools/check_exchange.py

Every rank renders `steps` batches of its own frames; with exchange='p2p' the frames are pushed by the copy engine into the clip on rank 0
(CUDA IPC mapping), with exchange='allgather' NCCL gathers them.  Rank 0 then compares the assembled clip with the frames every rank kept
locally (sent through an independent NCCL gather at the end) - bit for bit - and prints the per-step cost of both exchanges.
With --torso the engines run the torso head (synthetic.StubTorsoModel as the warper, the clip constants of begin_clip(), kp_d per frame);
--no-weight-fuse runs its weight_fuse=False configuration and --torso-v1 its torso_model_version 'v1' (synthetic.StubTorsoModelV1); either implies
--torso.
With --concat-debug the engines run the secc2plane head with out_mode='concat_debug' (exchange='p2p'): rank 0's clip of debug strips, whose
depth panel is normalised over every rank's frames, must equal the clip one GPU renders from the same frames alone."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from real3dportrait_b200 import engine, renderer as ren, synthetic as syn   # noqa: E402


def concat_debug(rank, world, dev):
    """Rank 0's concat_debug clip at `world` GPUs == the clip of a single-GPU engine over every rank's frames, bit for bit."""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))
    import real3dportrait_b200 as r3
    import secc2plane_reference as s2p_ref
    B, steps = 4, 3

    def make(**kw):
        bb = r3.SegFormerSECC2PlaneBackbone()
        bb.load_state_dict(s2p_ref.make_params({k: v.shape for k, v in bb.state_dict().items()}, 7), strict=True)
        eng = engine.FrameEngine(batch=B, sr_mode='tc', device=dev, hp={'num_samples_fine': 0}, secc2plane=bb, out_uint8=True,
                                 out_mode='concat_debug', **kw)
        eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_params(seed=5))
        c = s2p_ref.make_inputs(1, 512, 1)
        eng.begin_planes(syn.make_planes(1, seed=1).to(dev), c[0].to(dev), c[1].to(dev))
        return eng

    def frames_of(r, s):
        tgt = s2p_ref.make_inputs(B, 512, 100 * r + s)[2].to(dev)
        return tgt, syn.make_cameras(B, seed=100 * r + s + 50).to(dev), syn.make_jitter(B, 4096, 48, 0, seed=100 * r + s + 70)[0].to(dev)
    ref_gt = ((torch.randint(0, 256, (1, 3, 512, 512), generator=torch.Generator().manual_seed(5)).float() - 127.5) / 127.5).to(dev)
    eng = make(world=world, rank=rank, dist=dist, exchange='p2p')
    eng.open_clip(steps * B, ref_gt_img=ref_gt)
    for s in range(steps):
        tgt, cams, u = frames_of(rank, s)
        eng.step(None, cams, u, cond_tgt=tgt, frame_index=s * B)
    clip = eng.close_clip()
    ok = True
    if rank == 0:
        one = make()
        one.open_clip(world * steps * B, ref_gt_img=ref_gt)
        for r in range(world):
            for s in range(steps):
                tgt, cams, u = frames_of(r, s)
                one.step(None, cams, u, cond_tgt=tgt, frame_index=(r * steps + s) * B)
        ok = torch.equal(clip, one.close_clip())
        print(f'concat_debug world={world}: rank 0 clip == single-GPU clip: {ok}')
    dist.barrier()
    return ok


def main():
    rank, world, local = int(os.environ['RANK']), int(os.environ['WORLD_SIZE']), int(os.environ['LOCAL_RANK'])
    torch.cuda.set_device(local)
    dev = torch.device('cuda', local)
    dist.init_process_group('nccl', device_id=dev)
    if '--concat-debug' in sys.argv[1:]:
        ok = concat_debug(rank, world, dev)
        if rank == 0:
            print('EXCHANGE_OK' if ok else 'EXCHANGE_MISMATCH')
        dist.destroy_process_group()
        return
    cfg = {}
    if '--no-weight-fuse' in sys.argv[1:]:
        cfg['weight_fuse'] = False
    if '--torso-v1' in sys.argv[1:]:
        cfg['torso_model_version'] = 'v1'
    torso = '--torso' in sys.argv[1:] or bool(cfg)
    B, steps = 4, 6
    planes = ren.planes_to_channels_last(syn.make_planes(B * 2, seed=10 + rank).to(dev)).data
    cams = syn.make_cameras(B * 2, seed=20 + rank).to(dev)
    u = syn.make_jitter(B * 2, 4096, 48, 0, seed=30 + rank)[0].to(dev)
    res = [(ren.PlanesCL(planes[i * B:(i + 1) * B]), cams[i * B:(i + 1) * B], u[i * B:(i + 1) * B]) for i in range(2)]
    kw, kp_d = {}, [None, None]
    if torso:
        kp = (torch.rand(B * 2, 68, 3, generator=torch.Generator().manual_seed(40 + rank)) * 2 - 1).to(dev)
        kp_d = [kp[i * B:(i + 1) * B] for i in range(2)]
        res = [r + (None, kp_d[i]) for i, r in enumerate(res)]
        kw = {'torso_model': syn.StubTorsoModelV1() if 'torso_model_version' in cfg else syn.StubTorsoModel()}
        consts = syn.make_warp_inputs(1, seed=7)
    ok = True
    for u8 in (True, False):
        for mode in ('p2p', 'allgather'):
            hp = dict(syn.WARP_HPARAMS, num_samples_fine=0, **cfg) if torso else {'num_samples_fine': 0}
            eng = engine.FrameEngine(batch=B, sr_mode='tc', device=dev, world=world, rank=rank, dist=dist, hp=hp, out_uint8=u8, exchange=mode, **kw)
            eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_warp_params(seed=6, weight_fuse=cfg.get('weight_fuse', True)) if torso else syn.make_sr_params(seed=5))
            if torso:
                eng.begin_clip(*(consts[k].to(dev) for k in ('ref_torso_rgb', 'ref_bg_rgb', 'segmap', 'kp_s')))
            eng.prepare(res)
            clip = eng.open_clip(steps * B) if mode == 'p2p' else None
            local_frames, gathered = [], []
            torch.cuda.synchronize(); dist.barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for s in range(steps):
                out = eng.step(*res[s % 2][:3], frame_index=s * B, **({'kp_d': kp_d[s % 2]} if torso else {}))
                if mode == 'allgather':
                    eng.wait_gather()
                    gathered.append(out.clone())
                    local_frames.append(out[rank * B:(rank + 1) * B].clone())
                else:
                    local_frames.append(out.clone())
            eng.wait_gather()
            e1.record()
            if mode == 'p2p':
                clip = eng.close_clip()
            torch.cuda.synchronize(); dist.barrier()
            mine = torch.cat(local_frames)                                            # [steps*B, ...]
            everyone = [torch.empty_like(mine) for _ in range(world)]
            dist.all_gather(everyone, mine)
            if rank == 0:
                want = torch.cat(everyone)                                            # rank-major: rank r's frame f at r*steps*B + f
                if mode == 'p2p':
                    good = torch.equal(clip, want)
                else:
                    got = torch.cat([torch.cat([g[r * B:(r + 1) * B] for g in gathered]) for r in range(world)])
                    good = torch.equal(got, want)
                ok = ok and good
                print(f'exchange={mode:9s} frames={"uint8" if u8 else "fp32 "} world={world}: clip == per-rank frames: {good}; '
                      f'{e0.elapsed_time(e1) / steps:.3f} ms/step (compute + exchange, {steps} steps)')
            del eng
    if rank == 0:
        print('EXCHANGE_OK' if ok else 'EXCHANGE_MISMATCH')
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
