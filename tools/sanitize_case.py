"""Small end-to-end case for compute-sanitizer (memcheck / racecheck are ~100x slower: tiny shapes).
    compute-sanitizer --tool memcheck python tools/sanitize_case.py
Covers: streaming render kernel (single pass), two-pass tensor-core render kernel, tri-grid variant, tensor-core SR (all four conv launches,
FIR, edge) with fp16 and with split operands, uint8 epilogue, stand-alone sampler, the torso head (`warp`: alpha-cat / blend kernels, plain convs,
SynthesisBlockNoUp tail, per-clip cache) and large_sr (`large`: residual epilogue, plain ToRGB), both in 'tc' and 'tc_exact'.
`torso_engine`: the torso head's one-launch input kernel (64^2 and 128^2 sources, both split values) and one FrameEngine step of the torso
head with uint8 frames per warper setting (split graphs, whole graph).
`torso_nofuse`: the unweighted three-way concat (shared and per-frame third operand, both split values) and one FrameEngine step at batch 2 of
the weight_fuse=False head (block1 without a skip image) per sr_mode, with uint8 frames."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import real3dportrait_b200 as r3                                   # noqa: E402
from real3dportrait_b200 import synthetic as syn                   # noqa: E402


def main():
    dev = 'cuda'
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(1)
    what = sys.argv[1] if len(sys.argv) > 1 else 'all'
    dec = r3.OSGDecoder(32, {'decoder_lr_mul': 1, 'decoder_output_dim': 32})
    dec.load_state_dict(syn.make_decoder_params(seed=4), strict=True)
    dec = dec.to(dev).eval()
    if what in ('all', 'render'):
        N, res = 1, 16
        planes = torch.randn(N, 3, 32, 24, 24, generator=g).to(dev)
        cam = syn.make_cameras(N, seed=2).to(dev)
        o, d = r3.RaySampler()(cam[:, :16].reshape(-1, 4, 4), cam[:, 16:25].reshape(-1, 3, 3), res)
        for S, Si in ((12, 0), (12, 12)):
            u_c, u_f = syn.make_jitter(N, res * res, S, Si, seed=3)
            opts = dict(syn.RENDERING_OPTIONS, depth_resolution=S, depth_resolution_importance=Si, u_coarse=u_c.to(dev), u_fine=None if u_f is None else u_f.to(dev))
            out = r3.ImportanceRenderer()(planes, dec, o, d, opts)
            torch.cuda.synchronize()
            print('render', S, Si, float(out[0].abs().mean()))
        grids = torch.randn(N, 3, 96, 16, 16, generator=g).to(dev)
        hp = {'enable_rescale_plane_regulation': False, 'triplane_feature_type': 'trigrid_v2', 'triplane_depth': 3}
        u_c, _ = syn.make_jitter(N, res * res, 12, 0, seed=3)
        out = r3.ImportanceRenderer(hp=hp)(grids, dec, o, d, dict(syn.RENDERING_OPTIONS, depth_resolution=12, u_coarse=u_c.to(dev)))
        torch.cuda.synchronize()
        print('trigrid', float(out[0].abs().mean()))
    if what in ('all', 'sample'):
        planes = torch.randn(2, 3, 32, 24, 24, generator=g).to(dev)
        coords = (torch.rand(2, 1000, 3, generator=g) * 1.4 - 0.7).to(dev)                 # some points outside the box
        f = r3.sample_from_planes(None, planes, coords, box_warp=1.0)
        torch.cuda.synchronize()
        print('sample', float(f.abs().mean()))
    for mode in (('tc', 'tc_exact') if what == 'all' else (('tc',) if what == 'sr' else (('tc_exact',) if what == 'sr_exact' else ()))):
        sr = r3.SuperresolutionHybrid8XDC(channels=32, img_resolution=512, sr_num_fp16_res=0, sr_antialias=True, sr_mode=mode)
        sr.load_state_dict(syn.make_sr_params(seed=5), strict=True)
        sr = sr.to(dev).eval()
        fimg = (torch.rand(1, 32, 64, 64, generator=g) * 2 - 1).to(dev)
        for u8 in (False, True):
            img = sr(fimg[:, :3].contiguous(), fimg, torch.ones(1, 14, 512, device=dev), noise_mode='none', out_uint8=u8)
            torch.cuda.synchronize()
            print('sr', mode, u8, float(img.float().abs().mean()))
    for mode in (('tc', 'tc_exact') if what in ('all', 'warp') else ()):
        m = r3.SuperresolutionHybrid8XDC_Warp(channels=32, img_resolution=512, sr_num_fp16_res=0, sr_antialias=True, hp=syn.WARP_HPARAMS, sr_mode=mode,
                                              torso_model=syn.StubTorsoModel())
        m.load_state_dict(syn.make_sr_warp_params(seed=6), strict=True)
        m = m.to(dev).eval()
        fimg = (torch.rand(1, 32, 64, 64, generator=g) * 2 - 1).to(dev)
        wimg = torch.rand(1, 1, 64, 64, generator=g).to(dev)
        inp = {k: v.to(dev) for k, v in syn.make_warp_inputs(1, seed=7).items()}
        args = (fimg[:, :3].contiguous(), fimg, torch.ones(1, 14, 512, device=dev), inp['ref_torso_rgb'], inp['ref_bg_rgb'], wimg, inp['segmap'],
                inp['kp_s'], inp['kp_d'])
        with torch.no_grad():
            img, _ = m(*args, noise_mode='none')
            m.begin_clip(inp['ref_torso_rgb'], inp['ref_bg_rgb'])
            img_c, _ = m(*args, noise_mode='none')
            m.end_clip()
        torch.cuda.synchronize()
        print('warp', mode, float(img.abs().mean()), float(img_c.abs().mean()))
    if what in ('all', 'torso_engine'):
        from real3dportrait_b200 import _capi as capi, engine
        for res in (64, 128):
            for split in (0, 1):
                N, C = 1, 32
                x = torch.randn(N, res, res, C, generator=g).to(dev)
                w = torch.rand(N, res * res, 1, generator=g).to(dev)
                y = torch.empty(N, 128, 128, 64 * (1 + split), device=dev, dtype=torch.float16)
                rgb0, rgb256, w256 = torch.empty(N, 3, 128, 128, device=dev), torch.empty(N, 3, 256, 256, device=dev), torch.empty(N, 1, 256, 256, device=dev)
                capi.check(capi.lib().r3dp_sr_warp_input(capi.ptr(x), capi.ptr(w), N, C, res, res, 128, capi.ptr(y, torch.float16), capi.ptr(rgb0),
                                                         capi.ptr(rgb256), capi.ptr(w256), split, capi.stream()))
                torch.cuda.synchronize()
                print('warp_input', res, split, float(rgb256.abs().mean()), float(w256.mean()))
        inp = {k: v.to(dev) for k, v in syn.make_warp_inputs(1, seed=7).items()}
        for in_graph in (False, True):
            eng = engine.FrameEngine(batch=1, sr_mode='tc', hp=dict(syn.WARP_HPARAMS, num_samples_fine=0), torso_model=syn.StubTorsoModel(),
                                     out_uint8=True, warper_in_graph=in_graph)
            eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_warp_params(seed=6))
            eng.begin_clip(inp['ref_torso_rgb'], inp['ref_bg_rgb'], inp['segmap'], inp['kp_s'])
            planes, cam = syn.make_planes(1, seed=3).to(dev), syn.make_cameras(1, seed=4).to(dev)
            u_c, _ = syn.make_jitter(1, 4096, 48, 0, seed=5)
            out = eng.step(planes, cam, u_c.to(dev), kp_d=inp['kp_d'])
            torch.cuda.synchronize()
            print('torso_engine', in_graph, eng.graph is not None, float(out.float().mean()))
    if what in ('all', 'torso_nofuse'):
        from real3dportrait_b200 import _capi as capi, engine
        for split in (0, 1):
            wide = 1 + split
            N, H, W = 2, 3, 5
            xs = [torch.randn(n, H, W, 256 * wide, generator=g).half().to(dev) for n in (N, N, N, 1)]
            out = torch.empty(N, H, W, 768 * wide, device=dev, dtype=torch.float16)
            fn = capi.lib().r3dp_sr_tcx_cat3 if split else capi.lib().r3dp_sr_cat3
            for xc in (xs[2], xs[3]):
                capi.check(fn(capi.ptr(xs[0], torch.float16), 256, 256 * wide, capi.ptr(xs[1], torch.float16), 256, 256 * wide, capi.ptr(xc, torch.float16),
                              256, 256 * wide, int(xc.shape[0] == 1), N, H, W, capi.ptr(out, torch.float16), capi.stream()))
                torch.cuda.synchronize()
                print('cat3', split, xc.shape[0], float(out.float().abs().mean()))
        inp = {k: v.to(dev) for k, v in syn.make_warp_inputs(1, seed=7).items()}
        for mode in ('tc', 'tc_exact'):
            eng = engine.FrameEngine(batch=2, sr_mode=mode, hp=dict(syn.WARP_HPARAMS, num_samples_fine=0, weight_fuse=False), torso_model=syn.StubTorsoModel(),
                                     out_uint8=True)
            eng.load_params(syn.make_decoder_params(seed=4), syn.make_sr_warp_params(seed=6, weight_fuse=False))
            eng.begin_clip(inp['ref_torso_rgb'], inp['ref_bg_rgb'], inp['segmap'], inp['kp_s'])
            planes, cam = syn.make_planes(2, seed=3).to(dev), syn.make_cameras(2, seed=4).to(dev)
            u_c, _ = syn.make_jitter(2, 4096, 48, 0, seed=5)
            out = eng.step(planes, cam, u_c.to(dev), kp_d=inp['kp_d'].expand(2, -1, -1).contiguous())
            torch.cuda.synchronize()
            print('torso_nofuse', mode, eng.graph is not None, float(out.float().mean()))
    for mode in (('tc', 'tc_exact') if what in ('all', 'large') else ()):
        sr = r3.SuperresolutionHybrid8XDC(channels=32, img_resolution=512, sr_num_fp16_res=0, sr_antialias=True, large_sr=True, sr_mode=mode,
                                          resblocks_in_large_sr=1)
        sr.load_state_dict(syn.make_sr_large_params(seed=8, n_res=1), strict=True)
        sr = sr.to(dev).eval()
        fimg = (torch.rand(1, 32, 64, 64, generator=g) * 2 - 1).to(dev)
        img = sr(fimg[:, :3].contiguous(), fimg, torch.ones(1, 14, 512, device=dev), noise_mode='none')
        torch.cuda.synchronize()
        print('large', mode, float(img.abs().mean()))


if __name__ == '__main__':
    main()
