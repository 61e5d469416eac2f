"""Small end-to-end case for compute-sanitizer (memcheck / racecheck are ~100x slower: tiny shapes).
    compute-sanitizer --tool memcheck python tools/sanitize_case.py
Covers: streaming render kernel (single pass), two-pass tensor-core render kernel, tri-grid variant, tensor-core SR (all four conv launches,
FIR, edge) with fp16 and with split operands, uint8 epilogue, stand-alone sampler."""
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


if __name__ == '__main__':
    main()
