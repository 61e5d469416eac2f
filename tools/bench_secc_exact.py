"""SegFormerSECC2PlaneBackbone in precision='tc_exact' on one GPU (512^2 SECC input, batch 4): its time and what it buys.

Prints one JSON line with the card's name, power limit and SM clocks read in the same call, and:
  backbone_ms     one forward per call, arms alternating, median of 3 CUDA-event windows: this library in `tc` and `tc_exact`, and PyTorch
                  running the same network (the float64-checked restatement tests/secc2plane_reference.py, fp32 nn ops) with torch's default
                  TF32 setting and with TF32 off (the fp32-grade alternative)
  accuracy        each arm's planes against the float64 restatement, max |err| / max |ref|
  clip_step_ms    FrameEngine(sr_mode='tc_exact', out_uint8=True, secc2plane=..., secc_renderer=...) fed coefficients, prepare()d graphs,
                  with a `tc` and a `tc_exact` backbone, alternating
  frame_error     the final image (sr_mode='tc_exact', fp32 frames in [-1, 1]) of the plain head fed (canonical, SECC) plane pairs, max |err|
                  against the same render + SR fed the float64 restatements' planes (Img2PlaneModel and the backbone, rounded to fp32), so the
                  render and SR are common to every arm and the difference is the plane networks' share:
                    a  tc backbone,       float64 canonical planes
                    b  tc_exact backbone, float64 canonical planes (begin_planes(cano_planes=...) with fp32 planes)
                    c  tc_exact backbone, Img2PlaneModel's tc canonical planes
                    d  tc backbone,       Img2PlaneModel's tc canonical planes (the default clip)

    python tools/bench_secc_exact.py [--batch 4] [--iters 20]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]
import img2plane_reference as iref  # noqa: E402
import secc2plane_reference as ref  # noqa: E402
import real3dportrait_b200 as r3  # noqa: E402
from real3dportrait_b200 import engine, synthetic as syn  # noqa: E402
from real3dportrait_b200.renderer import PlanesCL  # noqa: E402

DEV = 'cuda:0'


def _smi(q):
    return subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader', '-i', '0'], capture_output=True, text=True).stdout.strip()


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def alternate(arms, iters, clocks):
    """Warm every arm (with its own TF32 setting), then 3 rounds of the arms in turn -> {arm: {'ms': median, 'runs_ms': [...]}}."""
    res = {k: [] for k in arms}
    with torch.no_grad():
        for fn in arms.values():
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        for _ in range(3):
            for k, fn in arms.items():
                res[k].append(timed(fn, iters))
            clocks.append(_smi('clocks.sm'))
    return {k: {'ms': round(statistics.median(v), 3), 'runs_ms': [round(t, 3) for t in v]} for k, v in res.items()}


def backbone(precision, seed=7):
    m = r3.SegFormerSECC2PlaneBackbone(precision=precision)
    m.load_state_dict(ref.make_params({k: v.shape for k, v in m.state_dict().items()}, seed), strict=True)
    return m.to(DEV).eval()


def with_tf32(on, fn):
    def run():
        saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
        if on is not None:
            torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = on
        try:
            return fn()
        finally:
            torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved
    return run


def rel(got, want):
    return float((got.double() - want).abs().max()) / float(want.abs().max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=4)
    ap.add_argument('--iters', type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_secc_exact needs a CUDA device')
    B, H = args.batch, 512
    out = {'gpu': _smi('name,power.limit,clocks.sm,clocks.max.sm'), 'size': H, 'batch': B}
    clocks = []
    tc, ex = backbone('tc'), backbone('tc_exact')
    sd32 = {k: v.to(DEV) for k, v in tc.state_dict().items()}
    sd64 = ref.to64(sd32, DEV)
    cano, src, tgt = (t.to(DEV) for t in ref.make_inputs(B, H, 3))
    x = torch.cat([cano.expand(B, -1, -1, -1), src.expand(B, -1, -1, -1), tgt], 1).contiguous()

    # ---- the backbone per call
    arms = {'tc': lambda: tc(x), 'tc_exact': lambda: ex(x), 'torch_tf32_default': with_tf32(None, lambda: ref.forward(sd32, x)),
            'torch_tf32_off': with_tf32(False, lambda: ref.forward(sd32, x))}
    out['backbone_ms'] = alternate(arms, args.iters, clocks)
    with torch.no_grad():
        want = ref.forward(sd64, x.double())
        out['accuracy'] = {k: float(f'{rel(fn(), want):.3e}') for k, fn in arms.items()}
    del want

    # ---- the clip step fed coefficients, tc vs tc_exact backbone
    r = r3.SECC_Renderer(H, device=DEV, **syn.write_bfm_folder(tempfile.mkdtemp(prefix='r3dp_bfm_'), seed=0))
    cs = syn.make_coeffs(1, seed=2)
    coeff_src = torch.cat([cs['id'], cs['exp']], 1).to(DEV)
    drv = syn.make_coeffs(B, seed=3)
    coeff = torch.cat([drv['id'], drv['exp']], 1).to(DEV)
    cams = syn.make_cameras(B, seed=1).to(DEV)
    u_c = syn.make_jitter(B, 4096, 48, 0, seed=2)[0].to(DEV)
    cano_planes = syn.make_planes(1, seed=0).to(DEV)
    engines = {}
    for name, bb in (('tc_backbone', tc), ('tc_exact_backbone', ex)):
        e = engine.FrameEngine(batch=B, sr_mode='tc_exact', hp={'num_samples_fine': 0}, out_uint8=True, secc2plane=bb, secc_renderer=r)
        e.load_params(syn.make_decoder_params(seed=4), syn.make_sr_params(seed=5))
        with torch.no_grad():
            e.begin_planes(cano_planes, coeff_src=coeff_src)
            e.prepare([(coeff, cams, u_c)])
        engines[name] = e
    out['clip_step_ms'] = alternate({k: (lambda e=e: e.step(None, cams, u_c, coeff=coeff)) for k, e in engines.items()}, args.iters, clocks)
    del engines

    # ---- the final image's error from the plane networks
    i2p = r3.Img2PlaneModel()
    isd = iref.make_params({k: v.shape for k, v in i2p.state_dict().items()}, 5)
    i2p.load_state_dict(isd, strict=True)
    i2p = i2p.to(DEV).eval()
    img = iref.make_inputs(1, H, 11).to(DEV)
    EB = 2
    direct = engine.FrameEngine(batch=EB, sr_mode='tc_exact', hp={'num_samples_fine': 0}, out_uint8=False, use_graph=False)
    direct.load_params(syn.make_decoder_params(seed=4), syn.make_sr_params(seed=5))
    cams2, u2 = cams[:EB].contiguous(), syn.make_jitter(EB, 4096, 48, 0, seed=2)[0].to(DEV)
    with torch.no_grad():
        cano64 = iref.forward({k: (v.to(DEV, torch.float64) if v.is_floating_point() else v.to(DEV)) for k, v in isd.items()}, img.double())
        cano_ref = r3.canonical_planes_cl(cano64.float())
        cano_tc = r3.canonical_planes_cl(i2p(img))
        secc64 = ref.forward(sd64, x[:EB].double()).float()                       # [EB,3,32,256,256]
        secc_ref = PlanesCL(secc64.permute(0, 3, 4, 1, 2).contiguous(), 'hwpc')
        planes = {}
        for name, bb in (('tc', tc), ('tc_exact', ex)):
            bb.begin_clip(cano[:1], src[:1])
            planes[name] = bb.planes_cl(tgt[:EB].contiguous())
        want = direct.step((cano_ref, secc_ref), cams2, u2).double().clone()
        arms = {'a_tc_backbone_f64_cano': (cano_ref, planes['tc']), 'b_tc_exact_backbone_f64_cano': (cano_ref, planes['tc_exact']),
                'c_tc_exact_backbone_img2plane_tc_cano': (cano_tc, planes['tc_exact']), 'd_tc_backbone_img2plane_tc_cano': (cano_tc, planes['tc'])}
        err = {}
        for k, pair in arms.items():
            got = direct.step(pair, cams2, u2).double()
            err[k] = float(f'{float((got - want).abs().max()):.3e}')
        err['secc_planes_rel'] = {k: float(f'{rel(p.data.permute(0, 3, 4, 1, 2), secc64.double()):.3e}') for k, p in planes.items()}
        err['cano_planes_rel_img2plane_tc'] = float(f'{rel(i2p(img), cano64):.3e}')
        err['image_range'] = float(f'{float(want.abs().max()):.3e}')
    out['frame_error'] = err
    out['sm_clock_samples'] = clocks
    print(json.dumps(out))


if __name__ == '__main__':
    main()
