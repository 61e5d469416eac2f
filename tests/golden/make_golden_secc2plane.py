"""Generate tests/golden/secc2plane_small.npz by running the REFERENCE's own SegFormerSECC2PlaneBackbone (modules/real3d/segformer.py:673-733)
on seeded synthetic parameters and inputs, in float64 on the CPU.

    R3DP_REFERENCE=<reference checkout> python tests/golden/make_golden_secc2plane.py

timm and mmcv are not needed: tests/secc2plane_reference.py puts minimal shims for what segformer.py imports in sys.modules first, and
torch.load returns an empty state_dict for the missing mit_b0.pth while the class is built (every weight comes from the seeded set, loaded
with strict=True).  The shim's mmcv ConvModule is a bias-free Conv2d -> BatchNorm2d `bn` -> ReLU (mmcv's bias='auto' with a norm), so the
fixture pins fuse_head.linear_fuse to that reading of mmcv.

Stored: the planes [1,3,32,64,64] of a 128^2 'cano_src_tgt' input on every second row and column (`planes_s2`, float32), plus the seeds;
the parameters and inputs are regenerated from the seeds (make_params / make_inputs)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if not os.environ.get('R3DP_REFERENCE'):
    sys.exit('set R3DP_REFERENCE to a checkout of the reference project')
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import secc2plane_reference as ref  # noqa: E402

PARAM_SEED, INPUT_SEED, H = 7, 11, 128


def main():
    torch.set_grad_enabled(False)
    Ref = ref.reference_class(os.environ['R3DP_REFERENCE'])
    m = Ref(mode='b0', out_channels=96, pncc_cond_mode='cano_src_tgt').eval()
    sd = ref.make_params({k: v.shape for k, v in m.state_dict().items()}, PARAM_SEED)
    m.load_state_dict(sd, strict=True)
    cano, src, tgt = ref.make_inputs(1, H, INPUT_SEED)
    x = torch.cat([cano, src, tgt], 1)
    m = m.double()
    m.prenet.resample_filter = m.prenet.resample_filter.float()     # conv2d_resample.py:77 asserts an fp32 filter (unused by a 1x1 layer)
    planes = m(x.double())
    out = os.path.join(HERE, 'secc2plane_small.npz')
    np.savez_compressed(out, planes_s2=planes[..., ::2, ::2].float().numpy(), param_seed=np.int64(PARAM_SEED), input_seed=np.int64(INPUT_SEED),
                        size=np.int64(H))
    print(out, os.path.getsize(out), 'bytes')


if __name__ == '__main__':
    main()
