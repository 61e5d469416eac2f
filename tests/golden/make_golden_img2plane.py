"""Generate tests/golden/img2plane_small.npz by running the REFERENCE's own Img2PlaneModel (modules/img2plane/img2plane_model.py:12-81) on
seeded synthetic parameters and inputs, in float64 on the CPU.

    R3DP_REFERENCE=<reference checkout> python tests/golden/make_golden_img2plane.py

timm, pretrainedmodels and the global hparams are shimmed by tests/img2plane_reference.py, which also makes every socket connection raise
before the class is built; the constructor's ImageNet weights come from a locally built torchvision resnet34(weights=None) (every weight
is then replaced by the seeded set, loaded with strict=True).

Stored: the planes [1,3,32,64,64] of a 128^2 'rgb' input on every second row and column (`planes_s2`, float32), plus the seeds; the
parameters and input are regenerated from the seeds (make_params / make_inputs)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if not os.environ.get('R3DP_REFERENCE'):
    sys.exit('set R3DP_REFERENCE to a checkout of the reference project')
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import img2plane_reference as ref  # noqa: E402

PARAM_SEED, INPUT_SEED, H = 5, 9, 128
HP = {'img2plane_input_mode': 'rgb', 'img2plane_backbone_scale': 'standard', 'triplane_feature_type': 'triplane', 'triplane_depth': 1}


def main():
    torch.set_grad_enabled(False)
    Ref = ref.reference_class(os.environ['R3DP_REFERENCE'], HP)
    m = Ref(out_channels=96, hp=HP).eval()
    sd = ref.make_params({k: v.shape for k, v in m.state_dict().items()}, PARAM_SEED)
    m.load_state_dict(sd, strict=True)
    x = ref.make_inputs(1, H, INPUT_SEED)
    planes = m.double()(x.double())
    out = os.path.join(HERE, 'img2plane_small.npz')
    np.savez_compressed(out, planes_s2=planes[..., ::2, ::2].float().numpy(), param_seed=np.int64(PARAM_SEED), input_seed=np.int64(INPUT_SEED),
                        size=np.int64(H))
    print(out, os.path.getsize(out), 'bytes')


if __name__ == '__main__':
    main()
