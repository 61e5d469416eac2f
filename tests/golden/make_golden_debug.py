"""Generate tests/golden/debug_frames.npz by running the REFERENCE's own GeneFace2Infer.forward_secc2video (inference/real3d_infer.py),
unmodified, with inp['out_mode'] = 'concat_debug' and low_memory_usage = False, on the CPU:

    R3DP_REFERENCE=<reference checkout> python tests/golden/make_golden_debug.py

The method's model is a stub whose forward replays given {'image', 'image_raw', 'image_depth'} frame by frame; the frames the method
hands its imageio writer are captured.  What real3d_infer.py imports but this method does not use (mediapipe, torchshow, librosa, the
3DMM fit, the segmenter, the SECC renderer, deep_3drecon, ...) is replaced by stubs in sys.modules; numpy 2 gets the aliases the
reference's modules still name; imageio is a fake whose writer keeps the frames; os.system (the ffmpeg mux) does nothing and
Tensor.cuda is the identity.

Stored: the inputs as 64^2 fields (debug_frames_reference.quirk_inputs; the 512^2 tensors are their nearest x8 replication) and the
captured uint8 frames [N,512,2560,3], for the case 'quirks' (3 frames) and 'flat' (3 frames of constant depth: panel 3 is 0 / 0)."""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if not os.environ.get('R3DP_REFERENCE'):
    sys.exit('set R3DP_REFERENCE to a checkout of the reference project')
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import torch  # noqa: E402

from debug_frames_reference import full_inputs, quirk_inputs  # noqa: E402

CASES = [('quirks', 3, 0, False), ('flat', 3, 1, True)]          # (name, frames, seed, constant depth); smooth_features_xd needs 3 frames
FRAMES = []                                                      # what the fake imageio writer receives


def stub_modules():
    class Stub(types.ModuleType):
        def __getattr__(self, name):
            if name.startswith('__'):
                raise AttributeError(name)
            return type(name, (), {})

    for m in ('mediapipe', 'torchshow', 'librosa', 'utils', 'utils.commons', 'utils.commons.hparams', 'utils.commons.tensor_utils',
              'utils.commons.ckpt_utils', 'utils.commons.image_utils', 'utils.commons.meters', 'deep_3drecon',
              'deep_3drecon.deep_3drecon_models', 'deep_3drecon.deep_3drecon_models.bfm', 'deep_3drecon.secc_renderer',
              'data_util', 'data_util.face3d_helper', 'data_gen', 'data_gen.utils', 'data_gen.utils.process_image',
              'data_gen.utils.process_image.fit_3dmm_landmark', 'data_gen.utils.process_image.extract_lm2d',
              'data_gen.utils.process_video', 'data_gen.utils.process_video.fit_3dmm_landmark',
              'data_gen.utils.process_video.extract_segment_imgs', 'data_gen.eg3d', 'data_gen.eg3d.convert_to_eg3d_convention',
              'data_gen.utils.mp_feature_extractors', 'data_gen.utils.mp_feature_extractors.mp_segmenter'):
        sys.modules[m] = Stub(m)
    for k, v in (('VisibleDeprecationWarning', UserWarning), ('float', float), ('int', int), ('bool', bool)):
        if not hasattr(np, k):
            setattr(np, k, v)

    class Writer:
        def append_data(self, frame):
            FRAMES.append(np.array(frame, copy=True))

        def close(self):
            pass

    imageio = types.ModuleType('imageio')
    imageio.get_writer = lambda *a, **k: Writer()
    sys.modules['imageio'] = imageio
    os.system = lambda cmd: 0
    torch.Tensor.cuda = lambda self, *a, **k: self


class ReplayModel:
    """secc2video_model stand-in: forward() returns the next frame's given outputs."""

    def __init__(self, image, image_raw, image_depth):
        self.outs = [{'image': image[i:i + 1], 'image_raw': image_raw[i:i + 1], 'image_depth': image_depth[i:i + 1]}
                     for i in range(image.shape[0])]
        self.i = 0

    def forward(self, img=None, camera=None, cond=None, ret=None, **kw):
        out = self.outs[self.i]
        self.i += 1
        return out


def run_case(GeneFace2Infer, t):
    N = t['image'].shape[0]
    g = torch.Generator().manual_seed(0)
    batch = {'drv_secc': t['drv_secc'], 'camera': torch.zeros(N, 25), 'src_kp': torch.rand(N, 68, 2, generator=g),
             'drv_kp': torch.rand(N, 68, 2, generator=g), 'cano_secc': torch.zeros(1, 3, 512, 512), 'src_secc': torch.zeros(1, 3, 512, 512),
             'ref_gt_img': t['ref_gt_img'], 'ref_head_img': torch.zeros(1, 3, 512, 512), 'ref_torso_img': torch.zeros(1, 3, 512, 512),
             'bg_img': torch.zeros(1, 3, 512, 512), 'segmap': torch.zeros(1, 6, 512, 512)}
    inp = {'low_memory_usage': False, 'out_mode': 'concat_debug', 'out_name': 'debug.mp4', 'src_image_name': 'src.png',
           'drv_pose_name': 'drv.mp4', 'drv_audio_name': 'drv.mp4'}
    infer = GeneFace2Infer.__new__(GeneFace2Infer)
    infer.secc2video_model = ReplayModel(t['image'], t['image_raw'], t['image_depth'])
    FRAMES.clear()
    infer.forward_secc2video(batch, inp)
    assert len(FRAMES) == N and FRAMES[0].shape == (512, 2560, 3) and FRAMES[0].dtype == np.uint8, (len(FRAMES), FRAMES[0].shape)
    return np.stack(FRAMES)


def main():
    stub_modules()
    ref = os.environ['R3DP_REFERENCE']
    sys.path.insert(0, ref)
    cwd = os.getcwd()
    os.chdir(ref)                                                 # real3d_infer.py appends './' to sys.path
    try:
        from inference.real3d_infer import GeneFace2Infer
    finally:
        os.chdir(cwd)
    out = {}
    for name, N, seed, flat in CASES:
        fields = quirk_inputs(N, seed, constant_depth=flat)
        out.update({f'{name}.{k}': v for k, v in fields.items()})
        out[f'{name}.frames'] = run_case(GeneFace2Infer, full_inputs(fields))
    path = os.path.join(HERE, 'debug_frames.npz')
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
