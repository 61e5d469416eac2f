"""Generate tests/golden/source_small.npz by running the REFERENCE's own source-image functions on synthetic inputs:
inpaint_torso_job and extract_background (data_gen/utils/process_video/extract_segment_imgs.py) and
MediapipeSegmenter._seg_out_img_with_segmap (data_gen/utils/mp_feature_extractors/mp_segmenter.py), with cv2, scipy and sklearn.

    R3DP_REFERENCE=<reference checkout> python tests/golden/make_golden_source.py

mediapipe and the reference's utils.commons / split_video_to_imgs modules are replaced by stubs in sys.modules (none of them is used by
these functions).  Inputs are regenerated from the stored parameters with synthetic.make_source_image / make_segmap; stored are the uint8
outputs, the case parameters (JSON) and numpy's 0.98 ** np.arange(53) of the generating machine."""
import json
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

from real3dportrait_b200 import synthetic as syn  # noqa: E402
from source_reference import BG_FRAMES, BG_H, BG_W, bg_inputs, case_inputs  # noqa: E402

# (name, H, W, seed, make_segmap keywords, roll the head's lowest row onto the last row)
TORSO_CASES = [
    ('portrait', 512, 512, 0, {}, False),
    ('wrap_neck', 96, 128, 1, {}, True),                               # neck on row 0 under head on row H-1
    ('wrap_torso', 96, 128, 2, {'torso_top': 0.45, 'neck_width': 0.0}, True),   # torso on row 0 under head on row H-1
    ('neck_gaps', 128, 96, 3, {'neck_gaps': 12}, False),
    ('wide_neck', 96, 128, 4, {'neck_width': 0.25}, False),            # neck columns with no head above them
    ('no_torso', 96, 128, 5, {'torso': False}, False),
    ('fractional', 128, 128, 6, {'fractional': True}, False),
]


def stub_modules():
    class Stub(types.ModuleType):
        def __getattr__(self, name):
            if name.startswith('__'):
                raise AttributeError(name)
            return type(name, (), {})

    for m in ('mediapipe', 'mediapipe.tasks', 'mediapipe.tasks.python', 'mediapipe.tasks.python.vision', 'utils', 'utils.commons',
              'utils.commons.tensor_utils', 'utils.commons.os_utils', 'utils.commons.multiprocess_utils',
              'data_gen.utils.process_video.split_video_to_imgs'):
        sys.modules[m] = Stub(m)


def roll_rows(H, W, seed, kw):
    seg = syn.make_segmap(H, W, seed, **kw)
    head_rows = np.nonzero((seg[1] + seg[3] + seg[5]).any(1))[0]
    return int(H - 1 - head_rows.max())


def main():
    stub_modules()
    sys.path.insert(0, os.environ['R3DP_REFERENCE'])
    from data_gen.utils.mp_feature_extractors.mp_segmenter import MediapipeSegmenter
    from data_gen.utils.process_video.extract_segment_imgs import extract_background, inpaint_torso_job

    out, cases = {}, []
    for name, H, W, seed, kw, roll in TORSO_CASES:
        kw = dict(kw)
        if roll:
            kw['roll'] = roll_rows(H, W, seed, kw)
        img, seg = case_inputs(H, W, seed, kw)
        out[f'{name}.torso'] = inpaint_torso_job(img, seg)[0]
        out[f'{name}.head'] = MediapipeSegmenter._seg_out_img_with_segmap(None, img, seg, 'head')[0]
        out[f'{name}.bg'] = extract_background([img], [seg], 'knn')
        cases.append({'name': name, 'H': H, 'W': W, 'seed': seed, 'kw': kw})
    for n in BG_FRAMES:
        frames, segs = bg_inputs(n)
        out[f'bg{n}'] = extract_background(list(frames), list(segs), 'knn')
    out['cases'] = np.array(json.dumps(cases))
    out['bg_frames'] = np.array(BG_FRAMES, np.int64)
    out['bg_size'] = np.array([BG_H, BG_W], np.int64)
    out['tab_neck'] = 0.98 ** np.arange(53)
    path = os.path.join(HERE, 'source_small.npz')
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
