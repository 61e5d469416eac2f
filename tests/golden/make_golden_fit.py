"""Generate tests/golden/fit_small.npz by running the REFERENCE's own fit_3dmm_for_a_image (data_gen/utils/process_image/fit_3dmm_landmark.py)
and fit_3dmm_for_a_video (data_gen/utils/process_video/fit_3dmm_landmark.py, id_mode='global') verbatim, on the CPU, on the synthetic BFM
(synthetic.write_bfm_folder(..., mp468=True)).

    R3DP_REFERENCE=<reference checkout> python tests/golden/make_golden_fit.py

Stand-ins go into sys.modules first: numpy 1's numpy.lib.function_base and numpy.core.numeric (imported, not used), cv2 (imread / VideoCapture return black 512^2 frames; the fit reads only their size and count), the
mediapipe landmarker module, utils.commons' multiprocess helpers, deep_3drecon.secc_renderer and deep_3drecon.util.load_mats, and the
deep_3drecon packages without their __init__.  ParametricFaceModel.to and Tensor.cuda are patched to stay on the CPU.  Both modules build
their model at import from the relative path deep_3drecon/BFM, so they are imported (and run) with a temporary cwd holding that folder;
the landmarks go in the *_lms.npy file each function looks for.

Landmarks: smooth trajectories projected through the synthetic model in float64 (fit_reference.make_landmarks), 512^2 pixels with y
down, +-0.3 px noise, 10 junk iris points.  A case must be well conditioned: the reference's own float32 deviation from float64 at most
MAX_REL_DEV of its outputs' magnitude, else the next seed is tried.  Per case k: `c<k>_lms` [T,478,2], `c<k>_meta` = [T, video, seed], the
reference's outputs
(`c<k>_id` [1,80], `_exp` [T,64], `_euler`, `_trans` [T,3]) and the reference's own float32 deviation from the float64 restatement
(tests/fit_reference.py), max |ref - f64| per output (`c<k>_dev` = [id, exp, euler, trans]).

Every case runs a second time with the lr-0.005 optimizer's step() a no-op; the outputs must be bit-identical, which proves that the
reference's fine stage (the 50-iteration batches) does not reach its returned coefficients."""
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get('R3DP_REFERENCE')
if not REF:
    sys.exit('set R3DP_REFERENCE to a checkout of the reference project')
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, ROOT)

import fit_reference as fref  # noqa: E402
from real3dportrait_b200 import synthetic as syn  # noqa: E402

IMG = 512
#: (T, video): the image, and videos below, at and around one fine-stage batch of 50 frames
CASES = [(1, False), (1, True), (2, True), (37, True), (50, True), (51, True), (120, True)]
#: a case enters the fixture only if the reference's own float32 deviation from float64 is at most this fraction of its outputs' magnitude
#: (at least 1): a larger one marks a fit whose rounding the Adam loop amplifies, where the bar built from it would say little
MAX_REL_DEV = 1e-4
SEED_TRIES = 4
N_FRAMES = {'n': 1}


def stand_ins():
    class Capture:
        def __init__(self, name):
            self.left = N_FRAMES['n']

        def isOpened(self):
            return True

        def read(self):
            self.left -= 1
            return (True, np.zeros((IMG, IMG, 3), np.uint8)) if self.left >= 0 else (False, None)

    cv2 = types.ModuleType('cv2')
    cv2.imread = lambda name: np.zeros((IMG, IMG, 3), np.uint8)
    cv2.cvtColor = lambda img, code: img
    cv2.COLOR_BGR2RGB = 4
    cv2.VideoCapture = Capture
    sys.modules['cv2'] = cv2
    lmk = types.ModuleType('data_gen.utils.mp_feature_extractors.face_landmarker')
    lmk.MediapipeLandmarker = None
    lmk.read_video_to_frames = lambda name: np.zeros((N_FRAMES['n'], IMG, IMG, 3), np.uint8)
    sys.modules[lmk.__name__] = lmk
    mp = types.ModuleType('utils.commons.multiprocess_utils')
    mp.multiprocess_run_tqdm = None
    sys.modules[mp.__name__] = mp
    osu = types.ModuleType('utils.commons.os_utils')
    osu.multiprocess_glob = None
    sys.modules[osu.__name__] = osu
    secc = types.ModuleType('deep_3drecon.secc_renderer')
    secc.SECC_Renderer = None
    sys.modules[secc.__name__] = secc
    mats = types.ModuleType('deep_3drecon.util.load_mats')
    mats.transferBFM09 = None
    sys.modules[mats.__name__] = mats
    fb = types.ModuleType('numpy.lib.function_base')                       # both files import these two names and use neither
    fb.quantile = np.quantile
    sys.modules.setdefault(fb.__name__, fb)
    nn_ = types.ModuleType('numpy.core.numeric')
    nn_.require = np.require
    sys.modules.setdefault(nn_.__name__, nn_)
    for name in ('deep_3drecon', 'deep_3drecon.deep_3drecon_models', 'deep_3drecon.util'):
        m = types.ModuleType(name)
        m.__path__ = [os.path.join(REF, *name.split('.'))]
        sys.modules[name] = m
    sys.path.insert(0, REF)
    from deep_3drecon.deep_3drecon_models import bfm
    to = bfm.ParametricFaceModel.to
    bfm.ParametricFaceModel.to = lambda self, device: to(self, 'cpu')
    torch.Tensor.cuda = lambda self, *a, **k: self


def import_reference():
    import importlib.util
    mods = []
    for name, rel in (('fit_image', 'data_gen/utils/process_image/fit_3dmm_landmark.py'), ('fit_video', 'data_gen/utils/process_video/fit_3dmm_landmark.py')):
        spec = importlib.util.spec_from_file_location(name, os.path.join(REF, rel))
        m = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(m)
        mods.append(m)
    return mods[0].fit_3dmm_for_a_image, mods[1].fit_3dmm_for_a_video


def run(fns, work, k, lms, video, dead_fine):
    fit_image, fit_video = fns
    np.save(os.path.join(work, 'lms_2d', f'c{k}_lms.npy'), lms if video else lms[0])
    N_FRAMES['n'] = lms.shape[0]
    step = torch.optim.Adam.step
    if dead_fine:
        def step_unless_fine(self, *a, **kw):
            if self.param_groups[0]['lr'] == 0.005:
                return None
            return step(self, *a, **kw)
        torch.optim.Adam.step = step_unless_fine
    try:
        if video:
            out = fit_video(os.path.join(work, 'video', f'c{k}.mp4'), save=False)
        else:
            out = fit_image(os.path.join(work, 'images_512', f'c{k}.png'), device='cpu', save=False)
    finally:
        torch.optim.Adam.step = step
    return {n: np.asarray(out[n]) for n in ('id', 'exp', 'euler', 'trans')}


def main():
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    cwd = os.getcwd()
    out = {}
    with tempfile.TemporaryDirectory() as work:
        syn.write_bfm_folder(os.path.join(work, 'deep_3drecon'), seed=0, mp468=True)
        model = fref.load(os.path.join(work, 'deep_3drecon', 'BFM'))
        for d in ('lms_2d', 'video', 'images_512'):
            os.makedirs(os.path.join(work, d))
        stand_ins()
        os.chdir(work)
        try:
            fns = import_reference()
            for k, (T, video) in enumerate(CASES):
                for attempt in range(SEED_TRIES):                 # the first seed whose fit is well conditioned
                    seed = 10 + k + 100 * attempt
                    lms, _ = fref.make_landmarks(model, T, seed=seed, img_size=IMG)
                    got = run(fns, work, k, lms, video, dead_fine=False)
                    want = fref.fit(model, lms, IMG, video=video)
                    dev = [float(np.abs(got[n].astype(np.float64) - want[n]).max()) for n in ('id', 'exp', 'euler', 'trans')]
                    if all(d <= MAX_REL_DEV * max(1.0, float(np.abs(want[n]).max())) for d, n in zip(dev, ('id', 'exp', 'euler', 'trans'))):
                        break
                    print(f'case {k}: seed {seed} ill-conditioned (deviation {max(dev):.1e}), next seed', flush=True)
                else:
                    raise AssertionError(f'case {k}: no well-conditioned seed in {SEED_TRIES} tries')
                again = run(fns, work, k, lms, video, dead_fine=True)
                for n in got:
                    assert got[n].dtype == np.float32 and np.array_equal(got[n], again[n]), (k, n, 'the fine stage reached the output')
                pre = f'c{k}_'
                out[pre + 'lms'] = lms
                out[pre + 'meta'] = np.array([T, int(video), seed], np.int64)
                for n in got:
                    out[pre + n] = got[n]
                out[pre + 'dev'] = np.array(dev)
                print(f'case {k}: T={T} video={video}: fine stage dead (bit-identical without it); reference float32 deviation '
                      f'id {dev[0]:.2e} exp {dev[1]:.2e} euler {dev[2]:.2e} trans {dev[3]:.2e}; |id| {np.abs(got["id"]).max():.2f} '
                      f'|exp| {np.abs(got["exp"]).max():.2f}', flush=True)
        finally:
            os.chdir(cwd)
    path = os.path.join(HERE, 'fit_small.npz')
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
