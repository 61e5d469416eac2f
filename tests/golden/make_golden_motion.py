"""Generate tests/golden/motion_small.npz by running the REFERENCE's own clip-motion code on the synthetic head (synthetic.make_bfm with
make_keypoints): Face3DHelper.reconstruct_lm2d (data_util/face3d_helper.py), get_eg3d_convention_camera_pose_intrinsic
(data_gen/eg3d/convert_to_eg3d_convention.py), smooth_camera_sequence, smooth_features_xd and mirror_index (inference/infer_utils.py).

    R3DP_REFERENCE=<reference checkout> python tests/golden/make_golden_motion.py

real3d_infer.py itself needs mediapipe, so its pose steps (:282-309) and the key-point steps (:271-273, :428-431, :450-452, :463-464) are
restated below with line references.  Stand-ins go into sys.modules first: an empty librosa (infer_utils.py imports it, these functions do not
use it), and the deep_3drecon and deep_3drecon.deep_3drecon_models packages without their __init__ (which import kornia and the
reconstructor), so that bfm.py loads on its own.

Per case k: the inputs (`c<k>_id`, `_exp`, `_src_euler`, `_src_trans`, `_src_exp`, `_pose_euler` / `_pose_trans` unless static,
`_meta` = [T, P, map_to_init_pose]), the reference's outputs (`_cameras` [T,25], `_kp_s` [1,68,3], `_kp_d` [T,68,3]) and the reference's
own float32 deviation from the float64 restatement (tests/motion_reference.py), max |ref - f64| per output (`_dev` = [cameras, kp_s, kp_d])."""
import os
import sys
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

import motion_reference as mref  # noqa: E402
from real3dportrait_b200 import synthetic as syn  # noqa: E402

# (T, P (0 = static), map_to_init_pose, seed, straddle): P = 1, P < T (several mirror turns), P > T; T down to 3
CASES = [(3, 0, True, 1, False), (8, 1, True, 2, False), (8, 20, False, 3, False), (57, 20, True, 4, False), (57, 300, True, 5, False),
         (250, 20, False, 6, False), (250, 300, True, 7, False), (57, 0, False, 8, False), (57, 40, True, 9, True), (250, 40, False, 10, True)]


def reference():
    sys.modules.setdefault('librosa', types.ModuleType('librosa'))
    for name in ('deep_3drecon', 'deep_3drecon.deep_3drecon_models'):
        m = types.ModuleType(name)
        m.__path__ = [os.path.join(REF, *name.split('.'))]
        sys.modules[name] = m
    sys.path.insert(0, REF)
    from inference.infer_utils import mirror_index, smooth_camera_sequence, smooth_features_xd
    from data_util.face3d_helper import Face3DHelper
    from data_gen.eg3d.convert_to_eg3d_convention import get_eg3d_convention_camera_pose_intrinsic
    return mirror_index, smooth_camera_sequence, smooth_features_xd, Face3DHelper, get_eg3d_convention_camera_pose_intrinsic


def run_reference(fns, helper, c, T, map_to_init_pose):
    mirror_index, smooth_camera_sequence, smooth_features_xd, _, get_cam = fns
    src_id = torch.from_numpy(c['id'])
    src_exp, src_euler, src_trans = (torch.from_numpy(c[k]) for k in ('src_exp', 'src_euler', 'src_trans'))
    # real3d_infer.py:271-273
    src_kp = helper.reconstruct_lm2d(src_id, src_exp, src_euler, src_trans)
    src_kp = torch.clamp((src_kp - 0.5) / 0.5, -1, 1)
    # :282-296
    if c['pose'] is None:
        euler, trans = src_euler.repeat([T, 1]), src_trans.repeat([T, 1])
    else:
        eulers, trans_all = torch.from_numpy(c['pose'][0]), torch.from_numpy(c['pose'][1])
        index_lst = [mirror_index(i, len(eulers)) for i in range(T)]
        euler, trans = eulers[index_lst], trans_all[index_lst]
    # :299
    trans[:, -1] = trans[0:1, -1].repeat([trans.shape[0]])
    # :303-307
    if map_to_init_pose:
        euler = euler + (src_euler - euler[0:1])
        trans = trans + (src_trans - trans[0:1])
    # :310-316
    ret = get_cam({'euler': euler.cpu(), 'trans': trans.cpu()})
    camera = np.concatenate([ret['c2w'].reshape([-1, 16]), ret['intrinsics'].reshape([-1, 9])], axis=-1)
    camera = torch.tensor(smooth_camera_sequence(camera, kernel_size=7)).float()
    # :428-431 (id = src_id.repeat, real3d_infer.py:269), :450-452, :463-464
    drv_kp = helper.reconstruct_lm2d(src_id.repeat([T, 1]), torch.from_numpy(c['exp']), euler, trans)
    drv_kp = torch.clamp((drv_kp - 0.5) / 0.5, -1, 1)
    drv_kp = smooth_features_xd(drv_kp.reshape([-1, 68 * 2]), kernel_size=7).reshape([-1, 68, 2])
    z = lambda k: torch.cat([k, torch.zeros(k.shape[:-1] + (1,))], -1).numpy()    # noqa: E731
    return camera.numpy(), z(src_kp), z(drv_kp)


def main():
    import tempfile
    fns = reference()
    with tempfile.TemporaryDirectory() as d:
        kw = syn.write_bfm_folder(d, seed=0, keypoints=True)
        helper = fns[3](bfm_dir=kw['bfm_folder'], keypoint_mode='lm68', use_gpu=False)
        model = mref.load(kw['bfm_folder'])
    assert [fns[0](i, 3) for i in range(12)] == [mref.mirror_index(i, 3) for i in range(12)]
    out = {}
    for k, (T, P, mp, seed, straddle) in enumerate(CASES):
        c = mref.make_case(T, P, seed, straddle=straddle)
        got = run_reference(fns, helper, c, T, mp)
        want = mref.clip(model, c['id'], c['exp'], c['src_euler'], c['src_trans'], c['src_exp'], c['pose'], mp)
        dev = [float(np.abs(g.astype(np.float64) - w).max()) for g, w in zip(got, want)]
        pre = f'c{k}_'
        for name in ('id', 'exp', 'src_euler', 'src_trans', 'src_exp'):
            out[pre + name] = c[name]
        if c['pose'] is not None:
            out[pre + 'pose_euler'], out[pre + 'pose_trans'] = c['pose']
        out[pre + 'meta'] = np.array([T, P, int(mp)], np.int64)
        out[pre + 'cameras'], out[pre + 'kp_s'], out[pre + 'kp_d'] = got
        out[pre + 'dev'] = np.array(dev)
        clamped = float((np.abs(got[2][..., :2]) >= 1).mean())
        print(f'case {k}: T={T} P={P} map={mp} straddle={straddle}: reference float32 deviation cameras {dev[0]:.2e} kp_s {dev[1]:.2e} '
              f'kp_d {dev[2]:.2e}; {clamped:.1%} of kp_d at the clamp')
    path = os.path.join(HERE, 'motion_small.npz')
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
