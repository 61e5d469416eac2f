"""Float64 restatement of a clip's motion (real3d_infer.py:271-321, 428-452 with Face3DHelper.reconstruct_lm2d,
get_eg3d_convention_camera_pose_intrinsic, smooth_camera_sequence and smooth_features_xd), written from their sources; the checker of
ClipMotion.  numpy and scipy.

  pose      frame i: driving row mirror_index(i, P) (static: the source pose), trans z of frame 0, + (src - pose[0]) with map_to_init_pose
  camera    R = (Rz Ry Rx)^T, c = 0.27 (-R (t - [0,0,10])) + [0, 0.006, 0.161], c2w = [[R diag(1,-1,-1), c], [0,0,0,1]], K = _fix_intrinsics
  smoothing window [max(0, i-3), min(T, i+4)): translation mean, scipy Rotation.mean; intrinsics unchanged
  key pts   the BFM rows at keypoints as stored (no - 1); kp = clamp((-x_ndc, -y_ndc), -1, 1) of the SECC vertex pass, z = 0
  kp_d      7-tap box filter over frames padded with the flipped first and last three frames

The reference computes these in float32 (the key points, and the camera before its float64 smoothing); tests/golden/motion_small.npz
stores its deviation from this restatement per case, and REF_DEV bounds it over every case of the fixture (tests/test_cpu_motion.py)."""
from __future__ import annotations

import os

import numpy as np

from secc_render_reference import rotation, shape

HALF = 3
FOCAL, CENTER = 1015.0, 112.0
#: the reference's float32 deviation from this restatement, max over the fixture's cases (cameras, kp_s, kp_d): 4.4e-7, 1.01e-6, 9.7e-7
REF_DEV = (4.5e-7, 1.05e-6, 1.0e-6)
INTRINSICS = np.array([[2985.29 / 700, 0, 0.5], [0, 2985.29 / 700, 0.5], [0, 0, 1]])


def load(bfm_folder, minus_one=False):
    """BFM_model_front.mat -> the gathered key-point model: mean [68,3], id_base [204,80], exp_base [204,64] (float32 values in float64),
    keypoints [68] as stored (minus_one=True: ParametricFaceModel's 0-based landmarks, for the off-by-one test)."""
    from scipy.io import loadmat
    m = loadmat(os.path.join(bfm_folder, 'BFM_model_front.mat'))
    mean = m['meanshape'].astype(np.float32).reshape(-1, 3)
    mean = mean - np.mean(mean, axis=0, keepdims=True)
    kp = np.squeeze(m['keypoints']).astype(np.int64) - (1 if minus_one else 0)
    rows = (3 * kp[:, None] + np.arange(3)[None]).reshape(-1)
    return {'mean': mean[kp].astype(np.float64), 'id_base': m['idBase'].astype(np.float32)[rows].astype(np.float64),
            'exp_base': m['exBase'].astype(np.float32)[rows].astype(np.float64), 'keypoints': kp}


def mirror_index(index, len_seq):
    turn, res = index // len_seq, index % len_seq
    return res if turn % 2 == 0 else len_seq - res - 1


def poses(src_euler, src_trans, pose, T, map_to_init_pose=True, dtype=np.float64):
    """-> euler, trans [T,3] in dtype (real3d_infer.py:282-309; float32 reproduces the reference's pose bit for bit)."""
    se, st = np.asarray(src_euler, dtype).reshape(1, 3), np.asarray(src_trans, dtype).reshape(1, 3)
    if pose is None:
        e, t = np.repeat(se, T, 0), np.repeat(st, T, 0)
    else:
        de, dt = np.asarray(pose[0], dtype).reshape(-1, 3), np.asarray(pose[1], dtype).reshape(-1, 3)
        idx = [mirror_index(i, len(de)) for i in range(T)]
        e, t = de[idx].copy(), dt[idx].copy()
    t[:, 2] = t[0, 2]
    if map_to_init_pose:
        e = e + (se - e[0:1])
        t = t + (st - t[0:1])
    return e, t


def raw_cameras(euler, trans):
    """-> c2w [T,4,4] of get_eg3d_convention_camera_pose_intrinsic."""
    e = np.asarray(euler, np.float64)
    R = np.transpose(rotation(e), (0, 2, 1))
    t = np.asarray(trans, np.float64).copy()
    t[:, 2] -= 10.0
    c = -np.einsum('bij,bj->bi', R, t) * 0.27
    c[:, 1] += 0.006
    c[:, 2] += 0.161
    pose = np.tile(np.eye(4), (len(e), 1, 1))
    pose[:, :3, :3] = R @ np.diag([1.0, -1.0, -1.0])
    pose[:, :3, 3] = c
    return pose


def smooth_cameras(c2w):
    """smooth_camera_sequence(kernel_size=7) on [T,4,4] -> cameras [T,25] float64."""
    from scipy.spatial.transform import Rotation
    T = len(c2w)
    out = c2w.copy()
    for i in range(T):
        s, e = max(0, i - HALF), min(T, i + HALF + 1)
        out[i, :3, 3] = c2w[s:e, :3, 3].mean(0)
        out[i, :3, :3] = Rotation.from_matrix(c2w[s:e, :3, :3]).mean().as_matrix()
    return np.concatenate([out.reshape(T, 16), np.tile(INTRINSICS.reshape(1, 9), (T, 1))], 1)


def keypoints(model, id, exp, euler, trans):
    """-> kp [T,68,2] = clamp((lm2d - 0.5) / 0.5, -1, 1) = clamp((-x_ndc, -y_ndc)) of the vertex pass (lm2d: lm2d below)."""
    return np.clip(2 * lm2d(model, id, exp, euler, trans) - 1, -1, 1)


def lm2d(model, id, exp, euler, trans):
    """Face3DHelper.reconstruct_lm2d -> [T,68,2]: (f x / z + c, 224 - (f y / z + c)) / 224 with z = 10 - z, i.e. ((1 - x_ndc) / 2,
    (1 - y_ndc) / 2)."""
    s, _ = shape(model, id, exp)
    v = np.einsum('bij,bnj->bni', rotation(euler), s) + np.asarray(trans, np.float64)[:, None]
    z = 10.0 - v[..., 2]
    return np.stack([(FOCAL * v[..., 0] / z + CENTER) / 224, (224 - (FOCAL * v[..., 1] / z + CENTER)) / 224], -1)


def smooth_kp(kp):
    """smooth_features_xd(kp [T,...], 7): reflect-pad 3 frames each side (edge repeated), box filter.  T >= 3."""
    T = kp.shape[0]
    if T < HALF:
        raise ValueError('smooth_features_xd needs at least 3 frames')
    k = np.asarray(kp, np.float64)
    pad = np.concatenate([k[:HALF][::-1], k, k[T - HALF:][::-1]], 0)
    return sum(pad[d:d + T] for d in range(2 * HALF + 1)) / (2 * HALF + 1)


def clip(model, id, exp, src_euler, src_trans, src_exp, pose=None, map_to_init_pose=True):
    """-> cameras [T,25], kp_s [1,68,3], kp_d [T,68,3] float64.  The pose steps run in float64 on the float32 inputs."""
    dt = np.float64
    exp = np.asarray(exp, np.float64)
    T = exp.shape[0]
    id = np.broadcast_to(np.asarray(id, np.float64), (T, id.shape[1])) if np.asarray(id).shape[0] == 1 else np.asarray(id, np.float64)
    e, t = poses(src_euler, src_trans, pose, T, map_to_init_pose, dt)
    cams = smooth_cameras(raw_cameras(e, t))
    kp_s = keypoints(model, id[:1], src_exp, np.asarray(src_euler, dt).reshape(1, 3), np.asarray(src_trans, dt).reshape(1, 3))
    kp_d = smooth_kp(keypoints(model, id, exp, e, t))
    z = lambda k: np.concatenate([k, np.zeros(k.shape[:-1] + (1,))], -1)    # noqa: E731
    return cams, z(kp_s), z(kp_d)


def make_case(T, P, seed, yaw=0.6, trans=0.15, straddle=False):
    """Inputs of one clip on the synthetic head: id [1,80], exp [T,64], the source fit and a driving pose (None if P == 0), float32 numpy.
    straddle=True: a pose sequence whose camera quaternions flip sign between neighbouring frames (see below).  Every pose with pitch
    crossing 0 already takes the quaternion's w through 0 (the camera rotation is then close to pi about x)."""
    rng = np.random.default_rng(seed)
    f = np.float32
    c = {'id': rng.normal(size=(1, 80)).astype(f), 'exp': rng.normal(size=(T, 64)).astype(f),
         'src_exp': rng.normal(size=(1, 64)).astype(f),
         'src_euler': (rng.uniform(-1, 1, (1, 3)) * yaw * np.array([0.2, 1.0, 0.2])).astype(f),
         'src_trans': (rng.normal(size=(1, 3)) * trans * np.array([1.0, 1.0, 0.3])).astype(f)}
    if P == 0:
        c['pose'] = None
    else:
        s = np.linspace(0, 1, P)[:, None]
        e = np.sin(2 * np.pi * (s * rng.uniform(0.5, 2, (1, 3)) + rng.uniform(0, 1, (1, 3)))) * yaw * np.array([0.3, 1.0, 0.3])
        e = e + 0.02 * rng.normal(size=(P, 3))
        t = np.sin(2 * np.pi * (s * rng.uniform(0.5, 2, (1, 3)) + rng.uniform(0, 1, (1, 3)))) * trans * 2 + 0.01 * rng.normal(size=(P, 3))
        if straddle:
            # pitch around -pi/2: the camera rotation is 3 pi / 2 - pitch about x, where from_matrix switches from its x branch to its
            # trace branch and the quaternion of one frame is close to minus that of its neighbour
            e[:, 0] = -np.pi / 2 + np.linspace(-0.08, 0.08, P) + 0.01 * rng.normal(size=P)
        c['pose'] = (e.astype(f), t.astype(f))
    return c
