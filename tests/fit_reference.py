"""Float64 restatement of the 3DMM landmark fit (data_gen/utils/process_image/fit_3dmm_landmark.py:85-236, fit_3dmm_for_a_image, and
data_gen/utils/process_video/fit_3dmm_landmark.py:131-360, fit_3dmm_for_a_video with id_mode='global'), written from their semantics; the
checker of Fit3DMM.  torch, any device and dtype; the gradients come from torch autograd, independently of the kernels' hand-derived ones.

  model     468 key points: the BFM rows at index_mp468_from_mesh35709.npy (negative entries -> vertex 0), mean recentred (float32, as
            the reference's data), basis [468,3,80+64]
  geometry  p = (Rz Ry Rx) shape + trans, z = 10 - p_z, proj = 1015 (x, y) / z + 112
  lms       [:468], y = H - y, / (H / 224)
  loss      mean over T 468 2 of w (proj - lms)^2; image: eye 5, lips 2; video: eye 3, upper eye 20, lips 5; unmatched 0
  stage 1   200 Adam steps (lr 0.1) on euler, trans with id = exp = 0
  stage 2   200 steps: + lambda_id mean(id^2) + lambda_exp mean(exp^2) (image 0.3 / 0.05, video 0.2 / 0.6), video also the Laplacian
            loss on exp, 0.3 x on euler and trans; id / exp with a fresh Adam, euler / trans continue theirs (steps 201-400)

The reference's fine stage (50-iteration batches at lr 0.005) writes its results into temporary copies (`exp_para[sel_ids].data = ...`
with a numpy index), so its outputs are the stage-2 state; fit(..., fine=True) runs that dead stage anyway, for timing the reference's
loop (tools/bench_fit.py)."""
from __future__ import annotations

import os

import numpy as np
import torch

N_KP, N_ID, N_EXP = 468, 80, 64
FOCAL, CENTER, CAMERA_DISTANCE = 1015.0, 112.0, 10.0
UNMATCHED = [93, 127, 132, 234, 323, 356, 361, 454]
UPPER_EYE = [161, 160, 159, 158, 157] + [388, 387, 386, 385, 384]
EYE = [33, 246, 161, 160, 159, 158, 157, 173, 133, 155, 154, 153, 145, 144, 163, 7] + \
      [263, 466, 388, 387, 386, 385, 384, 398, 362, 382, 381, 380, 374, 373, 390, 249]
INNER_LIP = [78, 191, 80, 81, 82, 13, 312, 311, 310, 415, 308, 324, 318, 402, 317, 14, 87, 178, 88, 95]
OUTER_LIP = [61, 185, 40, 39, 37, 0, 267, 269, 270, 409, 291, 375, 321, 405, 314, 17, 84, 181, 91, 146]
#: (lambda_id, lambda_exp, lambda_lap) of the image and the video fit
LAMBDAS = {False: (0.3, 0.05, 0.0), True: (0.2, 0.6, 1.0)}


def weights(video: bool) -> np.ndarray:
    """cal_lan_loss_mp's per-point weights [468] (the image and the video file differ)."""
    w = np.ones(N_KP)
    w[EYE] = 3 if video else 5
    if video:
        w[UPPER_EYE] = 20
    w[INNER_LIP] = 5 if video else 2
    w[OUTER_LIP] = 5 if video else 2
    w[UNMATCHED] = 0
    return w


def load(bfm_folder: str) -> dict:
    """-> mean [468,3], basis [468,3,144] (float32 values in float64), index [468] as used (negative -> 0)."""
    from scipy.io import loadmat
    m = loadmat(os.path.join(bfm_folder, 'BFM_model_front.mat'))
    mean = m['meanshape'].astype(np.float32).reshape(-1, 3)
    mean = mean - np.mean(mean, axis=0, keepdims=True)
    idx = np.load(os.path.join(bfm_folder, 'index_mp468_from_mesh35709.npy')).astype(np.int64)
    idx[idx < 0] = 0
    basis = np.concatenate([m['idBase'].astype(np.float32).reshape(-1, 3, N_ID), m['exBase'].astype(np.float32).reshape(-1, 3, N_EXP)], -1)
    return {'mean': mean[idx].astype(np.float64), 'basis': basis[idx].astype(np.float64), 'index': idx}


def rotation(euler: torch.Tensor) -> torch.Tensor:
    """[T,3] -> Rz Ry Rx [T,3,3] (compute_rotation returns its transpose and multiplies row vectors)."""
    x, y, z = euler[:, 0], euler[:, 1], euler[:, 2]
    o, n = torch.ones_like(x), torch.zeros_like(x)
    rx = torch.stack([o, n, n, n, x.cos(), -x.sin(), n, x.sin(), x.cos()], -1).reshape(-1, 3, 3)
    ry = torch.stack([y.cos(), n, y.sin(), n, o, n, -y.sin(), n, y.cos()], -1).reshape(-1, 3, 3)
    rz = torch.stack([z.cos(), -z.sin(), n, z.sin(), z.cos(), n, n, n, o], -1).reshape(-1, 3, 3)
    return rz @ ry @ rx


def project(mean: torch.Tensor, basis: torch.Tensor, id_: torch.Tensor, exp: torch.Tensor, euler: torch.Tensor, trans: torch.Tensor):
    """compute_for_landmark_fit: id [1|T,80], exp [T,64], euler, trans [T,3] -> [T,468,2] in the 224 image, y up."""
    T = exp.shape[0]
    q = torch.cat([id_.expand(T, -1), exp], 1)
    shape = mean[None] + torch.einsum('vak,tk->tva', basis, q)
    p = torch.einsum('tab,tvb->tva', rotation(euler), shape) + trans[:, None]
    z = CAMERA_DISTANCE - p[..., 2:]
    return FOCAL * p[..., :2] / z + CENTER


def prepare_lms(lms, img_size: int, dtype, device) -> torch.Tensor:
    """mediapipe pixels [T,468|478,2] (y down) -> the fit's targets [T,468,2]."""
    lms = torch.as_tensor(np.asarray(lms, np.float32)).to(device=device, dtype=dtype)
    lms = lms.reshape(-1, lms.shape[-2], 2)[:, :N_KP].clone()
    lms[..., 1] = img_size - lms[..., 1]
    return lms / (img_size / (2 * CENTER))


def lap_loss(x: torch.Tensor) -> torch.Tensor:
    """cal_lap_loss: (-1/2, 1, -1/2) over frames with replicated ends, squared, mean."""
    xp = torch.cat([x[:1], x, x[-1:]], 0)
    return ((xp[1:-1] - 0.5 * (xp[:-2] + xp[2:])) ** 2).mean()


def fit(model: dict, lms, img_size: int = 512, video: bool = False, dtype=torch.float64, device='cpu', fine: bool = False) -> dict:
    """The reference's fit -> {'id' [1,80], 'exp' [T,64], 'euler' [T,3], 'trans' [T,3]} as numpy arrays of dtype."""
    tgt = prepare_lms(lms, img_size, dtype, device)
    T = tgt.shape[0]
    mean = torch.as_tensor(model['mean']).to(device, dtype)
    basis = torch.as_tensor(model['basis']).to(device, dtype)
    w = torch.as_tensor(weights(video)).to(device, dtype)[None, :, None]
    lam_id, lam_exp, lam_lap = LAMBDAS[video]
    z = lambda *s: torch.zeros(*s, device=device, dtype=dtype, requires_grad=True)  # noqa: E731
    id_, exp, euler, trans = z(1, N_ID), z(T, N_EXP), z(T, 3), z(T, 3)

    def lan():
        return (w * (project(mean, basis, id_, exp, euler, trans) - tgt) ** 2).mean()

    opt_frame = torch.optim.Adam([euler, trans], lr=0.1)
    for _ in range(200):
        loss = lan()
        opt_frame.zero_grad()
        loss.backward()
        opt_frame.step()
    opt_idexp = torch.optim.Adam([id_, exp], lr=0.1)
    for _ in range(200):
        loss = lan() + lam_id * (id_ * id_).mean() + lam_exp * (exp * exp).mean()
        if video:
            loss = loss + lam_lap * (lap_loss(exp) + 0.3 * lap_loss(euler) + 0.3 * lap_loss(trans))
        opt_idexp.zero_grad()
        opt_frame.zero_grad()
        loss.backward()
        opt_idexp.step()
        opt_frame.step()
    if fine:
        _dead_fine_stage(mean, basis, w, tgt, id_, exp, euler, trans, video)
    return {k: v.detach().cpu().numpy() for k, v in (('id', id_), ('exp', exp), ('euler', euler), ('trans', trans))}


def _dead_fine_stage(mean, basis, w, tgt, id_, exp, euler, trans, video):
    """The reference's fine stage as it runs (batches of 50 frames, 1 for the image; 50 steps at lr 0.005), its results discarded as the
    reference's are."""
    T = exp.shape[0]
    lam_id, lam_exp, lam_lap = LAMBDAS[video]
    bs = 50 if video else 1
    for i in range((T - 1) // bs + 1):
        sel = np.arange(max(T - bs, 0), T) if (i + 1) * bs > T else np.arange(i * bs, i * bs + bs)
        s_exp, s_e, s_t = (x.detach()[sel].clone().requires_grad_(True) for x in (exp, euler, trans))
        s_id = id_.detach().clone().requires_grad_(not video)
        opt = torch.optim.Adam([s_exp, s_e, s_t] + ([] if video else [s_id]), lr=0.005)
        for _ in range(50):
            loss = (w * (project(mean, basis, s_id, s_exp, s_e, s_t) - tgt[sel]) ** 2).mean()
            loss = loss + lam_id * (s_id * s_id).mean() + lam_exp * (s_exp * s_exp).mean()
            if video:
                loss = loss + lam_lap * (lap_loss(s_exp) + 0.3 * lap_loss(s_e) + 0.3 * lap_loss(s_t))
            opt.zero_grad()
            loss.backward()
            opt.step()


def gradient(model: dict, lms, id_, exp, euler, trans, img_size: int = 512, video: bool = True, stage: int = 2):
    """Float64 autograd gradient of one iteration's loss at the given parameters -> (d id [1,80], d exp [T,64], d euler, d trans [T,3]);
    stage 1: the landmark loss only (id and exp held at their values)."""
    tgt = prepare_lms(lms, img_size, torch.float64, 'cpu')
    mean, basis = torch.as_tensor(model['mean']), torch.as_tensor(model['basis'])
    w = torch.as_tensor(weights(video))[None, :, None]
    lam_id, lam_exp, lam_lap = LAMBDAS[video]
    p = [torch.tensor(np.asarray(x, np.float64), requires_grad=True) for x in (id_, exp, euler, trans)]
    loss = (w * (project(mean, basis, *p) - tgt) ** 2).mean()
    if stage == 2:
        loss = loss + lam_id * (p[0] * p[0]).mean() + lam_exp * (p[1] * p[1]).mean()
        if video:
            loss = loss + lam_lap * (lap_loss(p[1]) + 0.3 * lap_loss(p[2]) + 0.3 * lap_loss(p[3]))
    loss.backward()
    return tuple(x.grad.numpy() for x in p)


def make_landmarks(model: dict, T: int, seed: int, img_size: int = 512, noise: float = 0.3) -> tuple:
    """Landmarks of known smooth trajectories projected through the model: mediapipe pixels [T,478,2] (y down, sub-pixel noise, 10 junk
    iris points) and the truth {'id', 'exp', 'euler', 'trans'}."""
    rng = np.random.default_rng(seed)
    t = np.arange(T)[:, None] / 25.0
    ph = rng.uniform(0, 2 * np.pi, size=(1, 3 + 3 + N_EXP))
    fr = rng.uniform(0.2, 1.0, size=(1, 3 + 3 + N_EXP))
    wave = np.sin(2 * np.pi * fr * t + ph)
    # Head poses within +-0.1 rad and the head 11 units from the camera (trans z = -1): with larger poses nearer the camera, the reference's
    # Adam (lr 0.1) starts to oscillate in the yaw / x-translation valley of some frames once they converge, and the oscillation amplifies
    # rounding by orders of magnitude, so float32 runs of the same fit disagree in their leading digits (DESIGN.md, "3DMM fit").
    truth = {'id': rng.normal(size=(1, N_ID)) * 0.6,
             'euler': wave[:, :3] * np.array([0.04, 0.1, 0.024]) + rng.normal(size=(1, 3)) * 0.02,
             'trans': wave[:, 3:6] * np.array([0.02, 0.016, 0.04]) + np.array([0.0, 0.02, 0.08]) * rng.uniform(-1, 1, size=(1, 3))
             + np.array([0.0, 0.0, -1.0]),
             'exp': wave[:, 6:] * 0.8 + rng.normal(size=(1, N_EXP)) * 0.3}
    with torch.no_grad():
        proj = project(*(torch.as_tensor(x, dtype=torch.float64) for x in (model['mean'], model['basis'], truth['id'], truth['exp'],
                                                                                 truth['euler'], truth['trans']))).numpy()
    px = proj * (img_size / (2 * CENTER))
    px[..., 1] = img_size - px[..., 1]
    px = px + rng.uniform(-noise, noise, size=px.shape)
    iris = rng.uniform(0, img_size, size=(T, 10, 2))
    return np.concatenate([px, iris], 1).astype(np.float32), truth
