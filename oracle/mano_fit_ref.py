"""numpy / torch statement of utils/mano_from_3djoint (convert2mano.py, AIK.py, utils.py) for the host tests and the eager GPU comparison
of renderih_b200.mano_from_3djoint.  Nothing here calls the reference."""
import math

import numpy as np
import torch

LEFT = ['Wrist_L'] + ['%sFinger%d_L' % (f, i) for f in ('Thumb', 'Index', 'Middle', 'Ring', 'Pinky') for i in range(1, 5)]
RIGHT = [n[:-1] + 'R' for n in LEFT]
SNAP_PARENT = [0, 0, 1, 2, 3, 0, 5, 6, 7, 0, 9, 10, 11, 0, 13, 14, 15, 0, 17, 18, 19]
KINEMATIC_TREE = [2, 3, 4, 6, 7, 8, 10, 11, 12, 14, 15, 16, 18, 19, 20]
ID2ROT = {2: 13, 3: 14, 4: 15, 6: 1, 7: 2, 8: 3, 10: 4, 11: 5, 12: 6, 14: 10, 15: 11, 16: 12, 18: 7, 19: 8, 20: 9}


def get_3djoints(csv_data, frame_idx=0):
    """convert2mano.get_3djoints: per name, every column containing it except 'End' columns, in column order."""
    out = []
    for names in (LEFT, RIGHT):
        vals = [csv_data[k][frame_idx] for n in names for k in csv_data.keys() if n in k and 'End' not in k]
        out.append(np.array(vals).reshape(-1, 3))
    return tuple(out)


def axangle2mat(axis, angle):
    """transforms3d.axangles.axangle2mat(axis, angle, is_normalized=False) (published formula)."""
    x, y, z = axis
    n = math.sqrt(x * x + y * y + z * z)
    with np.errstate(invalid='ignore', divide='ignore'):
        x, y, z = np.float64(x) / n, np.float64(y) / n, np.float64(z) / n
    c, s = math.cos(angle), math.sin(angle)
    C = 1 - c
    xs, ys, zs, xC, yC, zC = x * s, y * s, z * s, x * C, y * C, z * C
    xyC, yzC, zxC = x * yC, y * zC, z * xC
    return np.array([[x * xC + c, xyC - zs, zxC + ys], [xyC + zs, y * yC + c, yzC - xs], [zxC - ys, yzC + xs, z * zC + c]])


def adaptive_IK(T_, P_):
    """AIK.adaptive_IK: T, P [21,3] -> [1,16,3,3] float64."""
    T, P = np.asarray(T_, np.float64), np.asarray(P_, np.float64)
    R, Rk, q = {}, {}, {0: T[0]}
    idx = [1, 5, 9, 13, 17]
    H = (T[idx] - T[0]).T @ (P[idx] - P[0])
    U, S, Vt = np.linalg.svd(H)
    V = Vt.T
    R0 = V @ U.T
    if abs(np.linalg.det(R0) + 1) < 1e-6 and (abs(S) < 1e-4).sum():
        V = V.copy()
        V[:, 2] = -V[:, 2]
        R0 = V @ U.T
    for k in [0] + idx:
        R[k] = R0
    with np.errstate(invalid='ignore', divide='ignore'):
        for k in KINEMATIC_TREE:
            pa = SNAP_PARENT[k]
            q[pa] = R[pa] @ (T[pa] - T[SNAP_PARENT[pa]]) + q[SNAP_PARENT[pa]]
            dp = np.linalg.inv(R[pa]) @ (P[k] - q[pa])
            dt = T[k] - T[pa]
            cr = np.cross(dt, dp)
            axis = cr / (np.linalg.norm(cr) + 1e-8)
            alpha = np.arccos(np.dot(dt, dp) / ((np.linalg.norm(dt) + 1e-8) * (np.linalg.norm(dp) + 1e-8)))
            Rk[k] = axangle2mat(axis, alpha) @ axangle2mat(dt, 0.0)
            R[k] = R[pa] @ Rk[k]
    out = np.zeros((1, 16, 3, 3))
    out[0, 0] = R0
    for k, v in ID2ROT.items():
        out[0, v] = Rk[k]
    return out


def prescale(template, joints):
    """convert2mano.py:166-168 on a float32 template [21,3] and float64 joints [21,3] -> P."""
    ratio = np.linalg.norm(template[9] - template[0]) / np.linalg.norm(joints[9] - joints[0])
    P = joints * ratio
    return P - P[0] + template[0]


def lr_schedule(lr, n):
    """The learning rate each of the n steps uses: lr, then lr * (n - i) / n set after step i (convert2mano.py:199-200)."""
    return [lr] + [lr * (n - i) / n for i in range(n - 1)]


def ori_pose(layer, pose_R, mat2aa):
    """convert2mano.py:222-228: [mat2aa(pose_R[:, 0]), pca2axis(mat2aa(pose_R[:, 1:])) - hands_mean] -> [B,48]."""
    B = pose_R.shape[0]
    aa = mat2aa(pose_R.reshape(-1, 3, 3)).reshape(B, 48)
    return torch.cat([aa[:, :3], layer.pca2axis(aa[:, 3:]) - layer.hands_mean], 1)


def eager_fit(layer, pose_R, joints, mat2aa, iterations=200, lr=0.1):
    """The reference loop (convert2mano.py:175-200) batched: torch.optim.Adam over pose_R [B,16,3,3] and beta [B,10] with `layer` and
    `mat2aa`, loss = sum over frames of each frame's mean |(j - j0) - target|.  -> (pose_R, beta, per-iteration losses [n,B])."""
    B = pose_R.shape[0]
    pose = torch.nn.Parameter(pose_R.float().clone())
    beta = torch.nn.Parameter(torch.zeros(B, 10, device=pose_R.device))
    target = ((joints - joints[:, 0:1]) / 100).float()
    opt = torch.optim.Adam([pose, beta], lr=lr)
    hist = []
    for i in range(iterations):
        _, j = layer(pose[:, 0], mat2aa(pose[:, 1:].reshape(-1, 3, 3)).reshape(B, 45), beta)
        per = ((j - j[:, 0:1]) - target).abs().mean(dim=(1, 2))
        hist.append(per.detach().clone())
        opt.zero_grad()
        per.sum().backward()
        opt.step()
        for g in opt.param_groups:
            g['lr'] = lr * (iterations - i) / iterations
    return pose.detach(), beta.detach(), torch.stack(hist)
