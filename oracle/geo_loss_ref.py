"""Independent float64 torch statement of the pose optimiser's hand-prior and contact terms for both hands
(pose_data_optimize/hocontact/postprocess/geo_loss.py, geo_optimizer_both_batch.py:567-616,705-757, scripts/HandPoseConverter.py),
written from the math: anchors, contact energy, quaternion-norm, edge length and the ergonomics prior on the converter's joint frames.
Autograd through it gives gradients with the reference's semantics.  `flags` marks samples with an angle within rounding of a point
where the loss or its gradient jumps (the in-place zeroing of negative bend angles, the atan2 branch cut) or of a degree limit.

TEST INFRASTRUCTURE -- never imported by the product package.
"""
import math

import numpy as np
import torch

from oracle import manopth_ref as M

HPC_BETAS = [0.5082395, -0.39488167, -1.7484332, 1.6630946, 0.34428665, -1.37387, 0.38293332, 1.196094, 0.6538949, -0.94331187]
WEIGHTS = (1.0, 1.0, 10.0, 1.0)           # the optimiser's weights of quat-norm, edge, contact (lambda_contact_loss) and ergonomics
# ergonomics index t = joint t + 1
BEND = [(-25, 70), (-4, 110), (-8, 90), (-25, 80), (-7, 100), (-8, 90), (-22, 70), (-8, 90), (-8, 90), (-25, 70), (-10, 100), (-8, 90),
        (-20, 40), (-35, 50), (-10, 100)]
SPLANK = {0: (-25, 15), 3: (-15, 15), 9: (-25, 15), 6: (-20, 30), 12: (-30, 30)}
NO_TWIST_SPLANK = [1, 2, 4, 5, 7, 8, 10, 11, 13, 14]
NO_TWIST = [0, 3, 6, 9]
THUMB_BASE = 12
KINK_TOL_DEG = 1e-3


def edges(faces):
    """First-seen undirected edges of faces [F,3]: (0,1), (1,2), (0,2) of each face -> [E,2] int64 with each pair as list({i, j})."""
    out, seen = [], set()
    for f in np.asarray(faces, dtype=np.int64):
        for a, b in ((f[0], f[1]), (f[1], f[2]), (f[0], f[2])):
            s = frozenset((int(a), int(b)))
            if s not in seen:
                seen.add(s)
                out.append(list({int(a), int(b)}))
    return np.asarray(out, dtype=np.int64)


def converter(side, joints, transf):
    """Joint frames of HandPoseConverter at the rest pose -> (invM_U_n_0, invU_M_n_1) [16,3,3] float64."""
    joints, R = np.asarray(joints, np.float64), np.asarray(transf, np.float64)[:, :3, :3]
    sign = 1.0 if side == 'right' else -1.0
    chains = [[0, 13, 14, 15], [0, 1, 2, 3], [0, 4, 5, 6], [0, 10, 11, 12], [0, 7, 8, 9]]
    out21 = [5, 6, 7, 9, 10, 11, 17, 18, 19, 13, 14, 15, 1, 2, 3]    # output joint of native joint k + 1
    frames = [np.eye(3) if side == 'right' else np.diag([1.0, -1.0, -1.0])]
    for k in range(15):
        x = sign * (joints[out21[k]] - joints[out21[k] + 1])
        x = R[k + 1].T @ x
        up = np.array([0.0, sign, 0.0]) if k < 12 else np.array([1.0, sign, sign])
        z = np.cross(x, up)
        y = np.cross(z, x)
        frames.append(np.stack([v / np.linalg.norm(v) for v in (x, y, z)], 1))
    U = [R[i] @ frames[i] for i in range(16)]
    inv_m0, inv_u1 = np.tile(np.eye(3), (16, 1, 1)), np.tile(np.eye(3), (16, 1, 1))
    for ch in chains:
        for pos, a in enumerate(ch):
            prev = ch[pos - 1] if pos else 0
            inv_u1[a] = U[a].T @ R[a]
            inv_m0[a] = R[prev].T @ U[prev]
    return inv_m0, inv_u1


def rest(mano, side):
    """-> (identity-pose zero-beta vertices [778,3], the converter's rest joints [21,3] and transforms [16,4,4]) in float64."""
    tab = M.tables(mano, side)
    ident = torch.zeros(1, 16, 4, dtype=torch.float64)
    ident[..., 0] = 1
    v, _, _ = M.forward(tab, side, ident, None, None, 0)
    _, j, tf = M.forward(tab, side, ident, torch.tensor([HPC_BETAS], dtype=torch.float64), None, 9)
    return v[0], j[0].numpy(), tf[0].numpy()


def tables(mano_right, mano_left, fvi, aw, converters=None):
    """Everything the terms need: edges of the RIGHT faces, each side's rest edge lengths, the converter matrices (computed, or given as
    {side: (invM_U_n_0, invU_M_n_1)}), the anchor tables."""
    e = edges(mano_right['f'])
    out = {'edges': torch.from_numpy(e), 'fvi': torch.as_tensor(np.asarray(fvi), dtype=torch.int64),
           'aw': torch.as_tensor(np.asarray(aw), dtype=torch.float64), 'rest': {}, 'conv': {}}
    for side, mano in (('right', mano_right), ('left', mano_left)):
        v, j, tf = rest(mano, side)
        out['rest'][side] = (v[e[:, 0]] - v[e[:, 1]]).norm(dim=-1)
        m0, u1 = converters[side] if converters else converter(side, j, tf)
        out['conv'][side] = (torch.as_tensor(np.asarray(m0), dtype=torch.float64), torch.as_tensor(np.asarray(u1), dtype=torch.float64))
    return out


def anchors(verts, fvi, aw):
    """[B,778,3] -> [B,A,3]"""
    v0, v1, v2 = verts[:, fvi[:, 0]], verts[:, fvi[:, 1]], verts[:, fvi[:, 2]]
    return v0 + aw[:, 0:1] * (v1 - v0) + aw[:, 1:2] * (v2 - v0)


def local_frames(q, side, conv):
    """[B,16,4] unnormalised -> M = zero_ja^T ja [B,15,3,3] for joints 1..15."""
    p = q / q.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    if side == 'left':
        p = p * torch.tensor([1.0, 1.0, -1.0, -1.0], dtype=p.dtype, device=p.device)
    R = M.quat_to_rotmat(p)[:, 1:]
    A, C = conv[0][1:].transpose(1, 2), conv[1][1:].transpose(1, 2)
    Z = A @ C
    return Z.transpose(1, 2) @ (A @ R @ C)


def ergonomics(Mj):
    """hand_pose_ergonomics_loss on M [B,15,3,3] -> (term, kink flags [B])."""
    deg = 180.0 / math.pi
    x = Mj[..., :, 0]
    res = (Mj[:, NO_TWIST_SPLANK, 2, 0] ** 2).mean() + (Mj[:, NO_TWIST_SPLANK, 2, 1] ** 2).mean() + ((Mj[:, NO_TWIST_SPLANK, 2, 2] - 1) ** 2).mean()
    twist = (Mj[..., 2, 1] - Mj[..., 1, 2]) / 2
    res = res + (twist[:, NO_TWIST] ** 2).mean() + ((twist[:, THUMB_BASE] - 0.5).clamp(min=0) ** 2).mean()
    bend = torch.atan2(x[..., 1], x[..., 0]) * deg
    splank = torch.atan2(-x[..., 2], x[..., 0]) * deg
    near = lambda a, v: (a - v).abs() < KINK_TOL_DEG
    flags = near(bend[:, 7], 0) | near(bend[:, 10], 0) | (bend.abs() > 180 - KINK_TOL_DEG).any(1) | (splank.abs() > 180 - KINK_TOL_DEG).any(1)
    for t, (lo, hi) in SPLANK.items():
        res = res + ((torch.relu(splank[:, t] - hi) + torch.relu(lo - splank[:, t])) / deg).pow(2).mean()
        flags = flags | near(splank[:, t], lo) | near(splank[:, t], hi)
    for t, (lo, hi) in enumerate(BEND):
        res = res + ((torch.relu(bend[:, t] - hi) + torch.relu(lo - bend[:, t])) / deg).pow(2).mean()
        flags = flags | near(bend[:, t], lo) | near(bend[:, t], hi)
    b = torch.where(bend < 0, torch.zeros_like(bend), bend) / deg
    res = res + (b[:, 10] - b[:, 7] * 0.75).clamp(max=0).pow(2).mean()
    return res, flags


def terms(tab, q_r, q_l, v_r, v_l, anchor_id, elastic, mask):
    """-> ([quat_norm, edge, contact, ergonomics] as 0-dim tensors, kink flags [B]); both hands summed."""
    e = tab['edges']
    qn = edge = ergo = 0
    flags = torch.zeros(q_r.shape[0], dtype=torch.bool, device=q_r.device)
    for side, q, v in (('right', q_r, v_r), ('left', q_l, v_l)):
        qn = qn + (((q * q).sum(-1) - 1) ** 2).mean()
        edge = edge + (((v[:, e[:, 0]] - v[:, e[:, 1]]).norm(dim=-1) - tab['rest'][side]) ** 2).mean()
        r, f = ergonomics(local_frames(q, side, tab['conv'][side]))
        ergo, flags = ergo + r, flags | f
    a_main, a_sub = anchors(v_r, tab['fvi'], tab['aw']), anchors(v_l, tab['fvi'], tab['aw'])
    B, A, D = anchor_id.shape
    picked = a_main[torch.arange(B, device=a_main.device)[:, None, None], anchor_id.to(a_main.device).long()]           # [B,A,D,3]
    num = (elastic.to(picked) * ((a_sub[:, :, None] - picked) ** 2).sum(-1)).sum()
    total = int(mask.long().sum())
    contact = num / total if total > 0 else num * 0
    return [qn, edge, contact, ergo], flags


def weighted_case(tab, inp, weights=WEIGHTS, dtype=torch.float64):
    """inp: quat_r, quat_l [B,16,4], verts_r, verts_l [B,778,3], anchor_id, elastic, mask [B,A,D] -> (terms [4], gradients of the
    weighted total w.r.t. quat_r, quat_l, verts_r, verts_l, flags)."""
    leaves = [inp[k].to(dtype).clone().requires_grad_(True) for k in ('quat_r', 'quat_l', 'verts_r', 'verts_l')]
    t, flags = terms(tab, *leaves, inp['anchor_id'], inp['elastic'], inp['mask'])
    sum(w * x for w, x in zip(weights, t)).backward()
    return torch.stack([x.detach() for x in t]), [l.grad for l in leaves], flags
