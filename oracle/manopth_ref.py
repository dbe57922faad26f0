"""Independent float64 torch statement of the pose optimiser's quaternion hand model (pose_data_optimize/manopth/manopth/manolayer.py in
quat/quat mode without PCA), written from the math: quaternion -> rotation with entries over |q|^2, shape and pose blend shapes, the
joint regressor, the three-level kinematic chain, linear blend skinning, palm / finger-tip joints, the joint reordering and the
centring rule.  Autograd through it gives gradients with the reference's semantics.

TEST INFRASTRUCTURE -- never imported by the product package.
"""
import numpy as np
import torch

from renderih_b200.assets import synthetic_mano

PARENTS = [-1, 0, 1, 2, 0, 4, 5, 0, 7, 8, 0, 10, 11, 0, 13, 14]
OUTPUT_ORDER = [0, 13, 14, 15, 16, 1, 2, 3, 17, 4, 5, 6, 18, 10, 11, 12, 19, 7, 8, 9, 20]
TIPS = {'right': [745, 317, 444, 556, 673], 'left': [745, 317, 445, 556, 673]}
PALM = (95, 22)


def quat_to_rotmat(q):
    """[..., 4] (w, x, y, z), any norm -> [..., 3, 3] rotation of q / |q| (each entry of the unit-norm formula scaled by 1 / |q|^2)."""
    w, x, y, z = q.unbind(-1)
    n = (q * q).sum(-1)
    rows = [[w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)],
            [2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)],
            [2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z]]
    return torch.stack([torch.stack(r, -1) for r in rows], -2) / n[..., None, None]


def tables(mano, side):
    """float64 tensors of a MANO dict as the layer holds them (left hands: the x rows of shapedirs negated)."""
    t = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.float64)
    jr = mano['J_regressor']
    jr = jr.toarray() if hasattr(jr, 'toarray') else jr
    sd = t(mano['shapedirs']).clone()
    if side == 'left':
        sd[:, 0, :] = -sd[:, 0, :]
    return {'shapedirs': sd, 'posedirs': t(mano['posedirs']), 'v_template': t(mano['v_template']), 'J_regressor': t(jr), 'weights': t(mano['weights'])}


def _affine(R, t):
    """[..., 3, 3], [..., 3] -> [..., 4, 4]"""
    top = torch.cat([R, t[..., None]], -1)
    bottom = top.new_zeros(top.shape[:-2] + (1, 4))
    bottom[..., 0, 3] = 1
    return torch.cat([top, bottom], -2)


def forward(tab, side, quat, betas=None, trans=None, center_idx=None, root_palm=False, share_betas=False):
    """quat [B,16,4] or [B,64]; betas [B,10] or None (zeros); trans broadcastable to [B,3] or None -> verts [B,778,3], joints [B,21,3],
    transf [B,16,4,4], in the dtype and on the device of quat."""
    B = quat.shape[0]
    q = quat.reshape(B, 16, 4)
    if side == 'left':
        q = q * torch.tensor([1.0, 1.0, -1.0, -1.0], dtype=q.dtype, device=q.device)
    R = quat_to_rotmat(q)                                                   # [B,16,3,3]
    if betas is None:
        beta = q.new_zeros(B, 10)
    elif share_betas:
        beta = betas.mean(0, keepdim=True).expand(B, 10)
    else:
        beta = betas
    v_shaped = tab['v_template'].to(q)[None] + torch.einsum('vck,bk->bvc', tab['shapedirs'].to(q), beta)
    J = torch.einsum('jv,bvc->bjc', tab['J_regressor'].to(q), v_shaped)            # rest joints [B,16,3]
    eye = torch.eye(3, dtype=q.dtype, device=q.device)
    pose_feat = (R[:, 1:] - eye).reshape(B, 135)
    v_posed = v_shaped + torch.einsum('vck,bk->bvc', tab['posedirs'].to(q), pose_feat)
    G = []
    for i in range(16):
        p = PARENTS[i]
        if p < 0:
            G.append(_affine(R[:, 0], J[:, 0]))
        else:
            G.append(G[p] @ _affine(R[:, i], J[:, i] - J[:, p]))
    G = torch.stack(G, 1)                                                   # [B,16,4,4] global transforms
    A = G @ _affine(eye.expand(B, 16, 3, 3), -J)                            # rest pose -> posed, per joint
    T = torch.einsum('vj,bjrc->bvrc', tab['weights'].to(q), A)
    verts = (T[..., :3, :3] @ v_posed[..., None])[..., 0] + T[..., :3, 3]
    joints16 = G[:, :, :3, 3]
    if root_palm:
        joints16 = torch.cat([(verts[:, PALM[0]] + verts[:, PALM[1]])[:, None] / 2, joints16[:, 1:]], 1)
    joints = torch.cat([joints16, verts[:, TIPS[side]]], 1)[:, OUTPUT_ORDER]
    translate = trans is not None and bool(torch.any(trans != 0))
    tr = q.new_zeros(B, 3) if trans is None else trans.to(q).expand(B, 3)
    if translate:
        centre = q.new_zeros(B, 3)
        verts, joints = verts + tr[:, None], joints + tr[:, None]
    else:
        centre = joints[:, center_idx] if center_idx is not None else q.new_zeros(B, 3)
        verts, joints = verts - centre[:, None], joints - centre[:, None]
    transf = _affine(G[:, :, :3, :3], G[:, :, :3, 3] - centre[:, None] + tr[:, None])
    return verts, joints, transf


def weighted_case(inp, cfg, dtype=torch.float64):
    """A golden-style case: inputs dict (quat, betas, trans, weights wv / wj / wt) and cfg (side, betas 'rows' | 'none', trans
    'none' | 'zeros' | 'nonzero', center_idx, root_palm, share_betas) -> verts, joints, transf and the gradients of
    <verts, wv> + <joints, wj> + <transf, wt> w.r.t. quat, betas, trans (None where the input is absent)."""
    tab = tables(synthetic_mano(0, cfg['side']), cfg['side'])
    B = inp['quat'].shape[0]
    q = inp['quat'].to(dtype).requires_grad_(True)
    b = inp['betas'].to(dtype).requires_grad_(True) if cfg['betas'] == 'rows' else None
    t = {'none': None, 'zeros': torch.zeros(B, 3, dtype=dtype), 'nonzero': inp['trans'].to(dtype)}[cfg['trans']]
    if t is not None:
        t.requires_grad_(True)
    v, j, tf = forward(tab, cfg['side'], q, b, t, cfg['center_idx'], cfg['root_palm'], cfg['share_betas'])
    ((v * inp['wv'].to(dtype)).sum() + (j * inp['wj'].to(dtype)).sum() + (tf * inp['wt'].to(dtype)).sum()).backward()
    return v, j, tf, q.grad, None if b is None else b.grad, None if t is None else t.grad
