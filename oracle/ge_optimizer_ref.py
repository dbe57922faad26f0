"""Inputs and the eager driver of the two-hand pose optimiser's tests and benchmark (renderih_b200/ge_optimizer.py).

inputs() builds the keyword arguments of GeOptimizer.set_opt_val in the caller's form (batch_optimize_mocap_origin.py:706-734) from a
seed; nature_weights() picks discriminator weights whose mask splits those poses; build() makes a renderih_b200 GeOptimizer on the
synthetic MANO tensors, the reference's anchor tables (stored in tests/golden/geo_loss_synth.pt) and a closed convex-hull mesh for the
penetration term.  eager_optimize() is the reference's optimize() loop (geo_optimizer_both_batch.py:861-930) made of the same CUDA loss
modules, torch.optim.Adam and torch.optim.lr_scheduler.ReduceLROnPlateau; with sync=True it also synchronises with the host where the
reference does (the 11 .item() of loss_fn's dict, the print's four tensors; scheduler.step(loss) always calls float(loss)).
"""
import math
import os

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD_DIR = os.path.join(ROOT, 'tests', 'golden')
CALLER_SPLIT = ([0], list(range(1, 16)))              # hand_pose_gt / hand_pose_init of the caller (:716-717, :723-724)
THRESH = -math.log(1.5)                               # the nature mask p1 < 1.5 p0 is l0 - l1 > -ln 1.5


def poses(B, seed, scale=0.3):
    """Unnormalised [B,16,4] quaternions of both hands, the identity plus scale * N(0, 1)."""
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(B, 16, 4, generator=g) * scale + torch.tensor([1.0, 0.0, 0.0, 0.0]) for _ in range(2)]


def inputs(B, seed, split=(CALLER_SPLIT, CALLER_SPLIT), device='cpu', scale=0.3, shape_scale=0.5):
    """set_opt_val's keyword arguments (CPU tensors unless device is given): poses from poses(B, seed, scale), betas shape_scale *
    N(0, 1)."""
    q_r, q_l = poses(B, seed, scale)
    g = torch.Generator().manual_seed(10_000 + seed)
    tsl_r = torch.tensor([0.02, 0.0, 0.0]) + 0.01 * torch.randn(B, 3, generator=g)
    tsl_l = torch.tensor([-0.02, 0.0, 0.0]) + 0.01 * torch.randn(B, 3, generator=g)
    kw = dict(vertex_contact=(torch.rand(B, 108, generator=g) < 0.5).long(), contact_region=torch.zeros(B, 108, dtype=torch.long),
              anchor_id=torch.randint(0, 108, (B, 108, 4), generator=g), anchor_elasti=torch.rand(B, 108, 4, generator=g),
              anchor_padding_mask=(torch.rand(B, 108, 4, generator=g) < 0.3).long(),
              hand_shape_init=torch.randn(B, 20, generator=g) * shape_scale, hand_tsl_init=tsl_r, obj_tsl_init=tsl_l,
              obj_anchors=torch.randn(B, 108, 3, generator=g) * 0.05, obj_normals=torch.randn(B, 108, 3, generator=g),
              optimize_it=torch.ones(B, dtype=torch.bool), batch_size=B,
              consistent_mask=[torch.rand(B, 16, generator=g), torch.rand(B, 16, generator=g)], runtime_vis=9527)
    for name, q, (gi, vi) in (('hand_pose', q_r, split[0]), ('obj_pose', q_l, split[1])):
        kw[name + '_gt'] = (list(gi), q[:, list(gi)].contiguous())
        kw[name + '_init'] = (list(vi), q[:, list(vi)].contiguous())
    if device != 'cpu':
        kw = to_device(kw, device)
    return kw


def to_device(kw, device):
    out = {}
    for k, v in kw.items():
        if isinstance(v, torch.Tensor):
            out[k] = v.to(device)
        elif isinstance(v, tuple):
            out[k] = (v[0], v[1].to(device))
        elif isinstance(v, list):
            out[k] = [t.to(device) for t in v]
        else:
            out[k] = v
    return out


def nature_weights(B, seed, wseed, scale=40.0, rule='median', pose_scale=0.3):
    """(seed, pred_scale, pred_bias) of discriminator weights for poses(B, seed, pose_scale): 'median' puts the mask threshold half-way between the
    two middle rows of both hands, 'one_empty' between the hands' largest rows so that one hand's mask is empty, 'all' one logit below
    the lowest row, so that every row is masked and stays clear of the threshold."""
    from oracle import make_golden_nature, nature_ref
    sd = nature_ref.init_state_dict(wseed, scale)
    d = make_golden_nature._diffs(sd, *[F.normalize(q, dim=-1) for q in poses(B, seed, pose_scale)])
    if rule == 'all':                 # every row masked, the threshold `margin` = 1 logit below the lowest row
        return wseed, scale, (THRESH - float(d.min()) + 1.0, 0.0)
    if rule == 'median':
        v = d.flatten().sort().values
        k = v.numel() // 2
        bias = (THRESH - float(v[k - 1] + v[k]) / 2, 0.0) if v.numel() > 1 else (THRESH - float(v[0]) + 1.0, 0.0)
    else:
        lo, hi = sorted(float(d[h].max()) for h in range(2))
        bias = (THRESH - (lo + hi) / 2, 0.0)
    return wseed, scale, bias


def hull_faces():
    """A closed convex-hull mesh over 778 points on an ellipsoid and 16 interleaved parts: NewLoss's faces and part_vert."""
    from scipy.spatial import ConvexHull
    rng = np.random.default_rng(0)
    pts = rng.normal(size=(778, 3))
    pts *= np.array([1.0, 0.6, 0.35]) / np.linalg.norm(pts, axis=1, keepdims=True)
    return ConvexHull(pts).simplices, [np.arange(k, 778, 16) for k in range(16)]


def build(weights, lr=1e-2, n_iter=50, lambda_contact_loss=10.0, lambda_repulsion_loss=0.5, device='cuda'):
    """A renderih_b200 GeOptimizer on the synthetic MANO tensors with discriminator weights `weights` = (seed, scale, bias)."""
    from oracle import nature_ref
    from renderih_b200 import assets as A
    from renderih_b200.ge_optimizer import GeOptimizer
    geo = torch.load(os.path.join(GOLD_DIR, 'geo_loss_synth.pt'), weights_only=False)
    faces, parts = hull_faces()
    return GeOptimizer(device, lr=lr, n_iter=n_iter, mano_root={s: A.synthetic_mano(0, s) for s in ('right', 'left')},
                       lambda_contact_loss=lambda_contact_loss, lambda_repulsion_loss=lambda_repulsion_loss, mode='both',
                       discrim=nature_ref.init_state_dict(*weights), sdf_faces=faces, sdf_part_vert=parts,
                       anchor_face_vert_idx=geo['anchor_fvi'].numpy(), anchor_weight=geo['anchor_w'].numpy())


def assemble(gt_idx, gt_pose, var_idx, var_pose):
    """GeOptimizer.assemble_batch_pose_vec (:480-485)."""
    idx = torch.cat((torch.Tensor(gt_idx).long(), torch.Tensor(var_idx).long()))
    return torch.cat((gt_pose, var_pose), dim=1)[:, torch.argsort(idx), :]


def eager_optimize(opt, kw, n_iter, sync=False, history=None):
    """The reference's optimize() loop on opt's CUDA loss modules (opt: a renderih_b200 GeOptimizer after set_opt_val(**kw)), with
    torch.optim.Adam and ReduceLROnPlateau as set_opt_val builds them (:413-432) -> out_dict.  history, if a list, receives
    (float total, [lr of each group]) per iteration."""
    dev = opt.device
    kw = to_device(kw, dev)
    B = kw['batch_size']
    leaves = [kw['hand_tsl_init'].detach().clone().requires_grad_(True), kw['obj_tsl_init'].detach().clone().requires_grad_(True),
              kw['hand_pose_init'][1].detach().clone().requires_grad_(True), kw['obj_pose_init'][1].detach().clone().requires_grad_(True)]
    lr = opt.lr
    optimizer = torch.optim.Adam([{'params': [leaves[0]], 'lr': 0.01 * lr}, {'params': [leaves[1]], 'lr': 0.01 * lr},
                                  {'params': [leaves[2]], 'lr': 1 * lr}, {'params': [leaves[3]], 'lr': 1 * lr}], lr=lr)
    scheduler = torch.optim.lr_scheduler.ReduceLROnPlateau(optimizer, min_lr=1e-5, mode='min', factor=0.5, patience=20)
    shape = kw['hand_shape_init']
    coef = opt.coef_val
    pr = pl = None
    for _ in range(n_iter):
        optimizer.zero_grad()
        pr = assemble(kw['hand_pose_gt'][0], kw['hand_pose_gt'][1], kw['hand_pose_init'][0], leaves[2])
        pl = assemble(kw['obj_pose_gt'][0], kw['obj_pose_gt'][1], kw['obj_pose_init'][0], leaves[3])
        vr = opt.mano_layer(pr, shape[:, :10])[0] + leaves[0].unsqueeze(1)
        vl = opt.sub_mano_layer(pl, shape[:, 10:])[0] + leaves[1].unsqueeze(1)
        qn, edge, contact, ergo = opt.prior(pr, pl, vr, vl)
        pen = opt.anti_penetration_loss_fun(torch.cat((vr.unsqueeze(1), vl.unsqueeze(1)), 1)).mean()
        nat = opt.nature(F.normalize(pr, dim=-1)[:, 1:], F.normalize(pl, dim=-1)[:, 1:])
        if sync:      # :803-804 and :847-857 (the seven constant terms are .item()'d too)
            '{} {} {} {}'.format(nat, ergo, pen, 100 * coef['lambda_contact_loss'] * contact)
            zero = torch.zeros(1, device=dev)
            [t.detach().cpu().item() for t in (qn, zero, edge, zero, zero, zero, contact, zero, zero, zero, zero)]
        loss = qn + edge + 1 * coef['lambda_contact_loss'] * contact + 0.02 * coef['lambda_repulsion_loss'] * pen + ergo + nat
        loss.backward()
        optimizer.step()
        scheduler.step(loss)
        if history is not None:
            history.append((float(loss), [g['lr'] for g in optimizer.param_groups]))
    return dict(optimized_hand_pose=pr.detach().cpu(), optimized_hand_tsl=leaves[0].detach().cpu(),
                optimized_sub_hand_pose=pl.detach().cpu(), optimized_sub_hand_tsl=leaves[1].detach().cpu())


LRS = [1e-4, 1e-4, 1e-2, 1e-2]         # the four groups' lrs at lr = 1e-2


def torch_lrs(losses, lrs):
    """The lr of each group after every torch ReduceLROnPlateau step (the optimiser's settings) on the float32 losses."""
    params = [torch.zeros(1, requires_grad=True) for _ in lrs]
    opt = torch.optim.Adam([{'params': [p], 'lr': lr} for p, lr in zip(params, lrs)], lr=lrs[-1])
    sched = torch.optim.lr_scheduler.ReduceLROnPlateau(opt, min_lr=1e-5, mode='min', factor=0.5, patience=20)
    out = []
    for a in losses:
        sched.step(torch.tensor(a, dtype=torch.float32))
        out.append([g['lr'] for g in opt.param_groups])
    return out


def _exact_tie():
    """float32 values (b, a) with float(a) == float(b) * (1 - 1e-4) exactly."""
    for i in range(1, 200000):
        b = float(torch.tensor(10000.0 + i, dtype=torch.float32))
        a = b * (1.0 - 1e-4)
        if float(torch.tensor(a, dtype=torch.float32)) == a:
            return b, a
    raise AssertionError('no exact tie found')


def crafted_sequences():
    """Loss sequences for the scheduler checks: NaN, an exact tie at best * (1 - 1e-4), the min_lr floor, the eps rule, random."""
    b, a = _exact_tie()
    g = torch.Generator().manual_seed(0)
    return {'nan': [5.0, float('nan')] * 40 + [1.0] * 30,
            'exact_tie': [b] + [a] * 60 + [a * 0.5] + [a * 0.5] * 30,
            'min_lr_floor': [1.0] * 300,
            'eps_rule': [2.0, 1.0] + [1.0] * 150,
            'random': (torch.rand(300, generator=g) * 3 + torch.linspace(3, 0, 300)).tolist()}
