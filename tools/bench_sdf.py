"""Timing of the two-hand anti-penetration SDF loss (renderih_b200/sdf.py) at grid size 32 with interpenetrating posed hands: one
forward + backward of the fused `NewLoss`, and of the dense formulation the reference uses (our dense grid of both hands, then torch
grid_sample over the 16 parts), CUDA events around --iters calls after --warmup calls.  Faces: the closed MANO hand under the asset root
($RIH_ASSET_ROOT) when present, else the convex hull of 778 points on a perturbed ellipsoid (the same 1552-face size); "mesh" says which.
Prints one JSON line with the device name and power limit read in the same run, and per batch size the voxels the fused kernel evaluates
against the dense 2 * B * G^3.
usage: python tools/bench_sdf.py [--batches 64,2048,6144] [--iters 5] [--warmup 2] [--dense-max-batch 6144]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

G = 32


def _power_limit():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, timeout=30).stdout.decode().strip()
        return out or 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def _time(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def _faces_and_parts():
    from renderih_b200 import sdf as rs
    from renderih_b200.assets import default_asset_root
    root = default_asset_root()
    obj, pv = os.path.join(root, rs.CLOSED_HAND_OBJ), os.path.join(root, rs.PART_VERT)
    if os.path.exists(obj) and os.path.exists(pv):
        return rs.load_obj_faces(obj), rs.load_part_vert(pv), 'closed_mano'
    from scipy.spatial import ConvexHull
    rng = np.random.default_rng(0)
    p = rng.normal(size=(778, 3))
    p *= np.array([1.0, 0.6, 0.35]) / np.linalg.norm(p, axis=1, keepdims=True)
    return ConvexHull(p).simplices.astype(np.int64), [np.arange(k, 778, 16) for k in range(16)], 'hull'


def _hands(B, seed=0):
    from renderih_b200 import assets as A
    from renderih_b200.manolayer import ManoLayer, rodrigues_batch
    g = torch.Generator().manual_seed(seed)
    out = []
    for side in ('right', 'left'):
        layer = ManoLayer(A.synthetic_mano(0, side), center_idx=9, use_pca=True)
        rot = rodrigues_batch((torch.rand(B, 3, generator=g) - 0.5) * 2.0).cuda()
        v, _ = layer(rot, (torch.randn(B, 45, generator=g) * 0.6).cuda(), (torch.randn(B, 10, generator=g) * 0.5).cuda())
        out.append(v)
    return torch.stack(out, 1).contiguous()


def _touched_voxels(v, center, scale):
    """Distinct grid corners the other hand's vertices touch, summed over samples and both grids (what the fused kernel evaluates)."""
    B = v.shape[0]
    total = 0
    for h in (0, 1):
        x = (v[:, 1 - h] - center[:, h, None]) / scale[:, h, None, None]
        i0 = torch.floor((x + 1) / 2 * (G - 1)).long()
        ids = []
        for n in range(8):
            idx = i0 + torch.tensor([n & 1, (n >> 1) & 1, n >> 2], device=v.device)
            ok = ((idx >= 0) & (idx < G)).all(-1)
            vox = (idx[..., 2] * G + idx[..., 1]) * G + idx[..., 0] + torch.arange(B, device=v.device)[:, None] * G ** 3
            ids.append(torch.where(ok, vox, torch.full_like(vox, -1)).reshape(-1))
        u = torch.unique(torch.cat(ids))
        total += int((u >= 0).sum())
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batches', default='64,2048,6144')
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--dense-max-batch', type=int, default=6144, help='largest batch timed with the dense formulation')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_sdf.py needs a CUDA device')
    from renderih_b200.sdf import NewLoss, penetration, sdf
    faces, parts, mesh = _faces_and_parts()
    crit = NewLoss(faces=faces, part_vert=parts)
    part_idx = [torch.tensor(sorted(np.unique(np.asarray(list(p)))), device='cuda') for p in parts]
    res = {'device': torch.cuda.get_device_name(), 'power_limit': _power_limit(), 'grid_size': G, 'faces': int(len(faces)), 'mesh': mesh,
           'iters': args.iters, 'warmup': args.warmup}
    for B in [int(b) for b in args.batches.split(',')]:
        v = _hands(B).requires_grad_(True)

        def fused():
            crit(v).sum().backward()

        def dense():
            vd = v.detach()
            lo, hi = vd.min(dim=2)[0], vd.max(dim=2)[0]
            c, s = ((lo + hi) / 2)[:, :, None], (0.55 * (hi - lo).max(dim=-1)[0])[:, :, None, None]
            grids = [sdf(crit.faces, ((vd[:, h] - c[:, h]) / s[:, h]).contiguous(), G) for h in (0, 1)]
            total = 0
            for h in (0, 1):
                x = (v[:, 1 - h] - c[:, h]) / s[:, h]
                acc = torch.zeros(B, v.shape[2], device='cuda')
                for idx in part_idx:
                    val = torch.nn.functional.grid_sample(grids[h][:, None], x[:, idx].view(B, -1, 1, 1, 3), align_corners=True).view(B, -1)
                    acc = acc.index_add(1, idx, val)
                total = total + (acc / 4).sum(1)
            total.sum().backward()

        _, _, _, _, center, scale = penetration(v.detach(), crit.faces, crit._mult_for(v.shape[2]))
        row = {'fused_newloss_ms': round(_time(fused, args.iters, args.warmup), 3),
               'voxels_evaluated': _touched_voxels(v.detach(), center, scale), 'voxels_dense': 2 * B * G ** 3}
        if B <= args.dense_max_batch:
            row['dense_grid_grid_sample_ms'] = round(_time(dense, max(1, args.iters // 2), 1), 3)
            row['speedup_vs_dense'] = round(row['dense_grid_grid_sample_ms'] / row['fused_newloss_ms'], 2)
        with torch.no_grad():
            row['mean_loss'] = round(float(crit(v.detach()).mean()), 5)
        res['B%d' % B] = row
    print(json.dumps(res))


if __name__ == '__main__':
    main()
