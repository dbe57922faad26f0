"""Timing of the pose optimiser's prior and contact terms (renderih_b200/geo_loss.py) for both hands, CUDA events around --iters calls
after --warmup calls:
  1. the fused forward + backward of HandPriorLoss against our float64 oracle restatement (oracle/geo_loss_ref.py) run as float32 torch
     eager on the same GPU (the reference functions themselves are not timed);
  2. one full differentiable optimiser iteration -- both manopth hands, the translation adds, HandPriorLoss, NewLoss and the backward --
     run eagerly against the replay of the same iteration captured in one CUDA graph.
Synthetic MANO tensors, random anchor tables, D = 4 contacts per anchor.  Prints the device name and power limit read in the same run,
two tables, and one JSON line.  It lives with the other eager baselines because it runs the oracle; the product and tools/ never import it.
usage: python tests/baselines/bench_geo_loss.py [--batches 64,1024,8192] [--iter-batches 64,1024] [--iters 20] [--warmup 3]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_manopth import _power_limit, _time  # noqa: E402


def _inputs(B, dev, seed):
    from renderih_b200 import assets as A
    g = torch.Generator().manual_seed(seed)
    out = {}
    for s in ('right', 'left'):
        out['quat_' + s[0]] = (torch.randn(B, 16, 4, generator=g) * 0.4 + torch.tensor([1.0, 0, 0, 0])).to(dev)
        vt = torch.from_numpy(A.synthetic_mano(0, s)['v_template'])
        out['verts_' + s[0]] = (vt[None] + 0.003 * torch.randn(B, 778, 3, generator=g)).to(dev)
    out['anchor_id'] = torch.randint(0, 108, (B, 108, 4), generator=g).to(dev)
    out['elastic'] = torch.rand(B, 108, 4, generator=g).to(dev)
    out['mask'] = (torch.rand(B, 108, 4, generator=g) < 0.3).long().to(dev)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batches', default='64,1024,8192')
    ap.add_argument('--iter-batches', default='64,1024')
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_geo_loss: a CUDA device is required')
    from scipy.spatial import ConvexHull
    from oracle import geo_loss_ref as R
    from renderih_b200 import assets as A
    from renderih_b200.geo_loss import HandPriorLoss
    from renderih_b200.manopth import ManoLayer
    from renderih_b200.sdf import NewLoss
    dev = torch.device('cuda')
    rng = np.random.default_rng(0)
    fvi, aw = rng.integers(0, 778, size=(108, 3)), rng.uniform(0.0, 0.5, size=(108, 2))
    layers = {s: ManoLayer(center_idx=0, side=s, mano_root=A.synthetic_mano(0, s), use_pca=False, root_rot_mode='quat', joint_rot_mode='quat',
                           return_transf=True, return_full_pose=True).to(dev) for s in ('right', 'left')}
    prior = HandPriorLoss(layers['right'], layers['left'], face_vert_idx=fvi, anchor_weight=aw)
    tab = R.tables(A.synthetic_mano(0, 'right'), A.synthetic_mano(0, 'left'), fvi, aw)
    tab32 = {'edges': tab['edges'].to(dev), 'fvi': tab['fvi'].to(dev), 'aw': tab['aw'].float().to(dev),
             'rest': {s: v.float().to(dev) for s, v in tab['rest'].items()},
             'conv': {s: tuple(m.float().to(dev) for m in v) for s, v in tab['conv'].items()}}
    keys = ('quat_r', 'quat_l', 'verts_r', 'verts_l')
    rows = []
    for B in [int(b) for b in args.batches.split(',')]:
        inp = _inputs(B, dev, B)
        leaves = [inp[k].clone().requires_grad_(True) for k in keys]
        prior.set_contacts(inp['anchor_id'], inp['elastic'], inp['mask'])

        def fused():
            sum(w * t for w, t in zip(R.WEIGHTS, prior(*leaves))).backward()

        def eager():       # the oracle's contact branch decides on the host, as the reference does
            t, _ = R.terms(tab32, *leaves, inp['anchor_id'], inp['elastic'], inp['mask'])
            sum(w * x for w, x in zip(R.WEIGHTS, t)).backward()
        rows.append({'batch': B, 'fused_fwd_bwd_ms': round(_time(fused, args.iters, args.warmup), 4),
                     'eager_fp32_fwd_bwd_ms': round(_time(eager, args.iters, args.warmup), 4)})
    pts = rng.normal(size=(778, 3))
    pts *= np.array([1.0, 0.6, 0.35]) / np.linalg.norm(pts, axis=1, keepdims=True)
    newloss = NewLoss(faces=ConvexHull(pts).simplices, part_vert=[np.arange(k, 778, 16) for k in range(16)])
    it_rows = []
    for B in [int(b) for b in args.iter_batches.split(',')]:
        inp = _inputs(B, dev, B + 1)
        q = {s: inp['quat_' + s[0]].clone().requires_grad_(True) for s in ('right', 'left')}
        shape = torch.zeros(B, 20, device=dev, requires_grad=True)
        tsl = {s: torch.full((B, 3), 0.02 if s == 'right' else -0.02, device=dev).requires_grad_(True) for s in ('right', 'left')}
        prior.set_contacts(inp['anchor_id'], inp['elastic'], inp['mask'])
        leaves = [q['right'], q['left'], shape, tsl['right'], tsl['left']]

        def iteration():
            vr = layers['right'](q['right'], shape[:, :10])[0] + tsl['right'].unsqueeze(1)
            vl = layers['left'](q['left'], shape[:, 10:])[0] + tsl['left'].unsqueeze(1)
            qn, edge, contact, ergo = prior(q['right'], q['left'], vr, vl)
            pen = newloss(torch.cat((vr.unsqueeze(1), vl.unsqueeze(1)), 1)).mean()
            return torch.autograd.grad(qn + edge + 10.0 * contact + 0.02 * 0.5 * pen + ergo, leaves)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                iteration()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            iteration()
        it_rows.append({'batch': B, 'eager_ms': round(_time(iteration, args.iters, args.warmup), 4),
                        'graph_replay_ms': round(_time(graph.replay, args.iters, args.warmup), 4)})
    info = {'device': torch.cuda.get_device_name(), 'power_limit': _power_limit(), 'hands': 2, 'contacts_per_anchor': 4, 'iters': args.iters,
            'warmup': args.warmup, 'baseline': 'oracle/geo_loss_ref.py as float32 torch eager on the same GPU (ours, not the reference functions)'}
    print('device: %s, power limit: %s' % (info['device'], info['power_limit']))
    print('| batch | fused fwd+bwd | eager fp32 fwd+bwd |')
    print('|---|---|---|')
    for r in rows:
        print('| %d | %.3f ms | %.3f ms |' % (r['batch'], r['fused_fwd_bwd_ms'], r['eager_fp32_fwd_bwd_ms']))
    print('| batch | full iteration, eager | full iteration, graph replay |')
    print('|---|---|---|')
    for r in it_rows:
        print('| %d | %.3f ms | %.3f ms |' % (r['batch'], r['eager_ms'], r['graph_replay_ms']))
    print(json.dumps(dict(info, prior=rows, iteration=it_rows)))


if __name__ == '__main__':
    main()
