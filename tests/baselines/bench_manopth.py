"""Timing of the pose optimiser's quaternion hand model (renderih_b200/manopth.py) for both hands, as the optimiser runs it once per
iteration: the forward, and the forward + backward of a weighted sum of verts, joints and transf, CUDA events around --iters calls after
--warmup calls.  The baseline is our own float64 oracle restatement (oracle/manopth_ref.py) run as float32 torch eager on the same GPU; the
reference layer itself is not timed.  Synthetic MANO tensors; center_idx 0, per-hand betas, non-zero translation.  Prints the device
name and power limit read in the same run, a table, and one JSON line.
It lives with the other eager baselines because it runs the oracle; the product and tools/ never import it.
usage: python tests/baselines/bench_manopth.py [--batches 64,1024,8192] [--iters 20] [--warmup 3]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batches', default='64,1024,8192')
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_manopth: a CUDA device is required')
    from oracle import manopth_ref as M
    from renderih_b200 import assets as A
    from renderih_b200.manopth import ManoLayer
    dev = torch.device('cuda')
    sides = ('right', 'left')
    layers = {s: ManoLayer(center_idx=0, side=s, mano_root=A.synthetic_mano(0, s), use_pca=False, root_rot_mode='quat', joint_rot_mode='quat',
                           return_transf=True).to(dev) for s in sides}
    tabs = {s: {k: v.float().to(dev) for k, v in M.tables(A.synthetic_mano(0, s), s).items()} for s in sides}
    rows = []
    for B in [int(b) for b in args.batches.split(',')]:
        g = torch.Generator().manual_seed(B)
        inp = {}
        for s in sides:
            q = torch.randn(B, 16, 4, generator=g) * 0.3 + torch.tensor([1.0, 0, 0, 0])
            inp[s] = [t.to(dev).requires_grad_(True) for t in (q.reshape(B, 64), torch.randn(B, 10, generator=g), torch.randn(B, 3, generator=g) * 0.1)]
        w = [torch.randn(B, 778, 3, generator=g).to(dev), torch.randn(B, 21, 3, generator=g).to(dev), torch.randn(B, 16, 4, 4, generator=g).to(dev)]

        def ours(backward):
            for s in sides:
                out = layers[s](*inp[s])
                if backward:
                    sum((o * wi).sum() for o, wi in zip(out, w)).backward()

        def eager(backward):
            for s in sides:
                out = M.forward(tabs[s], s, inp[s][0], inp[s][1], inp[s][2], center_idx=0)
                if backward:
                    sum((o * wi).sum() for o, wi in zip(out, w)).backward()
        row = {'batch': B}
        for name, fn in (('fused', ours), ('eager_fp32', eager)):
            with torch.no_grad():
                row[name + '_fwd_ms'] = round(_time(lambda: fn(False), args.iters, args.warmup), 4)
            row[name + '_fwd_bwd_ms'] = round(_time(lambda: fn(True), args.iters, args.warmup), 4)
        rows.append(row)
    info = {'device': torch.cuda.get_device_name(), 'power_limit': _power_limit(), 'hands': 2, 'iters': args.iters, 'warmup': args.warmup,
            'baseline': 'oracle/manopth_ref.py as float32 torch eager on the same GPU (ours, not the reference layer)'}
    print('device: %s, power limit: %s' % (info['device'], info['power_limit']))
    print('| batch | fused fwd | eager fwd | fused fwd+bwd | eager fwd+bwd |')
    print('|---|---|---|---|---|')
    for r in rows:
        print('| %d | %.3f ms | %.3f ms | %.3f ms | %.3f ms |' % (r['batch'], r['fused_fwd_ms'], r['eager_fp32_fwd_ms'], r['fused_fwd_bwd_ms'],
                                                              r['eager_fp32_fwd_bwd_ms']))
    print(json.dumps(dict(info, rows=rows)))


if __name__ == '__main__':
    main()
