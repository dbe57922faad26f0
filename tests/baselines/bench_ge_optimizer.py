"""Timing of the two-hand pose optimiser (renderih_b200/ge_optimizer.py): GeOptimizer.optimize() -- one CUDA graph per iteration,
device-side Adam and ReduceLROnPlateau, one synchronisation per call -- against the eager driver oracle/ge_optimizer_ref.eager_optimize
built from the same CUDA loss modules with torch.optim.Adam and ReduceLROnPlateau, synchronising with the host where the reference does
(the 11 .item() of loss_fn's dict, the print's four tensors, float(loss) in scheduler.step).  Wall time around whole calls after one warm-up
call each, reported in ms per iteration.  Synthetic MANO tensors, the reference's anchor tables, a convex-hull mesh for the penetration
term.  Prints the device name and power limit read in the same run, one table and one JSON line.
usage: python tests/baselines/bench_ge_optimizer.py [--batches 64,1024,6144] [--iters 50] [--repeats 3]"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_manopth import _power_limit  # noqa: E402


def _wall(fn, repeats):
    fn()
    torch.cuda.synchronize()
    best = float('inf')
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t0)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batches', default='64,1024,6144')
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--repeats', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_ge_optimizer: a CUDA device is required')
    from oracle import ge_optimizer_ref as G
    dev = torch.cuda.current_device()
    rows = []
    for B in [int(b) for b in args.batches.split(',')]:
        opt = G.build(G.nature_weights(min(B, 1024), 5, 1005), n_iter=args.iters)
        kw = G.inputs(B, 5, device='cuda')

        def ours():
            opt.set_opt_val(**kw)
            opt.optimize()

        def eager():
            G.eager_optimize(opt, kw, args.iters, sync=True)
        opt.set_opt_val(**kw)
        t_ours, t_eager = _wall(ours, args.repeats), _wall(eager, args.repeats)
        rows.append({'batch': B, 'iters': args.iters, 'ours_ms_per_iter': 1e3 * t_ours / args.iters,
                     'eager_ms_per_iter': 1e3 * t_eager / args.iters, 'speedup': t_eager / t_ours})
    name = torch.cuda.get_device_name(dev)
    print('device: %s, power limit %s' % (name, _power_limit()))
    print('%6s %6s %12s %12s %8s' % ('B', 'iters', 'ours ms/it', 'eager ms/it', 'speedup'))
    for r in rows:
        print('%6d %6d %12.3f %12.3f %7.2fx' % (r['batch'], r['iters'], r['ours_ms_per_iter'], r['eager_ms_per_iter'], r['speedup']))
    print(json.dumps({'bench': 'ge_optimizer', 'device': name, 'power_limit': _power_limit(), 'rows': rows}))


if __name__ == '__main__':
    main()
