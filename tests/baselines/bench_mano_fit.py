"""Timing of fitting MANO to 3-D joints (renderih_b200/mano_from_3djoint.py): JointFitter.fit -- the IK kernel, then 200 iterations
replayed from one CUDA graph per hand, both hands -- against the reference's structure run eagerly on the same GPU: one 200-iteration
torch.optim.Adam loop per frame and hand (convert2mano.py:158-200) over the same CUDA ManoLayer and mat2aa.  CUDA events around whole
calls after a warm-up call; the eager loop is timed on --eager-frames frames and reported per frame.  Synthetic MANO and joints.  Prints
the device name and power limit read in the same run, one table and one JSON line.
usage: python tests/baselines/bench_mano_fit.py [--batches 1,1024,8192] [--eager-frames 4]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import mano_fit_ref as M  # noqa: E402
from renderih_b200 import assets, mano_from_3djoint as MF  # noqa: E402


def _events(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batches', default='1,1024,8192')
    ap.add_argument('--eager-frames', type=int, default=4)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_mano_fit: no CUDA device')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], stdout=subprocess.PIPE,
                       universal_newlines=True).stdout.strip().splitlines()[0]
    print('device: %s (name, power limit, max SM clock)' % q)
    fitter = MF.JointFitter({s: assets.synthetic_mano(0, s) for s in MF.SIDES}, 'cuda')
    g = torch.Generator().manual_seed(0)
    Bmax = max(int(b) for b in args.batches.split(','))
    J = {}
    for s in MF.SIDES:                      # the template in centimetres, moved by 40 cm, with 0.8 cm of noise per joint
        base = fitter.template[s].cpu() * 100
        J[s] = (base[None] + torch.randn(Bmax, 21, 3, generator=g, dtype=torch.float64) * 0.8 + 40).cuda()
    rows = []
    for B in (int(b) for b in args.batches.split(',')):
        run = lambda: fitter.fit(J['left'][:B], J['right'][:B])
        run()
        t = min(_events(run) for _ in range(3))
        rows.append({'B': B, 'graph_s': t, 'graph_frames_per_s': B / t})
    nE = args.eager_frames

    # every eager loop starts from frame 0's IK (pose64 of the B = 1 fit below); the start does not change the work per iteration
    eager_run = lambda: [M.eager_fit(fitter.mano_layer[s], fitter._sides[(s, 1, 200, 0.1)].pose64.float(), J[s][i:i + 1], MF.mat2aa)
                         for s in MF.SIDES for i in range(nE)]
    fitter.fit(J['left'][:1], J['right'][:1])
    eager_run()
    te = _events(eager_run) / nE
    for r in rows:
        r['eager_frames_per_s'] = 1.0 / te
        r['speedup'] = r['graph_frames_per_s'] / r['eager_frames_per_s']
    print('%8s %14s %16s %16s %9s' % ('frames', 'graph s', 'graph frames/s', 'eager frames/s', 'speedup'))
    for r in rows:
        print('%8d %14.4f %16.1f %16.2f %9.0f' % (r['B'], r['graph_s'], r['graph_frames_per_s'], r['eager_frames_per_s'], r['speedup']))
    print(json.dumps({'device': q, 'eager_s_per_frame_both_hands': te, 'rows': rows}))


if __name__ == '__main__':
    main()
