"""Timing of the pose optimiser's discriminator nature loss (renderih_b200/nature.py) on both hands, CUDA events around --iters calls
after --warmup calls: forward, and forward + backward, of NatureLoss against our float64 restatement (oracle/nature_ref.py) run as
float32 torch eager on the same GPU (the reference itself is not timed).  Weights: torch.nn.Linear's default initialisation with
layer_pred scaled by 40 and its bias set so that about half of the rows are masked; normalised random poses.  Prints the device name and
power limit read in the same run, the MLP's achieved rate from shape-derived multiply-add counts against the data sheet's 67 TFLOP/s
fp32, one table and one JSON line.  It lives with the other eager baselines because it runs the oracle; the product and tools/ never
import it.
usage: python tests/baselines/bench_nature.py [--batches 64,1024,8192] [--iters 20] [--warmup 3]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_manopth import _power_limit, _time  # noqa: E402

# multiply-adds per row: the forward MLP (45x512 + 4 x 512x512 + 512x2), and the same again for the input gradient
MACS_PER_ROW = 45 * 512 + 4 * 512 * 512 + 512 * 2
FP32_PEAK_TFLOPS = 67.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batches', default='64,1024,8192')
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_nature: a CUDA device is required')
    from oracle import make_golden_nature as golden
    from oracle import nature_ref as R
    from renderih_b200.nature import NatureLoss, Pos2dDiscriminator
    dev = torch.device('cuda')
    rows = []
    for B in [int(b) for b in args.batches.split(',')]:
        sd = R.init_state_dict(*golden.weights(('bench', min(B, 1024), B, 7, 40.0, 'median')))
        disc = Pos2dDiscriminator().to(dev).eval()
        disc.load_state_dict(sd)
        nature = NatureLoss(disc)
        sd32 = {k: v.to(dev) for k, v in sd.items()}
        right, left = (p.to(dev).requires_grad_(True) for p in golden.poses(B, B))

        def fused_fwd():
            with torch.no_grad():
                nature(right[:, 1:], left[:, 1:])

        def fused():
            nature(right[:, 1:], left[:, 1:]).backward()

        def eager_fwd():          # the oracle decides the empty masks on the host, as the reference does
            with torch.no_grad():
                R.nature_loss(sd32, right[:, 1:], left[:, 1:])

        def eager():
            loss, _ = R.nature_loss(sd32, right[:, 1:], left[:, 1:])
            loss.backward()
        t = {'fused_fwd_ms': _time(fused_fwd, args.iters, args.warmup), 'fused_fwd_bwd_ms': _time(fused, args.iters, args.warmup),
             'eager_fp32_fwd_ms': _time(eager_fwd, args.iters, args.warmup), 'eager_fp32_fwd_bwd_ms': _time(eager, args.iters, args.warmup)}
        macs = 2 * B * MACS_PER_ROW
        r = {'batch': B, **{k: round(v, 4) for k, v in t.items()},
             'fused_fwd_tflops': round(2 * macs / (t['fused_fwd_ms'] * 1e-3) / 1e12, 2),
             'fused_fwd_bwd_tflops': round(2 * 2 * macs / (t['fused_fwd_bwd_ms'] * 1e-3) / 1e12, 2)}
        rows.append(r)
    info = {'device': torch.cuda.get_device_name(), 'power_limit': _power_limit(), 'hands': 2, 'macs_per_row': MACS_PER_ROW,
            'fp32_peak_tflops_datasheet': FP32_PEAK_TFLOPS, 'iters': args.iters, 'warmup': args.warmup,
            'baseline': 'oracle/nature_ref.py as float32 torch eager on the same GPU (ours, not the reference)'}
    print('device: %s, power limit: %s' % (info['device'], info['power_limit']))
    print('| batch | fused fwd | eager fp32 fwd | fused fwd+bwd | eager fp32 fwd+bwd | MLP rate fwd / fwd+bwd (of 67 TFLOP/s) |')
    print('|---|---|---|---|---|---|')
    for r in rows:
        print('| %d | %.3f ms | %.3f ms | %.3f ms | %.3f ms | %.1f / %.1f TFLOP/s |' % (
            r['batch'], r['fused_fwd_ms'], r['eager_fp32_fwd_ms'], r['fused_fwd_bwd_ms'], r['eager_fp32_fwd_bwd_ms'], r['fused_fwd_tflops'],
            r['fused_fwd_bwd_tflops']))
    print(json.dumps(dict(info, rows=rows)))


if __name__ == '__main__':
    main()
