"""Per-shape timing of the attention core (forward / backward) at the 9 (Sq, Sk, d) shapes of the decoder (SURVEY 8 a2), batch 64 x 4 heads,
CUDA events, L2 flushed between launches.  Beside each time: the algorithmic HBM traffic of the fused tensor-core core (forward reads
q, k, v and writes o and 2 floats of row statistics per query row; backward reads q, k, v, o, dO and the statistics and writes dq, dk, dv)
and the rate that implies.  usage: python tools/bench_attn.py [--rows-fwd 0|4|8] [--rows-bwd 0|2|4] [--dropout 0.05]"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = [(63, 63, 64, 4), (64, 64, 64, 2), (63, 127, 64, 2), (126, 126, 32, 4), (64, 64, 32, 2), (126, 190, 32, 2),
          (252, 252, 16, 4), (64, 64, 16, 2), (252, 316, 16, 2)]     # (Sq, Sk, d, calls per forward)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rows-fwd', type=int, default=0)
    ap.add_argument('--rows-bwd', type=int, default=0)
    ap.add_argument('--dropout', type=float, default=0.05)
    ap.add_argument('--batch', type=int, default=64)
    ap.add_argument('--impl', default='simt', choices=['simt', 'tc'])
    ap.add_argument('--linear-mode', default='tf32x3')
    args = ap.parse_args()
    from renderih_b200 import ops
    from renderih_b200._lib import call
    call('rih_attn_set_row_blocks', args.rows_fwd, args.rows_bwd)
    ops.set_gemm_mode('simt', args.linear_mode)
    B, H = args.batch, 4
    flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
    tot_f = tot_b = 0.0
    print('impl=%s mode=%s rows_fwd=%d rows_bwd=%d dropout=%.2f' % (args.impl, args.linear_mode, args.rows_fwd, args.rows_bwd, args.dropout))
    for Sq, Sk, d, calls in SHAPES:
        q = torch.randn(B * Sq, H * d, device='cuda', requires_grad=True)
        k = torch.randn(B * Sk, H * d, device='cuda', requires_grad=True)
        v = torch.randn(B * Sk, H * d, device='cuda', requires_grad=True)
        go = torch.randn(B * Sq, H * d, device='cuda')
        tf = tb = 0.0
        reps = 5
        for it in range(reps + 2):
            flush.zero_()
            e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            e0.record()
            o = ops.attention(q, k, v, B, H, Sq, Sk, p_drop=args.dropout, impl=args.impl)
            e1.record()
            o.backward(go)
            e2.record()
            torch.cuda.synchronize()
            if it >= 2:
                tf += e0.elapsed_time(e1) / reps
                tb += e1.elapsed_time(e2) / reps
        fl = 4.0 * B * H * Sq * Sk * d
        by_f = 4.0 * B * H * (d * (2 * Sq + 2 * Sk) + 2 * Sq)
        by_b = 4.0 * B * H * (d * (4 * Sq + 4 * Sk) + 2 * Sq)
        print('Sq %3d Sk %3d d %2d x%d : fwd %7.1f us (%5.1f TF/s, %5.2f MB, %6.1f GB/s)   bwd %7.1f us (%5.1f TF/s, %5.2f MB, %6.1f GB/s)'
              % (Sq, Sk, d, calls, tf * 1e3, fl / tf / 1e9, by_f / 1e6, by_f / tf / 1e6, tb * 1e3, 2.5 * fl / tb / 1e9, by_b / 1e6, by_b / tb / 1e6))
        tot_f += tf * calls; tot_b += tb * calls
    print('per training step (24 cores): fwd %.3f ms  bwd %.3f ms' % (tot_f, tot_b))


if __name__ == '__main__':
    main()
