"""Micro-benchmark of the wgmma GEMM / conv kernels on the hot shapes (CUDA events, L2 flushed between reps).
usage: python tools/bench_gemm.py"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from renderih_b200 import ops  # noqa: E402
from renderih_b200._lib import call  # noqa: E402


def timeit(fn, reps=10):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    tot = 0.0
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    return tot / reps


def main():
    s = torch.cuda.current_stream().cuda_stream
    print('%-34s %6s %10s %10s %10s' % ('gemm M x N x K', 'mode', 'ms', 'TFLOP/s', 'GB/s'))
    for (M, N, K) in [(262144, 256, 64), (262144, 64, 256), (65536, 512, 128), (65536, 128, 512), (16384, 1024, 256), (4096, 2048, 512),
                      (16128, 64, 128), (8064, 128, 256), (4032, 256, 512), (20224, 64, 64)]:
        a = torch.randn(M, K, device='cuda'); b = torch.randn(N, K, device='cuda'); c = torch.empty(M, N, device='cuda')
        for nsplit in (1, 3):
            ms = timeit(lambda: call('rih_gemm_tf32', a.data_ptr(), K, 0, b.data_ptr(), K, 0, c.data_ptr(), N, M, N, K, None, 0, 0, 0, nsplit, s))
            print('%-34s %6d %10.4f %10.1f %10.0f' % ('%d x %d x %d' % (M, N, K), nsplit, ms, 2.0 * M * N * K / ms / 1e9, 4.0 * (M * K + N * K + M * N) / ms / 1e6))
    print('conv3x3 fwd / dgrad / wgrad (batch 64):')
    for (H, C) in [(64, 128), (32, 128), (16, 256), (8, 512), (64, 64)]:
        N = 64
        x = torch.randn(N * H * H, C, device='cuda', requires_grad=True)
        w = (torch.randn(C, C, 3, 3, device='cuda') * 0.03).contiguous(memory_format=torch.channels_last).requires_grad_(True)
        fl = 2.0 * N * H * H * C * 9 * C
        for mode in ('tf32', 'tf32x3'):
            ops.set_gemm_mode(mode, mode)
            ms = timeit(lambda: ops.conv2d(x.detach(), w.detach(), None, N, H, H, stride=1, pad=1))
            y = ops.conv2d(x, w, None, N, H, H, stride=1, pad=1)
            g = torch.randn_like(y)
            msb = timeit(lambda: torch.autograd.grad(y, [x, w], g, retain_graph=True))
            print('  %dx%d C=%d %-7s fwd %.3f ms (%.0f TFLOP/s)   dgrad+wgrad %.3f ms (%.0f TFLOP/s)' % (H, H, C, mode, ms, fl / ms / 1e9, msb, 2 * fl / msb / 1e9))
    ops.set_gemm_mode('simt', 'simt')


if __name__ == '__main__':
    main()
