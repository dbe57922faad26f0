"""Per-shape timing of the input-gradient GEMMs with and without the transposed-output form (rih_set_gemm_rs bit 1).

Every convolution input gradient of the ResNet-50 training step (batch 64, 256 x 256 images) and of HRNet-w48 (batch 32), in the step's
convolution arithmetic (tf32c), and the token decoder's Linear input gradients (tf32x3), each timed with CUDA events over `--iters` launches
after a warm-up, once with rih_set_gemm_rs(1) (the untransposed product: the weights are transposed in shared memory) and once with
rih_set_gemm_rs(3).  Column T tells whether the rih_set_gemm_rs(3) launch ran the transposed form (counted by the library,
rih_gemm_dgrad_t_launches); where it did not (fewer than 128 input channels / in-features: the transposed tile would leave rows empty),
both columns time the same kernel.  Prints one table row per shape with the achieved TFLOP/s (2 * M * N * K of the GEMM over the kernel
time) and, with --json, the rows as JSON.

    python tools/bench_dgrad.py [--iters 50] [--json out.json]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# (N, H, Cin, Cout, k, stride): input H x H, k x k filter, pad k // 2
RESNET50 = [(64, 64, 64, 64, 1, 1), (64, 64, 64, 64, 3, 1), (64, 64, 64, 256, 1, 1), (64, 64, 256, 64, 1, 1),
            (64, 64, 256, 128, 1, 1), (64, 64, 128, 128, 3, 2), (64, 32, 128, 512, 1, 1), (64, 64, 256, 512, 1, 2), (64, 32, 512, 128, 1, 1),
            (64, 32, 128, 128, 3, 1),
            (64, 32, 512, 256, 1, 1), (64, 32, 256, 256, 3, 2), (64, 16, 256, 1024, 1, 1), (64, 32, 512, 1024, 1, 2), (64, 16, 1024, 256, 1, 1),
            (64, 16, 256, 256, 3, 1),
            (64, 16, 1024, 512, 1, 1), (64, 16, 512, 512, 3, 2), (64, 8, 512, 2048, 1, 1), (64, 16, 1024, 2048, 1, 2), (64, 8, 2048, 512, 1, 1),
            (64, 8, 512, 512, 3, 1)]
HRNET48 = [(32, 128, 64, 64, 3, 2), (32, 64, 64, 64, 3, 1), (32, 64, 64, 256, 1, 1), (32, 64, 256, 64, 1, 1), (32, 64, 256, 48, 3, 1),
           (32, 64, 256, 96, 3, 2), (32, 64, 48, 48, 3, 1), (32, 32, 96, 96, 3, 1), (32, 16, 192, 192, 3, 1), (32, 8, 384, 384, 3, 1),
           (32, 32, 96, 192, 3, 2), (32, 16, 192, 384, 3, 2), (32, 64, 48, 96, 3, 2), (32, 32, 96, 48, 1, 1), (32, 16, 192, 48, 1, 1),
           (32, 8, 384, 48, 1, 1), (32, 16, 192, 96, 1, 1), (32, 8, 384, 96, 1, 1), (32, 8, 384, 192, 1, 1)]
# (M, N, K): dx[M, K] = dy[M, N] . w[N, K] -- the decoder's Linear input gradients
LINEAR = [(M, N, K) for M in (4032, 8064, 16128, 20224) for N, K in ((256, 256), (1024, 256), (256, 1024), (768, 256), (256, 64), (64, 256),
                                                                        (512, 512), (128, 128))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--json', default=None, help='also write the rows as JSON to this path')
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), 'bench_dgrad.py times kernels on the GPU'
    from renderih_b200 import ops
    from renderih_b200._lib import call, load
    load()
    p = ctypes.c_void_p

    def timed(fn, rs):
        call('rih_set_gemm_rs', rs)
        for _ in range(5):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.iters

    rows = []

    def dispatched_t(fn):
        n = ctypes.c_longlong(0)
        call('rih_gemm_dgrad_t_launches', ctypes.byref(n), 1)
        call('rih_set_gemm_rs', 3)
        fn()
        torch.cuda.synchronize()
        call('rih_gemm_dgrad_t_launches', ctypes.byref(n), 1)
        return n.value > 0

    def measure(kind, shape, flops, fn):
        transposed = dispatched_t(fn)
        old, new = timed(fn, 1), timed(fn, 3)
        r = {'kind': kind, 'shape': shape, 'transposed': transposed, 'old_ms': old, 'new_ms': new,
             'old_tflops': flops / old / 1e9, 'new_tflops': flops / new / 1e9, 'speedup': old / new}
        rows.append(r)
        print('%-14s %-28s %-3s %8.4f %8.4f %7.1f %7.1f %6.3f' % (kind, shape, 'T' if transposed else '-', old, new, r['old_tflops'],
                                                               r['new_tflops'], r['speedup']), flush=True)

    try:
        smi = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, timeout=30).stdout.decode().strip()
    except (OSError, subprocess.SubprocessError):
        smi = 'power limit / clocks not available'
    print('GPU: %s, %s (power limit, max SM clock)' % (torch.cuda.get_device_name(0), smi))
    print('%-14s %-28s %-3s %8s %8s %7s %7s %6s' % ('entry', 'shape', 'T', 'old ms', 'new ms', 'TF/s', 'TF/s', 'x'))
    ops.set_gemm_mode('tf32c', 'tf32x3')
    try:
        for net, geoms in (('resnet50', RESNET50), ('hrnet48', HRNET48)):
            for (N, H, Cin, Cout, k, s) in geoms:
                Ho = (H + 2 * (k // 2) - k) // s + 1
                dy = torch.randn(N * Ho * Ho, Cout, device='cuda')
                w = torch.randn(Cout, k * k * Cin, device='cuda')
                dx = torch.empty(N * H * H, Cin, device='cuda')
                geom = (ctypes.c_int * 13)(N, H, H, Cin, Ho, Ho, Cout, k, k, s, k // 2, Cin, Cout)
                # multiply-adds the kernels perform: stride 2 runs four parity classes over a quarter of the taps each
                flops = 2.0 * N * Ho * Ho * Cout * k * k * Cin

                def fn(dy=dy, w=w, dx=dx, geom=geom):
                    call('rih_conv2d_dgrad', p(dy.data_ptr()), p(w.data_ptr()), p(dx.data_ptr()), geom, 0, None, None)
                measure('conv_dgrad', '%s %s' % (net, (N, H, Cin, Cout, k, s)), flops, fn)
        for (M, N, K) in LINEAR:
            dy = torch.randn(M, N, device='cuda')
            w = torch.randn(N, K, device='cuda')
            dx = torch.empty(M, K, device='cuda')

            def fn(dy=dy, w=w, dx=dx, M=M, N=N, K=K):
                call('rih_linear_dgrad', p(dy.data_ptr()), N, p(w.data_ptr()), K, p(dx.data_ptr()), K, M, N, K, 0, 0, None)
            measure('linear_dgrad', str((M, N, K)), 2.0 * M * N * K, fn)
    finally:
        call('rih_set_gemm_rs', 3)
        ops.set_gemm_mode('simt', 'simt')
    for kind in ('conv_dgrad', 'linear_dgrad'):
        for t in (True, False):
            sel = [r for r in rows if r['kind'] == kind and r['transposed'] == t]
            if sel:
                o, n = sum(r['old_ms'] for r in sel), sum(r['new_ms'] for r in sel)
                print('%s %s: %d shapes, sum old %.3f ms, sum new %.3f ms (x%.3f)' % (kind, 'transposed' if t else 'untransposed', len(sel), o, n, o / n))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
