"""bench.py with the register-A bit mask of the wgmma GEMM (rih_set_gemm_rs) set before the run, so that kernel choices can be compared
A/B in one build: `--gemm-rs 1` selects the kernels in use before the transposed input gradients (bit 1) existed, 3 is the default.

    python tools/bench_gemm_rs.py --gemm-rs 1 --gpus 1 --steps 20 --warmup 5 [any other bench.py argument]
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    argv = sys.argv[1:]
    rs = 3
    if '--gemm-rs' in argv:
        i = argv.index('--gemm-rs')
        rs = int(argv[i + 1])
        del argv[i:i + 2]
    sys.argv = [os.path.join(ROOT, 'bench.py')] + argv
    import bench
    from renderih_b200 import _lib
    _lib.load()
    _lib.call('rih_set_gemm_rs', rs)
    a = bench.parse()
    if a.config == 'forward':
        bench.run_forward(a)
    elif a.config == 'train' and a.impl == 'ours':
        bench.run_ours(a)
    else:
        raise SystemExit('bench_gemm_rs.py: only --impl ours with --config train or forward')


if __name__ == '__main__':
    main()
