"""Throughput of the pose data pipeline's post-optimisation filters on the GPU: hand_collision_count (csrc/collision.cu) in frames/s at
B = 1024 and 6144 for hands apart, touching, deeply interpenetrating and coincident (the broad phase's worst case), with the mean box
tests and exact triangle tests per frame; ValidJudger.ComputeValidation's kernel at B = 6144; and, for context, the numpy oracle per
frame on 64 touching frames.  The reference itself (trimesh + python-fcl, one frame at a time) cannot be timed: neither library is
available.  The hands are the closed ellipsoid meshes of oracle/collision_ref.two_hand_frames (770 vertices, 1536 faces each, float32
vertices plus float64 translations, as the filter feeds them).  Prints the device and its power limit, a table and one JSON line.

    python tests/baselines/bench_collision.py [--iters 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import collision_ref as C  # noqa: E402
from renderih_b200 import assets  # noqa: E402
from renderih_b200.collision import hand_collision_count  # noqa: E402
from renderih_b200.valid_judge import ValidJudger  # noqa: E402


def timed(fn, iters):
    for _ in range(3):
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
    ap.add_argument('--iters', type=int, default=20)
    a = ap.parse_args()
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], stdout=subprocess.PIPE,
                       text=True).stdout.strip().splitlines()[0]
    print('device: %s (name, power limit, max SM clock)' % q)
    res = {'device': q, 'collision': {}}
    print('%-11s %6s %12s %12s %14s %14s' % ('regime', 'B', 'ms', 'frames/s', 'box tests', 'exact tests'))
    for B in (1024, 6144):
        for regime in ('apart', 'touching', 'deep', 'coincident'):
            va, vb, ta, tb, faces = C.two_hand_frames(B, regime, seed=B)
            d = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
            args = [d(va), d(vb), d(faces), d(ta), d(tb)]
            stats = torch.empty(B, 2, dtype=torch.int64, device='cuda')
            hand_collision_count(*args, stats=stats)
            s = stats.double().mean(0).tolist()
            ms = timed(lambda: hand_collision_count(*args), a.iters)
            print('%-11s %6d %12.3f %12.0f %14.0f %14.0f' % (regime, B, ms, B / ms * 1e3, s[0], s[1]))
            res['collision']['%s_%d' % (regime, B)] = {'ms': ms, 'frames_per_s': B / ms * 1e3, 'box_tests': s[0], 'exact_tests': s[1]}
    judger = ValidJudger({s: assets.synthetic_mano(0, s) for s in ('right', 'left')}, device='cuda')
    g = torch.Generator().manual_seed(0)
    ql, qr = (torch.randn(6144, 16, 4, generator=g).cuda() for _ in range(2))
    ms = timed(lambda: judger.scores(ql, qr), a.iters * 5)
    print('ValidJudger B=6144: %.4f ms (%.0f frames/s)' % (ms, 6144 / ms * 1e3))
    res['valid_judge_6144'] = {'ms': ms, 'frames_per_s': 6144 / ms * 1e3}
    va, vb, ta, tb, faces = C.two_hand_frames(64, 'touching', seed=64)
    t = time.perf_counter()
    C.counts(va.astype(np.float64) + ta[:, None], vb.astype(np.float64) + tb[:, None], faces)
    per = (time.perf_counter() - t) / 64 * 1e3
    print('numpy oracle, touching: %.1f ms per frame (host CPU)' % per)
    res['numpy_oracle_touching_ms_per_frame'] = per
    print(json.dumps(res))


if __name__ == '__main__':
    main()
