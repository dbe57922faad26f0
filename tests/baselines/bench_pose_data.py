"""Throughput of the pose data pipeline's augmentation on the GPU against the host: HandPoseArguer.argue_pose (csrc/pose_data.cu) at
--frames frames x argue_size 15 in augmented poses/s, with numpy's global-stream draws staged from the host (the reference's stream) and
with the device's Philox draws; the numpy / scipy statement of argue_pose (oracle/pose_data_ref.py, the reference's own vectorised scipy
calls) on --host-frames frames, reported per pose; and one full birth_data sweep (10 random levels x both hands, euler -> quaternion ->
axis-angle, written to a temporary directory) on the device path.  Each timing is a host clock around work that ends in a device
synchronise.  Prints the device and its power limit, a table and one JSON line.

    python tests/baselines/bench_pose_data.py [--frames 36000] [--host-frames 2000] [--birth-frames 3600] [--iters 5]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import pose_data_ref  # noqa: E402
from renderih_b200 import assets, pose_data  # noqa: E402

A = 15
MANO = {s: assets.synthetic_mano(0, s) for s in ('right', 'left')}


def clock(fn, iters):
    fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=36000)
    ap.add_argument('--host-frames', type=int, default=2000)
    ap.add_argument('--birth-frames', type=int, default=3600)
    ap.add_argument('--iters', type=int, default=5)
    a = ap.parse_args()
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], stdout=subprocess.PIPE,
                       text=True).stdout.strip().splitlines()[0]
    print('device: %s (name, power limit, max SM clock)' % q)
    rng = np.random.default_rng(0)
    euler = rng.uniform(-60, 90, size=(a.frames, 16, 3))
    arg = pose_data.HandPoseArguer(side='right', root=MANO)
    e_dev = torch.from_numpy(euler).cuda()
    poses = a.frames * A
    np.random.seed(0)
    t_np = clock(lambda: arg.argue_pose(euler, A, 'euler'), a.iters)                    # numpy in, numpy out, host draws
    t_dev = clock(lambda: arg.argue_pose(e_dev, A, 'euler', generator=1), a.iters)       # device in, device out, Philox
    he = euler[:a.host_frames]
    u = pose_data_ref.draw_uniforms(a.host_frames, A)
    t = time.perf_counter()
    pose_data_ref.argue_pose(he, u, 'HandPoseArguer')
    t_host = (time.perf_counter() - t) / (a.host_frames * A)
    data = {s: {'rot': euler[:a.birth_frames]} for s in ('right', 'left')}
    data['capture_frame_id'] = np.arange(a.birth_frames)
    with tempfile.TemporaryDirectory() as tmp:
        pose_data.birth_data(data, argue_size=A, out_dir=tmp, root=MANO, generator=3)    # warm-up
        t_birth = clock(lambda: pose_data.birth_data(data, argue_size=A, out_dir=tmp, root=MANO, generator=3), 1)
    birth_rows = a.birth_frames * A * 10 * 2 + 2 * a.birth_frames
    res = {'device': q, 'frames': a.frames, 'argue_size': A,
           'gpu_numpy_draws_poses_per_s': poses / t_np, 'gpu_philox_poses_per_s': poses / t_dev,
           'host_oracle_poses_per_s': 1.0 / t_host, 'host_frames': a.host_frames,
           'birth_frames': a.birth_frames, 'birth_rows': birth_rows, 'birth_data_s': t_birth}
    print('%-40s %14s' % ('path', 'poses/s'))
    print('%-40s %14.0f' % ('GPU, numpy draws (numpy in / out)', res['gpu_numpy_draws_poses_per_s']))
    print('%-40s %14.0f' % ('GPU, device Philox (CUDA in / out)', res['gpu_philox_poses_per_s']))
    print('%-40s %14.0f' % ('host numpy / scipy (%d frames)' % a.host_frames, res['host_oracle_poses_per_s']))
    print('birth_data, %d frames: %d rows in %.3f s' % (a.birth_frames, birth_rows, t_birth))
    print(json.dumps(res))


if __name__ == '__main__':
    main()
