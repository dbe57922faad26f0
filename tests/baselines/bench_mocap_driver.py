"""Timing of the mocap driver (renderih_b200/mocap_optimize.py) on synthetic mocap sequences of N frames, one batch of N frames.

* scene: the six scene-preparation passes main runs per frame (two fresh anchor passes, four batch passes with previous ids), as
  Scene.update_scene over the batch (ours) and as the eager per-frame path of oracle/mocap_ref.py (two batch-1 CUDA ManoLayer forwards
  copied to the host, numpy geometry and search, per frame), the latter timed over --eager-frames frames and reported per frame;
* optim: optimize_mocap end to end minus its scene time, i.e. the four attempts' 215 GeOptimizer iterations and the copies around them;
* end to end: optimize_mocap's wall time per frame.
Host wall clock around work that ends in a device synchronisation.  Prints the device name and power limit read in the same run, a table
and one JSON line.
usage: python tests/baselines/bench_mocap_driver.py [--frames 1024,6144] [--eager-frames 256]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_manopth import _power_limit  # noqa: E402


def _timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', default='1024,6144')
    ap.add_argument('--eager-frames', type=int, default=256)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_mocap_driver: a CUDA device is required')
    from oracle import ge_optimizer_ref as G
    from oracle import mocap_ref
    from renderih_b200 import assets as A
    from renderih_b200 import mocap_optimize as MO
    geo = torch.load(os.path.join(ROOT, 'tests', 'golden', 'mocap_synth.pt'), weights_only=False)
    fvi, aw, cls = (t.numpy() for t in geo['anchor_tables'])
    scene = MO.Scene(mano_root={s: A.synthetic_mano(0, s) for s in ('right', 'left')}, face_vert_idx=fvi, anchor_weight=aw, class_types=cls)
    rows = []
    for N in [int(n) for n in args.frames.split(',')]:
        raw = mocap_ref.synthetic_mocap(N, 11, joint_deg=5.0, root_deg=20.0)
        quat = [torch.from_numpy(MO.euler_to_mano_quat(raw[s]['rot'], s, *scene.converter[s])).cuda() for s in ('right', 'left')]
        tsl = [torch.from_numpy((raw[s]['loc'] / 100).astype(np.float32)).cuda() for s in ('right', 'left')]
        shape = torch.cat([torch.from_numpy(raw[s]['shape'].astype(np.float32)).squeeze(1) for s in ('right', 'left')], 1).cuda()
        sargs = (quat[0], quat[1], tsl[0], tsl[1], shape)

        def ours_scene():
            ids = None
            for p in range(6):
                ids = scene.update_scene(*sargs, anchor_id=None if p in (0, 1) else ids)['anchor_id']
        ours_scene()
        _, t_scene = _timed(ours_scene)
        fvi_h, aw_h, cls_h = mocap_ref.tables(scene)
        M = min(N, args.eager_frames)

        def eager_scene():
            for p in range(6):
                for f in range(M):
                    with torch.no_grad():
                        vm = scene.main_hand(quat[0][f:f + 1], shape[f:f + 1, :10])[0].cpu().numpy()
                        vs = scene.sub_hand(quat[1][f:f + 1], shape[f:f + 1, 10:])[0].cpu().numpy()
                    mocap_ref.scene_frames(vm, vs, tsl[0][f:f + 1].cpu().numpy(), tsl[1][f:f + 1].cpu().numpy(), fvi_h, aw_h, cls_h)
        _, t_eager = _timed(eager_scene)
        print('frames %d: scene %.4f ms/frame, eager per-frame scene %.3f ms/frame (over %d frames)' % (N, 1e3 * t_scene / N, 1e3 * t_eager / M, M),
              flush=True)
        # no penetration term, as in the golden file: the synthetic hull mesh is not a hand
        opt = G.build((1011, 1.0, (G.THRESH + 3.0, 0.0)), lambda_repulsion_loss=0.0)
        out, t_e2e = _timed(lambda: MO.optimize_mocap(raw, opt, scene, N, 1, 1.0))
        rows.append({'frames': N, 'scene_ms_per_frame': 1e3 * t_scene / N, 'eager_scene_ms_per_frame': 1e3 * t_eager / M,
                     'eager_frames_timed': M, 'scene_speedup': (t_eager / M) / (t_scene / N), 'optim_ms_per_frame': 1e3 * (t_e2e - t_scene) / N,
                     'end_to_end_ms_per_frame': 1e3 * t_e2e / N, 'end_to_end_s': t_e2e})
    name = torch.cuda.get_device_name(torch.cuda.current_device())
    print('device: %s, power limit %s' % (name, _power_limit()))
    print('%6s %14s %14s %8s %14s %14s' % ('frames', 'scene ms/fr', 'eager ms/fr', 'speedup', 'optim ms/fr', 'e2e ms/fr'))
    for r in rows:
        print('%6d %14.4f %14.3f %7.0fx %14.3f %14.3f' % (r['frames'], r['scene_ms_per_frame'], r['eager_scene_ms_per_frame'], r['scene_speedup'],
                                                        r['optim_ms_per_frame'], r['end_to_end_ms_per_frame']))
    print(json.dumps({'bench': 'mocap_driver', 'device': name, 'power_limit': _power_limit(), 'rows': rows}))


if __name__ == '__main__':
    main()
