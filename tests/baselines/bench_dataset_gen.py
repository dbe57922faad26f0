"""Throughput of dataset preparation (renderih_b200/dataset_gen.py) on the GPU against the reference's per-frame loop on the host.

* device: the device stage of a batch of B synthetic 334x512 frames held in memory, timed with CUDA events: both hands through ManoLayer,
  the geometry and crop box, the crop and frame sums, the 42 heatmaps as uint8 planes, the mask and the dense map with their uint8
  conversion;
* host: the reference's per-frame loop restated on the host for --host-frames frames: MANO at batch 1 (oracle/mano_ref, the numpy
  statement of the same layer), the numpy geometry and cut_img, cv2.warpAffine and the numpy HeatmapGenerator (the renderer, pytorch3d on
  a GPU in the reference, is left out of it);
* end to end: the device stage, the copies back and cv.imwrite of every JPEG (crop, 14 heatmaps, mask, dense) to a temporary directory on
  a thread pool; IO's share is the part of that time the device stage does not account for.

Prints the device and its power limit, a table and one JSON line.
    python tests/baselines/bench_dataset_gen.py [--batches 512 4096] [--host-frames 64] [--iters 5]
"""
import argparse
import concurrent.futures
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
from oracle import dataset_gen_ref, mano_ref  # noqa: E402
from renderih_b200 import assets, dataset_gen as dg  # noqa: E402
from renderih_b200.render import mano_two_hands_renderer  # noqa: E402

H, W = 512, 334


def inputs(B, rng):
    pose = {s: rng.normal(size=(B, 48)).astype(np.float32) * 0.3 for s in dg.SIDES}
    shape = {s: rng.normal(size=(B, 10)).astype(np.float32) * 0.5 for s in dg.SIDES}
    trans = {s: (rng.normal(size=(B, 3)) * 0.01 + [dx, 0, 0]).astype(np.float32) for s, dx in (('left', -0.04), ('right', 0.04))}
    R = np.tile(np.eye(3, dtype=np.float32), (B, 1, 1))
    t = np.tile(np.array([0, 0, 0.8], np.float32), (B, 1))
    K = np.tile(np.array([[1250.0, 0, W / 2], [0, 1250.0, H / 2], [0, 0, 1]]), (B, 1, 1))
    frames = rng.integers(0, 256, size=(B, H, W, 3), dtype=np.uint8)
    return pose, shape, trans, R, t, K, frames


def device_stage(mano, rend, pose, shape, trans, R, t, K, frames):
    """-> uint8 CUDA tensors (crops, planes, mask, dense) and the frame sums.  pose / shape / trans are host tensors, as parsed from JSON."""
    verts, joints = {}, {}
    for s in dg.SIDES:
        _, verts[s], joints[s] = mano.from_axis(s, pose[s][:, :3], pose[s][:, 3:], shape[s], trans[s])
    g = dg.geometry(verts, joints, R, t, K, crop=True)
    crops, sums = dg.crop_u8(frames, g['M'], dg.IMG_SIZE, sums=True)
    B = R.shape[0]
    j = g['j2d'] * dg.HEATMAP_SIZE / dg.IMG_SIZE
    planes = dg.heatmap_planes(torch.cat([j, torch.ones_like(j[..., :1])], -1).reshape(B * 2, 21, 3).contiguous())
    cams = g['K'].float()
    mask = rend.render_mask(cameras=cams, v3d_left=g['v3d'][:, 0], v3d_right=g['v3d'][:, 1])
    dense, _ = rend.render_densepose(cameras=cams, v3d_left=g['v3d'][:, 0], v3d_right=g['v3d'][:, 1])
    return crops, planes, dg._to_u8(mask, 255.0), dg._to_u8(dense, 255.0), sums


def host_frame(md, pose, shape, trans, R, t, K, frame):
    """One frame of interhand.py's and step 7's loops on the host."""
    import cv2
    v2d, j2d = [], []
    for s in dg.SIDES:
        rot = mano_ref.rodrigues(pose[s][:3][None].astype(np.float64))
        pca = (pose[s][3:] + md[s]['hands_mean']) @ np.linalg.inv(md[s]['hands_components'])
        v, j = mano_ref.mano_forward(md[s], rot, pca[None].astype(np.float32), shape[s][None])
        v, j = v[0] + trans[s], j[0] + trans[s]
        v2d.append(dataset_gen_ref.project(dataset_gen_ref.cam_xform(v, R, t), K))
        j2d.append(dataset_gen_ref.project(dataset_gen_ref.cam_xform(j, R, t), K))
    M, _, _ = dataset_gen_ref.cut(np.concatenate(v2d), dg.HAND_BBOX_RATIO, dg.IMG_SIZE, K)
    cv2.warpAffine(frame, M, dsize=(dg.IMG_SIZE, dg.IMG_SIZE))
    frame.mean()
    for j in j2d:
        dataset_gen_ref.heatmaps(j * dg.HEATMAP_SIZE / dg.IMG_SIZE, dg.HEATMAP_SIZE, dg.HEATMAP_SIGMA)


def main():
    import cv2
    ap = argparse.ArgumentParser()
    ap.add_argument('--batches', type=int, nargs='+', default=[512, 4096])
    ap.add_argument('--host-frames', type=int, default=64)
    ap.add_argument('--iters', type=int, default=5)
    a = ap.parse_args()
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], stdout=subprocess.PIPE,
                       text=True).stdout.strip().splitlines()[0]
    print('device: %s (name, power limit, max SM clock)' % q)
    md = {s: assets.synthetic_mano(0, s) for s in dg.SIDES}
    mano = dg._Mano(md, 'cuda')
    host_md = {s: dict(m, J_regressor=np.asarray(m['J_regressor'].todense())) for s, m in md.items()}
    rend = mano_two_hands_renderer(md, assets.synthetic_assets(0)['dense_coor'], img_size=dg.IMG_SIZE)
    rng = np.random.default_rng(0)
    res = {'device': q, 'frame': [H, W]}
    for B in a.batches:
        pose, shape, trans, R, t, K, frames = inputs(B, rng)
        dev = [{s: torch.from_numpy(x[s]) for s in dg.SIDES} for x in (pose, shape, trans)]
        dev += [torch.from_numpy(x).cuda() for x in (R, t, K, frames)]
        run = lambda: device_stage(mano, rend, *dev)
        run()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.iters):
            run()
        e1.record()
        torch.cuda.synchronize()
        t_dev = e0.elapsed_time(e1) / 1e3 / a.iters
        with tempfile.TemporaryDirectory() as tmp, concurrent.futures.ThreadPoolExecutor(8) as pool:
            t0 = time.perf_counter()
            crops, planes, mask, dense, _ = (x.cpu().numpy() for x in run())
            futs = []
            for b in range(B):
                futs.append(pool.submit(cv2.imwrite, os.path.join(tmp, 'c%d.jpg' % b), crops[b]))
                futs.append(pool.submit(cv2.imwrite, os.path.join(tmp, 'm%d.jpg' % b), mask[b]))
                futs.append(pool.submit(cv2.imwrite, os.path.join(tmp, 'd%d.jpg' % b), dense[b]))
                for k in range(14):
                    futs.append(pool.submit(cv2.imwrite, os.path.join(tmp, 'h%d_%d.jpg' % (b, k)), planes.reshape(B, 14, 64, 64, 3)[b, k]))
            for f in futs:
                f.result()
            t_e2e = time.perf_counter() - t0
        res['B%d' % B] = {'device_ms_per_frame': t_dev / B * 1e3, 'e2e_ms_per_frame': t_e2e / B * 1e3, 'io_share': max(0.0, 1 - t_dev / t_e2e)}
    n = a.host_frames
    pose, shape, trans, R, t, K, frames = inputs(n, rng)
    t0 = time.perf_counter()
    for b in range(n):
        host_frame(host_md, {s: pose[s][b] for s in pose}, {s: shape[s][b] for s in shape}, {s: trans[s][b] for s in trans}, R[b], t[b], K[b], frames[b])
    res['host_ms_per_frame'] = (time.perf_counter() - t0) / n * 1e3
    res['host_frames'] = n
    print('%-44s %12s' % ('path', 'ms / frame'))
    for B in a.batches:
        r = res['B%d' % B]
        print('%-44s %12.4f' % ('GPU device stage, B = %d' % B, r['device_ms_per_frame']))
        print('%-44s %12.4f   (IO share %.2f)' % ('GPU + copies + JPEG writes, B = %d' % B, r['e2e_ms_per_frame'], r['io_share']))
    print('%-44s %12.4f' % ('host per-frame loop (no renderer), %d frames' % n, res['host_ms_per_frame']))
    print(json.dumps(res))


if __name__ == '__main__':
    main()
