"""Timing of the two-hand renderer (renderih_b200/render.py) at batch 64, 256 x 256, both hands (2 x 1538 faces): render_rgb_orth (Phong),
render_mask, render_densepose (ambient) and hand_mask_iou, CUDA events around --iters calls after --warmup calls.  Prints one JSON line
with the device name and power limit read in the same run, and beside each time the bytes its outputs occupy over 3.35 TB/s (the H100 SXM
data-sheet HBM3 bandwidth): a floor, not a target -- the work is rasterisation, not streaming.  Uses the MANO meshes under the asset root
($RIH_ASSET_ROOT) when present, else the synthetic MANO stand-in (random faces: long slivers, far more pixels per face); "mesh" says which.
usage: python tools/bench_render.py [--batch 64] [--size 256] [--iters 20] [--warmup 5]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12


def _power_limit():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, timeout=30).stdout.decode().strip()
        return out or 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def _time(fn, iters, warmup):
    for _ in range(warmup):
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
    ap.add_argument('--batch', type=int, default=64)
    ap.add_argument('--size', type=int, default=256)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_render.py needs a CUDA device')
    from renderih_b200 import assets as A
    from renderih_b200.config import get_cfg_defaults
    from renderih_b200.manolayer import ManoLayer, rodrigues_batch
    from renderih_b200.render import hand_mask_iou, mano_two_hands_renderer
    B, S = args.batch, args.size
    root, cfg = A.default_asset_root(), get_cfg_defaults()
    paths = {s: os.path.join(root, cfg.MISC.MANO_PATH, 'MANO_%s.pkl' % s.upper()) for s in ('left', 'right')}
    if all(os.path.exists(p) for p in paths.values()):
        manos, mesh = {s: A.load_mano_dict(p) for s, p in paths.items()}, 'mano'
    else:
        manos, mesh = {s: A.synthetic_mano(0, s) for s in ('left', 'right')}, 'synthetic'
    rend = mano_two_hands_renderer(manos, A.synthetic_assets(0)['dense_coor'], img_size=S)
    g = torch.Generator().manual_seed(0)
    hands = []
    for side, dx in (('left', -0.04), ('right', 0.04)):
        layer = ManoLayer(manos[side], center_idx=9, use_pca=True)
        rot = rodrigues_batch((torch.rand(B, 3, generator=g) - 0.5) * 2.0).cuda()
        v, _ = layer(rot, (torch.randn(B, 45, generator=g) * 0.6).cuda(), (torch.randn(B, 10, generator=g) * 0.5).cuda())
        hands.append(v + torch.tensor([dx, 0.0, 0.0], device='cuda'))
    vl, vr = hands
    sl, sr = (1.8 + 0.4 * torch.rand(B, generator=g)).cuda(), (1.8 + 0.4 * torch.rand(B, generator=g)).cuda()
    tl, tr = ((torch.rand(B, 2, generator=g) - 0.5) * 0.3).cuda(), ((torch.rand(B, 2, generator=g) - 0.5) * 0.3).cuda()
    one = rend.faces_np[:len(rend.faces_np) // 2]
    px = B * S * S
    cases = {
        'render_rgb_orth': (lambda: rend.render_rgb_orth(sl, tl, sr, tr, vl, vr), px * 16),        # img fp32 x 3 + alpha
        'render_mask': (lambda: rend.render_mask(scale=sl, trans2d=tl, v3d_left=vl, v3d_right=vr), px * 16),
        'render_densepose': (lambda: rend.render_densepose(scale=sl, trans2d=tl, v3d_left=vl, v3d_right=vr), px * 16),
        'hand_mask_iou': (lambda: hand_mask_iou(vl, vr, one, S, scale=sl, trans2d=tl), B * 4),
    }
    alpha = rend.render_rgb_orth(sl, tl, sr, tr, vl, vr)[1]
    res = {'device': torch.cuda.get_device_name(), 'power_limit': _power_limit(), 'batch': B, 'img_size': S, 'faces': int(len(rend.faces_np)),
           'mesh': mesh, 'covered_fraction': round(float(alpha.mean()), 4), 'iters': args.iters, 'warmup': args.warmup}
    for name, (fn, nbytes) in cases.items():
        ms = _time(fn, args.iters, args.warmup)
        res[name] = {'ms': round(ms, 4), 'out_bytes': nbytes, 'hbm_floor_ms': round(nbytes / HBM_BYTES_PER_S * 1e3, 4)}
    print(json.dumps(res))


if __name__ == '__main__':
    main()
