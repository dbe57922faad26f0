#!/usr/bin/env python
"""BASELINE.json configs[1]: batch-64 eval-mode forward of HandNET_GCN (encoder + attention/GCN decoder + heads) on one H100, images/s.

Companion of bench.py (which measures configs[2], the training step).  Device-timed with CUDA events over a captured CUDA graph, inputs
resident in HBM (`value`), and end to end through the module's public call from pinned host batches with the result vertices read back
(`e2e`).  Prints one JSON line.   usage: python tools/bench_forward.py [--encoder resnet50|hrnet48|graph|newgraph] [--batch 64] [--steps 30]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
FWD_GFLOP = {'resnet50': 17.721, 'hrnet48': 56.201, 'graph': 13.268, 'newgraph': 13.283}     # SURVEY.md 8(d) / bench.py FLOPS (FlopCounterMode on the reference)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--encoder', default='resnet50', choices=list(FWD_GFLOP))
    ap.add_argument('--batch', type=int, default=None)
    ap.add_argument('--steps', type=int, default=30)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--gemm-mode', default='ref')
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), 'needs a CUDA device: there is no CPU path'
    from renderih_b200 import _lib, assets as A, ops
    from renderih_b200.config import load_cfg
    from renderih_b200.model import load_model
    _lib.load()
    conv_mode, lin_mode = {'ref': ('tf32c', 'tf32x3')}.get(args.gemm_mode, (args.gemm_mode, args.gemm_mode))
    ops.set_gemm_mode(conv_mode, lin_mode)
    cfg = load_cfg()
    B = args.batch or (32 if args.encoder == 'hrnet48' else 64)
    a = A.synthetic_assets(0)
    torch.manual_seed(cfg.SEED)
    if args.encoder in ('graph', 'newgraph'):
        from renderih_b200 import myhand
        build = myhand.load_graph_model if args.encoder == 'graph' else myhand.load_new_model
        model = build(cfg, assets=a, mano_assets={s: A.synthetic_mano(0, s) for s in ('left', 'right')}).cuda().eval()
    else:
        cfg.MODEL.ENCODER_TYPE = args.encoder
        model = load_model(cfg, assets=a).cuda().eval()
    g = torch.Generator().manual_seed(cfg.SEED)
    host = [torch.randn(B, 3, 256, 256, generator=g).pin_memory() for _ in range(2)]
    static_in = host[0].cuda()
    c0 = _lib.CALLS[0]
    with torch.no_grad():
        out = model(static_in)
    launches = _lib.CALLS[0] - c0
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.no_grad():
        for _ in range(2):
            model(static_in)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph), torch.no_grad():
        out = model(static_in)
    res = out[0]['verts3d']
    host_out = {k: torch.empty(v.shape, dtype=v.dtype).pin_memory() for k, v in res.items()}

    def timed(fn, n):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(n):
            fn(i)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    for _ in range(max(3, args.warmup)):
        graph.replay()
    ms_dev = timed(lambda i: graph.replay(), args.steps)

    def e2e(i):
        static_in.copy_(host[i % 2], non_blocking=True)
        graph.replay()
        for k in res:
            host_out[k].copy_(res[k], non_blocking=True)
        torch.cuda.current_stream().synchronize()
    for i in range(2):
        e2e(i)
    ms_e2e = timed(e2e, args.steps)
    gf = FWD_GFLOP[args.encoder]
    print(json.dumps({'metric': 'images/sec forward (eval) @batch%d 256x256' % B, 'value': B / (ms_dev * 1e-3), 'unit': 'images/s', 'n_gpus': 1,
                      'steps': args.steps, 'warmup': max(3, args.warmup), 'ms_per_step': ms_dev, 'higher_is_better': True,
                      'dtype': 'f32 storage; wgmma TF32 convolutions + 3xTF32 Linear GEMMs (bench.py `ref` mode)', 'data': 'synthetic',
                      'config': {'workload': 'BASELINE.json configs[1]: HandNET_GCN %s cfg, batch %d, 256x256, eval mode (running-stat BN folded), random-init weights, '
                                             'synthetic graph/MANO assets' % (args.encoder, B), 'cuda_graph': True,
                                 'algorithmic_gflop_per_image_fwd': gf},
                      'achieved_tflops': B / (ms_dev * 1e-3) * gf / 1e3,
                      'e2e': {'value': B / (ms_e2e * 1e-3), 'unit': 'images/s', 'ms_per_step': ms_e2e, 'h2d_bytes_per_step': B * 3 * 256 * 256 * 4,
                              'd2h_bytes_per_step': sum(v.numel() * 4 for v in res.values())},
                      'launches_per_step': launches}))


if __name__ == '__main__':
    main()
