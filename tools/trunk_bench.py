#!/usr/bin/env python
"""The convolution side of the step in isolation: ResNet-50 trunk (stem + layer1..4, train-mode BatchNorm) forward + backward at batch 64,
captured into a CUDA graph and replayed -- the serial, bandwidth-bound 55 % of the training step (tools/timeline.py).  Used to A/B the
environment switches that remain (RIH_PDL), one process per variant:

    RIH_PDL=1 python tools/trunk_bench.py  ->  one JSON line {variant flags, ms fwd, ms fwd+bwd}
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    from renderih_b200 import _lib, assets as A, ops
    from renderih_b200.config import load_cfg
    from renderih_b200.model import load_model
    _lib.load()
    ops.set_gemm_mode('tf32c', 'tf32x3')
    B = int(os.environ.get('RIH_TB_BATCH', '64'))
    cfg = load_cfg()
    torch.manual_seed(cfg.SEED)
    model = load_model(cfg, assets=A.synthetic_assets(0)).cuda().train()
    enc = model.encoder
    img = torch.randn(B, 3, 256, 256, device='cuda')

    def fwd():
        feats = enc.trunk(img)
        return sum(f[0].mean() for f in feats)

    def fwd_bwd():
        for p in enc.parameters():
            p.grad = None
        fwd().backward()

    res = {}
    for name, fn, ng in (('fwd_ms', fwd, True), ('fwd_bwd_ms', fwd_bwd, False)):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                if ng:
                    with torch.no_grad():
                        fn()
                else:
                    fn()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            if ng:
                with torch.no_grad():
                    fn()
            else:
                fn()
        for _ in range(3):
            g.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = 15
        e0.record()
        for _ in range(n):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
        res[name] = e0.elapsed_time(e1) / n
        del g
    flags = {k: v for k, v in os.environ.items() if k.startswith('RIH_')}
    print(json.dumps({'flags': flags, **res}))


if __name__ == '__main__':
    main()
