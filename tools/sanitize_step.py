#!/usr/bin/env python
"""One small eager training step (batch 2; bench arithmetic: wgmma TF32 convolutions + 3xTF32 Linears / attention; hand / grid / aux / weight-gradient
side streams on; fused loss; fused AdamW) for compute-sanitizer:

    compute-sanitizer --tool memcheck  --log-file gpurun_out/sanitizer_memcheck.log  python tools/sanitize_step.py
    compute-sanitizer --tool racecheck --log-file gpurun_out/sanitizer_racecheck.log python tools/sanitize_step.py

Prints the loss and a checksum of the flat gradient; exits non-zero on a non-finite result.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import numpy as np
    import torch
    from renderih_b200 import _lib, assets as A, ops
    from renderih_b200.config import load_cfg
    from renderih_b200.loss import GraphLoss, calc_loss_GCN
    from renderih_b200.model import load_model
    from renderih_b200.train import TrainStep
    _lib.load()
    mode = os.environ.get('RIH_SAN_MODE', 'ref')
    conv_mode, lin_mode = {'ref': ('tf32c', 'tf32x3')}.get(mode, (mode, mode))
    ops.set_gemm_mode(conv_mode, lin_mode)
    B = int(os.environ.get('RIH_SAN_BATCH', '2'))
    cfg = load_cfg()
    a = A.synthetic_assets(0)
    torch.manual_seed(1)
    model = load_model(cfg, assets=a).cuda().train()
    model.decoder.unsample_layer.weight.requires_grad_(False)
    g = torch.Generator().manual_seed(2)
    img = torch.randn(B, 3, 256, 256, generator=g).cuda()
    lab = {k: (torch.randn(*s, generator=g) * 0.05).cuda() for k, s in (('v3d_l', (B, 778, 3)), ('v3d_r', (B, 778, 3)), ('root_rel', (B, 3)))}
    lab.update({k: (torch.rand(B, 778, 2, generator=g) * 256).cuda() for k in ('v2d_l', 'v2d_r')})
    ml, mr = A.synthetic_mano(0, 'left'), A.synthetic_mano(0, 'right')
    jl = torch.from_numpy(np.asarray(ml['J_regressor'].todense(), dtype='float32'))
    jr = torch.from_numpy(np.asarray(mr['J_regressor'].todense(), dtype='float32'))
    gl, gr = GraphLoss(jl, ml['f'], 4, 'cuda'), GraphLoss(jr, mr['f'], 4, 'cuda')
    conv = model.decoder.converter
    z = torch.zeros(B, 21, 3, device='cuda')

    def loss_fn(out):
        return calc_loss_GCN(cfg, 0, gl, gr, conv['left'], conv['right'], out[0], out[1], out[2], out[3], None, None, None,
                             lab['v2d_l'], z[..., :2], lab['v2d_r'], z[..., :2], lab['v3d_l'], z, lab['v3d_r'], z, lab['root_rel'], 256)[0]
    step = TrainStep(model, loss_fn, img, use_graph=False)
    loss = step(img)
    torch.cuda.synchronize()
    gsum = float(step.flatp.grad.double().abs().sum())
    print('sanitize_step: mode %s batch %d loss %.6f |grad|_1 %.6e' % (mode, B, float(loss), gsum))
    if not (np.isfinite(float(loss)) and np.isfinite(gsum)):
        sys.exit(2)


if __name__ == '__main__':
    main()
