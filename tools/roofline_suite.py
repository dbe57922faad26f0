"""Launch each hot kernel of the path once (after warm-up) on a representative batch-64 shape, for one `ncu --set full` capture:

  ncu --set full --clock-control none --import-source on --profile-from-start off -o gpurun_out/suite python tools/roofline_suite.py

cudaProfilerStart/Stop bracket exactly one launch of: 3x3 conv 128->128 @64x64 (tf32c), 1x1 conv 64->256 @64x64 (HBM bound), a 3xTF32
token Linear, the batched attention GEMMs + softmax kernels (Sq 252, Sk 316, d 16), Chebyshev SpMM, BatchNorm backward, LayerNorm
backward, ManoLayer forward / backward.  `tools/summarize_ncu_suite.py` turns the exported raw page into profiles/*.csv."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from renderih_b200 import assets as A, ops  # noqa: E402
from renderih_b200.manolayer import ManoLayer  # noqa: E402
from renderih_b200.model import GraphCSR  # noqa: E402

B = 64
ops.set_gemm_mode('tf32c', 'tf32x3')
rt = torch.cuda.cudart()


def run(fn, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    rt.cudaProfilerStart()
    out = fn()
    torch.cuda.synchronize()
    rt.cudaProfilerStop()
    return out


# ---- convolutions
x = torch.randn(B * 64 * 64, 128, device='cuda')
w = (torch.randn(128, 128, 3, 3, device='cuda') * 0.03).contiguous(memory_format=torch.channels_last)
run(lambda: ops.conv2d(x, w, None, B, 64, 64, stride=1, pad=1))
x1 = torch.randn(B * 64 * 64, 64, device='cuda')
w1 = (torch.randn(256, 64, 1, 1, device='cuda') * 0.1).contiguous(memory_format=torch.channels_last)
run(lambda: ops.conv2d(x1, w1, None, B, 64, 64))
# ---- round 2: inference convolutions with the eval-mode BatchNorm folded into the epilogue (layer1 of the ResNet-50 trunk)
holder = torch.nn.Sequential(torch.nn.BatchNorm2d(256), torch.nn.BatchNorm2d(64)).cuda().eval()
resid = torch.randn(B * 64 * 64, 256, device='cuda')
x2 = torch.randn(B * 64 * 64, 64, device='cuda')
w2 = (torch.randn(64, 64, 3, 3, device='cuda') * 0.04).contiguous(memory_format=torch.channels_last)
with torch.no_grad():
    ops.bn_fold_refresh(holder)
    f256, f64 = holder[0]._rih_fold, holder[1]._rih_fold
    run(lambda: ops.conv2d_bn_eval(x1, w1, B, 64, 64, 1, 0, f256, order=0, relu=True, res=resid))      # conv3 + bn3 + identity + ReLU
    run(lambda: ops.conv2d_bn_eval(x1, w1, B, 64, 64, 1, 0, f256, order=0, relu=False))                # downsample conv + BN
    run(lambda: ops.conv2d_bn_eval(x2, w2, B, 64, 64, 1, 1, f64, order=0, relu=True))                  # conv2 3x3 64 -> 64 + bn2 + ReLU
# ---- token Linear (3xTF32)
t = torch.randn(B * 252, 128, device='cuda')
wl, bl = torch.randn(64, 128, device='cuda') * 0.1, torch.zeros(64, device='cuda')
run(lambda: ops.linear(t, wl, bl))
t2 = torch.randn(B * 252, 256, device='cuda')
wl2, bl3 = torch.randn(256, 256, device='cuda') * 0.06, torch.zeros(256, device='cuda')
run(lambda: ops.linear(t2, wl2, bl3, res=t2))          # 256 -> 256 with bias + residual (TMA-store epilogue reading the residual rows)
# ---- attention core on wgmma (forward + backward kernels)
q = torch.randn(B * 252, 64, device='cuda', requires_grad=True)
k = torch.randn(B * 316, 64, device='cuda', requires_grad=True)
v = torch.randn(B * 316, 64, device='cuda', requires_grad=True)
go = torch.randn(B * 252, 64, device='cuda')


def attn():
    o = ops.attention(q, k, v, B, 4, 252, 316, p_drop=0.0, impl='tc')
    o.backward(go)


run(attn)
# ---- Chebyshev SpMM
g = GraphCSR(A.synthetic_assets(0)['left_graph']['coarsen_graphs_L'][2]).to(torch.device('cuda'))
xc = torch.randn(B * g.V, 128, device='cuda')
run(lambda: ops.cheb(xc, g, B, g.V))
# ---- BatchNorm forward apply + backward, LayerNorm backward
xb = torch.randn(B * 64 * 64, 256, device='cuda', requires_grad=True)
gam, bet = torch.ones(256, device='cuda', requires_grad=True), torch.zeros(256, device='cuda', requires_grad=True)
rm, rv = torch.zeros(256, device='cuda'), torch.ones(256, device='cuda')
gb = torch.randn(B * 64 * 64, 256, device='cuda')


def bn():
    y = ops.batchnorm(xb, gam, bet, rm, rv, training=True, relu=True)
    y.backward(gb)


run(bn)
xl = torch.randn(B * 252, 64, device='cuda', requires_grad=True)
gl, bl2 = torch.ones(64, device='cuda', requires_grad=True), torch.zeros(64, device='cuda', requires_grad=True)
gy = torch.randn(B * 252, 64, device='cuda')


def ln():
    ops.layernorm(xl, gl, bl2).backward(gy)


run(ln)
# ---- ManoLayer forward + backward (128 hands)
layer = ManoLayer(A.synthetic_mano(0, 'right'), center_idx=9, use_pca=True)
root = torch.linalg.qr(torch.randn(128, 3, 3))[0].cuda()
pose = (torch.randn(128, 45) * 0.5).cuda().requires_grad_(True)
shape = torch.randn(128, 10).cuda().requires_grad_(True)


def mano():
    vv, jj = layer(root, pose, shape)
    (vv.sum() + jj.sum()).backward()


run(mano)
print('suite ok')
