"""The register-A main loop of the wgmma GEMM (rih_set_gemm_rs) against the shared-memory-transpose main loop it replaces, on the
convolution weight gradients of ResNet-50, HRNet-w48 and the RGB stem, in every tensor-core arithmetic mode.

Both main loops multiply the same fp32 bits in the same k order (k-blocks, k8 steps and, for 3xTF32, the hi*hi, lo*hi, hi*lo order), so
the results must be bitwise equal wherever the old path is itself deterministic.  Split-K launches reduce their partial tiles with TMA
reduce-adds in arrival order; there the two paths may differ by fp32 reordering of those partial sums.  Both are also held to the exact
SIMT path within the tolerances of tests/test_ops_gpu.py."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

torch.backends.cudnn.allow_tf32 = False     # the torch reference of the stem must be true fp32

DEV = 'cuda'
MODES = ('tf32c', 'tf32rn', 'tf32x3')
SIMT_TOL = {'tf32c': 3e-3, 'tf32rn': 3e-3, 'tf32x3': 1e-4}
REORDER_TOL = 2e-6       # split-K: relative to the tensor's max magnitude

# (N, H, Cin, Cout, k, stride): input H x H, k x k filter, pad k // 2.  The 3x3 and strided convolutions: 1x1 stride-1 weight gradients
# are plain GEMMs (rih_conv2d_wgrad hands them to the dense path, which keeps the shared-memory main loop).
RESNET50 = [(2, 64, 64, 64, 3, 1), (2, 64, 128, 128, 3, 2), (2, 64, 256, 512, 1, 2), (2, 32, 128, 128, 3, 1), (2, 32, 256, 256, 3, 2),
            (2, 32, 512, 1024, 1, 2), (2, 16, 256, 256, 3, 1), (2, 16, 512, 512, 3, 2), (2, 16, 1024, 2048, 1, 2), (2, 8, 512, 512, 3, 1)]
HRNET48 = [(2, 64, 64, 64, 3, 2), (2, 64, 256, 48, 3, 1), (2, 64, 256, 96, 3, 2), (2, 64, 48, 48, 3, 1), (2, 32, 96, 96, 3, 1),
           (2, 16, 192, 192, 3, 1), (2, 8, 384, 384, 3, 1), (2, 64, 48, 96, 3, 2), (2, 32, 96, 192, 3, 2), (2, 16, 192, 384, 3, 2),
           (2, 64, 48, 80, 3, 1)]


@pytest.fixture(scope='module')
def lib():
    from renderih_b200 import ops
    from renderih_b200._lib import call, load
    load()
    yield ops, call
    call('rih_set_gemm_rs', 1)
    ops.set_gemm_mode('simt', 'simt')


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-20))


def run(lib, mode, rs, fn):
    ops, call = lib
    ops.set_gemm_mode(mode, mode)
    call('rih_set_gemm_rs', rs)
    try:
        out = fn()
        torch.cuda.synchronize()
    finally:
        call('rih_set_gemm_rs', 1)
        ops.set_gemm_mode('simt', 'simt')
    return out


def old_vs_new(lib, mode, fn, what):
    """The register-A result, after checking it against the shared-memory path (run twice to see whether that one is deterministic)."""
    old1, old2 = run(lib, mode, 0, fn), run(lib, mode, 0, fn)
    new = run(lib, mode, 1, fn)
    if torch.equal(old1, old2):
        assert torch.equal(new, old1), '%s %s: register-A result differs from the shared-memory path (rel %.3e)' % (what, mode, rel(new, old1))
    else:
        assert rel(new, old1) < REORDER_TOL, '%s %s: rel %.3e' % (what, mode, rel(new, old1))
    return new


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('acc', (0, 1))
@pytest.mark.parametrize('N,H,Cin,Cout,k,stride', RESNET50 + HRNET48)
def test_conv_wgrad_register_a(lib, mode, acc, N, H, Cin, Cout, k, stride):
    ops, call = lib
    g = torch.Generator().manual_seed(N * 7919 + H * 131 + Cin * 17 + Cout + k + stride)
    Ho = (H + 2 * (k // 2) - k) // stride + 1
    x = torch.randn(N * H * H, Cin, generator=g).to(DEV)
    dy = torch.randn(N * Ho * Ho, Cout, generator=g).to(DEV)
    dw0 = torch.randn(Cout, k * k * Cin, generator=g).to(DEV)
    geom = (ctypes.c_int * 13)(N, H, H, Cin, Ho, Ho, Cout, k, k, stride, k // 2, Cin, Cout)
    flag = ctypes.c_int(0)
    ops.set_gemm_mode(mode, mode)
    try:
        call('rih_conv2d_tc_supported', geom, 2, ctypes.byref(flag))
    finally:
        ops.set_gemm_mode('simt', 'simt')
    assert flag.value == 1, 'not on the tensor-core path'
    n = ctypes.c_longlong(0)
    call('rih_conv2d_workspace', geom, 2, ctypes.byref(n))
    ws = torch.empty(max(n.value, 1), device=DEV)

    def fn():
        dw = dw0.clone()
        call('rih_conv2d_wgrad', ctypes.c_void_p(dy.data_ptr()), ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(dw.data_ptr()), geom, acc,
             ctypes.c_void_p(ws.data_ptr()), None)
        return dw
    what = 'conv wgrad %s' % ((N, H, Cin, Cout, k, stride),)
    new = old_vs_new(lib, mode, fn, what)
    exact = run(lib, 'simt', 1, fn)
    assert rel(new, exact) < SIMT_TOL[mode], '%s %s: rel %.3e vs exact fp32' % (what, mode, rel(new, exact))


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('acc', (0, 1))
@pytest.mark.parametrize('N', (2, 5))
def test_stem_wgrad_register_a(lib, mode, acc, N):
    _, call = lib
    H = W = 256
    g = torch.Generator().manual_seed(11 + N)
    img = torch.randn(N, 3, H, W, generator=g).to(DEV)
    dy = torch.randn(N * (H // 2) * (W // 2), 64, generator=g).to(DEV)
    dw0 = torch.randn(64, 224, generator=g).to(DEV)
    xp = torch.empty((N, H + 6, W + 8, 4), device=DEV)
    call('rih_nchw_to_nhwc4_pad', ctypes.c_void_p(img.data_ptr()), ctypes.c_void_p(xp.data_ptr()), N, H, W, None)

    def fn():
        dw = dw0.clone()
        call('rih_stem_conv_wgrad', ctypes.c_void_p(dy.data_ptr()), 64, ctypes.c_void_p(xp.data_ptr()), ctypes.c_void_p(dw.data_ptr()),
             N, H, W, acc, None)
        return dw
    new = old_vs_new(lib, mode, fn, 'stem wgrad')
    # exact reference: torch fp32 conv1 weight gradient.  w224 is [64][7][8][4]; its 8th column and 4th channel are padding (the 4th
    # channel of the image is zero, the 8th column meets real pixels), so only the [:, :, :7, :3] entries are compared.
    w = torch.zeros(64, 3, 7, 7, device=DEV, requires_grad=True)
    y = torch.nn.functional.conv2d(img, w, stride=2, padding=3)
    (gw,) = torch.autograd.grad(y, [w], dy.reshape(N, H // 2, W // 2, 64).permute(0, 3, 1, 2))
    ref = gw.permute(0, 2, 3, 1) + (dw0.reshape(64, 7, 8, 4)[:, :, :7, :3] if acc else 0)
    got = new.reshape(64, 7, 8, 4)[:, :, :7, :3]
    assert rel(got, ref) < SIMT_TOL[mode], 'stem wgrad %s: rel %.3e vs torch fp32' % (mode, rel(got, ref))
