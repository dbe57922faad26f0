"""Transposed-output input gradients and the remaining register-A operands of the wgmma GEMM (rih_set_gemm_rs bit 1) against the kernels
they replace (rih_set_gemm_rs(1)), on the convolution input gradients of ResNet-50 and HRNet-w48, the token decoder's Linear gradients, the
1x1 convolution weight gradients and the attention backward, in every tensor-core arithmetic mode.

dX^T = W^T dY^T multiplies the same fp32 bits in the same k order as dX = dY W (k-blocks, k8 steps and, for 3xTF32, the hi*hi, lo*hi, hi*lo
order of the untransposed product), so the results must be bitwise equal wherever the old path is itself deterministic.  Split-K launches
(the weight gradients) reduce their partial tiles in arrival order; there the two may differ by fp32 reordering of those partial sums.  Every
case is also held to the exact SIMT path within the tolerances of tests/test_ops_gpu.py, and every case checks through
rih_gemm_dgrad_t_launches that the transposed form ran exactly where the shape rule selects it (>= 128 input channels / in-features)."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

torch.backends.cuda.matmul.allow_tf32 = False

DEV = 'cuda'
MODES = ('tf32c', 'tf32rn', 'tf32x3')
SIMT_TOL = {'tf32c': 3e-3, 'tf32rn': 3e-3, 'tf32x3': 1e-4}
REORDER_TOL = 2e-6       # relative to the tensor's max magnitude
OLD, NEW = 1, 3          # rih_set_gemm_rs bit masks

# (N, H, Cin, Cout, k, stride): input H x H, k x k filter, pad k // 2 -- the input gradients of the training step's convolutions (batch 2).
# Cin >= 128 runs transposed; Cin = 64, 48, 96 keep the untransposed product.  Cin = 192 leaves 64 rows of its second m tile beyond Cin.
RESNET50 = [(2, 64, 64, 64, 3, 1), (2, 64, 256, 64, 1, 1), (2, 64, 64, 256, 1, 1), (2, 64, 256, 128, 1, 1), (2, 64, 128, 128, 3, 2),
            (2, 32, 128, 512, 1, 1), (2, 64, 256, 512, 1, 2), (2, 32, 512, 128, 1, 1), (2, 32, 128, 128, 3, 1), (2, 32, 256, 256, 3, 2),
            (2, 16, 256, 1024, 1, 1), (2, 32, 512, 1024, 1, 2), (2, 16, 1024, 256, 1, 1), (2, 16, 256, 256, 3, 1), (2, 16, 512, 512, 3, 2),
            (2, 8, 512, 2048, 1, 1), (2, 16, 1024, 2048, 1, 2), (2, 8, 2048, 512, 1, 1), (2, 8, 512, 512, 3, 1)]
HRNET48 = [(2, 64, 64, 64, 3, 2), (2, 64, 256, 48, 3, 1), (2, 64, 48, 48, 3, 1), (2, 32, 96, 96, 3, 1), (2, 16, 192, 192, 3, 1),
           (2, 8, 384, 384, 3, 1), (2, 16, 192, 384, 3, 2), (2, 32, 96, 192, 3, 2), (2, 64, 256, 96, 3, 2), (2, 16, 192, 48, 1, 1),
           (2, 8, 384, 96, 1, 1)]
# (M, N, K): dx[M, K] = dy[M, N] . w[N, K] and dw[N, K] = dy^T x of the decoder's Linears
LINEAR = [(4032, 256, 256), (4032, 1024, 256), (4032, 256, 1024), (8064, 768, 256), (16128, 256, 64), (16128, 64, 256), (20224, 512, 512),
          (20224, 128, 128), (4000, 256, 320), (20200, 512, 192), (8100, 96, 160)]
# (B, H, Sq, Sk, d) of the decoder's attention
ATTN = [(2, 4, 63, 63, 64), (2, 4, 252, 316, 16), (2, 4, 126, 190, 32), (5, 4, 63, 127, 64)]

BITWISE = [0, 0]         # [bitwise equal, compared] over the module


@pytest.fixture(scope='module')
def lib():
    from renderih_b200 import ops
    from renderih_b200._lib import call, load
    load()
    yield ops, call
    call('rih_set_gemm_rs', NEW)
    ops.set_gemm_mode('simt', 'simt')
    print('\ntransposed / register-A vs old kernels: %d of %d comparisons bitwise equal' % tuple(BITWISE))


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-20))


def t_launches(call):
    """transposed-output launches since the last call (the count is reset)"""
    n = ctypes.c_longlong(0)
    call('rih_gemm_dgrad_t_launches', ctypes.byref(n), 1)
    return n.value


def run(lib, conv_mode, lin_mode, rs, fn):
    ops, call = lib
    ops.set_gemm_mode(conv_mode, lin_mode)
    call('rih_set_gemm_rs', rs)
    try:
        out = fn()
        torch.cuda.synchronize()
    finally:
        call('rih_set_gemm_rs', NEW)
        ops.set_gemm_mode('simt', 'simt')
    return out


def old_vs_new(lib, mode, fn, what, transposed, lin_mode=None):
    """The new result, after checking it against the old kernels (run twice to see whether those are deterministic) and that the new
    setting ran the transposed form iff `transposed`."""
    call = lib[1]
    lm = lin_mode or mode
    t_launches(call)
    old1, old2 = run(lib, mode, lm, OLD, fn), run(lib, mode, lm, OLD, fn)
    assert t_launches(call) == 0, '%s: the old setting ran the transposed form' % what
    new = run(lib, mode, lm, NEW, fn)
    n = t_launches(call)
    assert (n > 0) == transposed, '%s %s: %d transposed launches, expected %s' % (what, mode, n, 'some' if transposed else 'none')
    if isinstance(new, torch.Tensor):
        old1, old2, new = [old1], [old2], [new]
    for o1, o2, n in zip(old1, old2, new):
        BITWISE[1] += 1
        BITWISE[0] += int(torch.equal(n, o1))
        if torch.equal(o1, o2):
            assert torch.equal(n, o1), '%s %s: differs from the old kernels (rel %.3e)' % (what, mode, rel(n, o1))
        else:
            assert rel(n, o1) < REORDER_TOL, '%s %s: rel %.3e' % (what, mode, rel(n, o1))
    return new[0] if len(new) == 1 else new


def conv_case(lib, N, H, Cin, Cout, k, stride, ldx_pad=0):
    ops, call = lib
    g = torch.Generator().manual_seed(N * 7919 + H * 131 + Cin * 17 + Cout + k + stride)
    Ho = (H + 2 * (k // 2) - k) // stride + 1
    ldx = Cin + ldx_pad
    dy = torch.randn(N * Ho * Ho, Cout, generator=g).to(DEV)
    w = torch.randn(Cout, k * k * Cin, generator=g).to(DEV)
    dx0 = torch.randn(N * H * H, ldx, generator=g).to(DEV)
    geom = (ctypes.c_int * 13)(N, H, H, Cin, Ho, Ho, Cout, k, k, stride, k // 2, ldx, Cout)
    # stride 2 + accumulate is served by the zero-inserted dY formulation, which needs this workspace (rih_conv2d_dgrad)
    ws = torch.empty(N * H * H * Cout if stride == 2 else 1, device=DEV)
    return dy, w, dx0, geom, ws


def conv_dgrad(call, dy, w, dx0, geom, ws, acc):
    def fn():
        dx = dx0.clone()
        call('rih_conv2d_dgrad', ctypes.c_void_p(dy.data_ptr()), ctypes.c_void_p(w.data_ptr()), ctypes.c_void_p(dx.data_ptr()), geom, acc,
             ctypes.c_void_p(ws.data_ptr()), None)
        return dx
    return fn


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('acc', (0, 1))
@pytest.mark.parametrize('N,H,Cin,Cout,k,stride', RESNET50 + HRNET48)
def test_conv_dgrad_transposed(lib, mode, acc, N, H, Cin, Cout, k, stride):
    ops, call = lib
    dy, w, dx0, geom, ws = conv_case(lib, N, H, Cin, Cout, k, stride)
    flag = ctypes.c_int(0)
    ops.set_gemm_mode(mode, mode)
    try:
        call('rih_conv2d_tc_supported', geom, 1, ctypes.byref(flag))
    finally:
        ops.set_gemm_mode('simt', 'simt')
    assert flag.value == 1, 'not on the tensor-core path'
    fn = conv_dgrad(call, dy, w, dx0, geom, ws, acc)
    what = 'conv dgrad %s' % ((N, H, Cin, Cout, k, stride),)
    new = old_vs_new(lib, mode, fn, what, Cin >= 128)
    exact = run(lib, 'simt', 'simt', NEW, fn)
    assert rel(new, exact) < SIMT_TOL[mode], '%s %s: rel %.3e vs exact fp32' % (what, mode, rel(new, exact))


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('N,H,Cin,Cout,k,stride', [(2, 16, 192, 192, 3, 1), (2, 16, 192, 48, 1, 1), (2, 16, 192, 384, 3, 2), (2, 32, 320, 64, 1, 1)])
def test_conv_dgrad_transposed_tail_rows_and_accumulate(lib, mode, N, H, Cin, Cout, k, stride):
    """Cin % 128 != 0: the rows of the last m tile beyond Cin (the next tap's weights) are computed but never stored -- the columns of a
    padded dX row beyond Cin keep their values -- and accumulate adds onto the existing dX."""
    _, call = lib
    dy, w, dx0, geom, ws = conv_case(lib, N, H, Cin, Cout, k, stride, ldx_pad=64)
    t_launches(call)
    store = run(lib, mode, mode, NEW, conv_dgrad(call, dy, w, dx0, geom, ws, 0))
    assert t_launches(call) > 0, 'not on the transposed form'
    assert torch.equal(store[:, Cin:], dx0[:, Cin:]), 'columns beyond Cin were written'
    exact = run(lib, 'simt', 'simt', NEW, conv_dgrad(call, dy, w, dx0, geom, ws, 0))
    assert rel(store[:, :Cin], exact[:, :Cin]) < SIMT_TOL[mode], 'rel %.3e vs exact fp32' % rel(store[:, :Cin], exact[:, :Cin])
    if stride == 1:      # stride-2 accumulation runs the zero-inserted formulation: its own check in test_conv_dgrad_transposed
        accd = run(lib, mode, mode, NEW, conv_dgrad(call, dy, w, dx0, geom, ws, 1))
        assert t_launches(call) > 0, 'not on the transposed form (accumulate)'
        assert torch.equal(accd[:, Cin:], dx0[:, Cin:]), 'columns beyond Cin were written (accumulate)'
        assert rel(accd[:, :Cin], dx0[:, :Cin] + store[:, :Cin]) < 1e-6, 'accumulate does not add onto dX'


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('acc', (0, 1))
@pytest.mark.parametrize('M,N,K', LINEAR)
def test_linear_dgrad_transposed_and_wgrad_register_a(lib, mode, acc, M, N, K):
    _, call = lib
    g = torch.Generator().manual_seed(M + 7 * N + 13 * K)
    dy = torch.randn(M, N, generator=g).to(DEV)
    w = torch.randn(N, K, generator=g).to(DEV)
    x = torch.randn(M, K, generator=g).to(DEV)
    dx0 = torch.randn(M, K, generator=g).to(DEV)
    dw0 = torch.randn(N, K, generator=g).to(DEV)

    def dgrad():
        dx = dx0.clone()
        call('rih_linear_dgrad', ctypes.c_void_p(dy.data_ptr()), N, ctypes.c_void_p(w.data_ptr()), K, ctypes.c_void_p(dx.data_ptr()), K,
             M, N, K, acc, 0, None)
        return dx

    def wgrad():
        dw = dw0.clone()
        call('rih_linear_wgrad', ctypes.c_void_p(dy.data_ptr()), N, ctypes.c_void_p(x.data_ptr()), K, ctypes.c_void_p(dw.data_ptr()), K,
             M, N, K, acc, 0, None)
        return dw
    for fn, what, tr in ((dgrad, 'linear dgrad', K >= 128), (wgrad, 'linear wgrad', False)):
        what = '%s %s' % (what, (M, N, K))
        new = old_vs_new(lib, mode, fn, what, tr)
        exact = run(lib, 'simt', 'simt', NEW, fn)
        assert rel(new, exact) < SIMT_TOL[mode], '%s %s: rel %.3e vs exact fp32' % (what, mode, rel(new, exact))


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('acc', (0, 1))
@pytest.mark.parametrize('N,H,Cin,Cout', [(2, 64, 64, 256), (2, 64, 256, 64), (2, 32, 512, 128), (2, 16, 1024, 256), (2, 8, 2048, 512),
                                          (2, 16, 192, 48)])
def test_conv1x1_wgrad_register_a(lib, mode, acc, N, H, Cin, Cout):
    _, call = lib
    g = torch.Generator().manual_seed(N + H + 3 * Cin + 5 * Cout)
    x = torch.randn(N * H * H, Cin, generator=g).to(DEV)
    dy = torch.randn(N * H * H, Cout, generator=g).to(DEV)
    dw0 = torch.randn(Cout, Cin, generator=g).to(DEV)
    geom = (ctypes.c_int * 13)(N, H, H, Cin, H, H, Cout, 1, 1, 1, 0, Cin, Cout)
    ws = torch.empty(1, device=DEV)

    def fn():
        dw = dw0.clone()
        call('rih_conv2d_wgrad', ctypes.c_void_p(dy.data_ptr()), ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(dw.data_ptr()), geom, acc,
             ctypes.c_void_p(ws.data_ptr()), None)
        return dw
    what = 'conv1x1 wgrad %s' % ((N, H, Cin, Cout),)
    new = old_vs_new(lib, mode, fn, what, False)
    exact = run(lib, 'simt', 'simt', NEW, fn)
    assert rel(new, exact) < SIMT_TOL[mode], '%s %s: rel %.3e vs exact fp32' % (what, mode, rel(new, exact))


@pytest.mark.parametrize('mode', ('tf32', 'tf32x3'))
@pytest.mark.parametrize('B,H,Sq,Sk,d', ATTN)
def test_attention_backward_register_a(lib, mode, B, H, Sq, Sk, d):
    ops, _ = lib
    g = torch.Generator().manual_seed(B + H + Sq + Sk + d)
    q0, k0, v0 = (torch.randn(B * S, H * d, generator=g).to(DEV) for S in (Sq, Sk, Sk))
    do = torch.randn(B * Sq, H * d, generator=g).to(DEV)

    def fn():
        q, k, v = (t.clone().requires_grad_(True) for t in (q0, k0, v0))
        o = ops.attention(q, k, v, B, H, Sq, Sk, impl='tc')
        return list(torch.autograd.grad(o, [q, k, v], do))
    what = 'attention bwd %s' % ((B, H, Sq, Sk, d),)
    new = old_vs_new(lib, 'simt', fn, what, False, lin_mode=mode)
    qh, kh, vh = (t.double().view(B, -1, H, d).transpose(1, 2).requires_grad_(True) for t in (q0, k0, v0))
    ref = torch.matmul(torch.softmax(torch.matmul(qh, kh.transpose(-1, -2)) / d ** 0.5, -1), vh).transpose(1, 2).reshape(B * Sq, H * d)
    refg = torch.autograd.grad(ref, [qh, kh, vh], do.double())
    tol = 5e-5 if mode == 'tf32x3' else 5e-3        # tests/test_ops_gpu.py::test_attention_tensor_core
    for a, r, n in zip(new, refg, 'qkv'):
        r = r.transpose(1, 2).reshape(a.shape)
        assert rel(a, r) < tol, '%s %s d%s: rel %.3e vs fp64' % (what, mode, n, rel(a, r))


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('M,N,K,ldx', [(4000, 256, 320, 384), (8100, 96, 160, 256), (20200, 512, 192, 196)])
def test_linear_dgrad_transposed_tail_rows_and_accumulate(lib, mode, M, N, K, ldx):
    """K % 128 != 0 and M % 128 != 0: the transposed tile's rows beyond K and columns beyond M are never stored -- the columns of a padded dX
    row beyond K keep their values -- and accumulate adds onto the existing dX."""
    _, call = lib
    g = torch.Generator().manual_seed(M + N + K + ldx)
    dy = torch.randn(M, N, generator=g).to(DEV)
    w = torch.randn(N, K, generator=g).to(DEV)
    dx0 = torch.randn(M + 1, ldx, generator=g).to(DEV)       # one row more than M: never written either

    def dgrad(acc):
        def fn():
            dx = dx0.clone()
            call('rih_linear_dgrad', ctypes.c_void_p(dy.data_ptr()), N, ctypes.c_void_p(w.data_ptr()), K, ctypes.c_void_p(dx.data_ptr()), ldx,
                 M, N, K, acc, 0, None)
            return dx
        return fn
    t_launches(call)
    store = run(lib, mode, mode, NEW, dgrad(0))
    accd = run(lib, mode, mode, NEW, dgrad(1))
    assert t_launches(call) == 2, 'not on the transposed form'
    for out in (store, accd):
        assert torch.equal(out[:, K:], dx0[:, K:]) and torch.equal(out[M:], dx0[M:]), 'elements outside dX[:M, :K] were written'
    exact = dy.double() @ w.double()
    assert rel(store[:M, :K], exact) < SIMT_TOL[mode], 'rel %.3e vs fp64' % rel(store[:M, :K], exact)
    assert rel(accd[:M, :K], dx0[:M, :K] + store[:M, :K]) < 1e-6, 'accumulate does not add onto dX'
