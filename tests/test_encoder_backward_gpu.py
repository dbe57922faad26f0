"""Train-mode forward and backward of the ResNet-50 encoder in the arithmetic bench.py runs, against fp64 with emulated TF32 operands.

Reference (section 0): every convolution of the fp64 reference multiplies the operands the tensor cores see and accumulates in fp64.
'tf32' / 'tf32c' drop the low 13 mantissa bits of both operands (the hardware's truncation), 'tf32c' then multiplies the product by
float32(1.000705) (the epilogue's compensation of the truncation bias), 'tf32rn' rounds them as split_tf32 does ((bits + 0x1000) &
0xFFFFE000: nearest, ties away from zero), 'tf32x3' and 'simt' are plain fp64.  Forward, input gradient and weight gradient each take the
operands of their own product (wgrad: emulated dY and emulated X).  A pass that does not run on the tensor cores in the kernel (1x1
gradients of outputs whose width is not a multiple of 4, convolutions whose geometry the implicit GEMM does not take, stride-2 input
gradients accumulated onto an alias, the 3-channel stem when the image needs a gradient) is exact fp32 there and plain fp64 here.  So
the kernel differs from the reference only by the order and rounding of its fp32 accumulation, and a missing or doubled 1.000705
(7e-4 relative) is 100x over the tolerances below.

  1. the BatchNorm node (ops.batchnorm) against fp64 F.batch_norm: every combination of training / eval, relu, residual, mask_input,
     statistics passed in / computed by rih_bn_colstats, num_batches_tracked and flat gradient targets for gamma and beta; C from 4 to
     2048, M from 63 (one partial block of rows) to 64^3 (the grid-stride row loop), a row stride wider than C; a residual ReLU
     BatchNorm whose x needs no gradient (its ReLU gate must still include the residual); channels with |mean| up to 30 std;
  2. fused BatchNorm statistics of every producer (conv2d 1x1 / 3x3 / stride 2 with direct stride 2 on and off, stem_conv, the im2col
     stem GEMM) in all five arithmetics, against fp64 column sums of the stored output, including a partial last row tile, Cout 64 / 160
     / 2048, a stream capped to 2 CTAs (one CTA flushes across column blocks) and the fall-backs to rih_bn_colstats;
  3. the encoder's convolution products (forward, dgrad, wgrad) at batch 3 and 64 against section 0, with alias accumulation and
     registered flat weight-gradient targets; the negative control: 'tf32' kernels against the 'tf32c' emulation must miss;
  4. blocks in train mode (the three stem forms + max-pool, bottlenecks, a resnet18 basic block, the aux decoder's stages, a resnet_mid
     level) in 'simt', 'tf32x3' and the bench arithmetic, with and without an input gradient and flat gradient targets;
  5. the whole ResNetSimple (trunk + both aux decoders) in the bench arithmetic at batch 4 and 16, and in 'simt' at batch 4 as the
     conditioning baseline.

Errors are max |ours - ref| / max |ref| per tensor unless stated.  Tolerances are about 4x the worst error measured on an H100 80GB HBM3
(700 W power limit), given in brackets:

  1. BatchNorm node:   outputs / gradients 1e-6 [2.1e-7]; running statistics 6e-7 [1.6e-7]; num_batches_tracked exact (+1 per training
                       call).  |mean| / std up to 30 with fused statistics: derived bound (test_batchnorm_large_mean_statistics_bound),
                       measured at 0.05 of it (3.8e-6 at |mean| / std = 26); with rih_bn_colstats (fp64 per element) 3.1e-7.
  2. fused statistics: 1e-6 of sum |y| and of sum y^2 per column (stated bound) [8.9e-8].
  3. products:         'tf32c' 5e-5 [1.3e-5], 'tf32rn' 5e-5 [1.2e-5], 'tf32' 5e-5 [1.6e-6], 'tf32x3' (plain fp64) 1.5e-4 [3.6e-5]; the
                       error grows with the reduction length (worst: y of the 3x3 / 2 512-channel convolution, K = 4608), so the H100
                       behaves as truncation (or nearest rounding) of the operands plus fp32 accumulation.  Negative control: 'tf32'
                       kernels against the 'tf32c' emulation measure 7.05e-4 in y, dx and dw, 14x the tolerance.
  4. blocks:           max-norm 'simt' 1e-5 [2.2e-6], 'tf32x3' 1.2e-4 [2.6e-5], bench 1.5e-3 [3.6e-4].  Inside a chain the two sides'
                       operands differ in their last fp32 bits, and TF32 rounding turns a last-bit difference that crosses a rounding
                       boundary into a 2^-11 one, hence bench > product level.  Bottlenecks and the basic block carry ReLU gates between
                       convolutions; off 'simt' (and for the identity bottleneck in 'simt' too) gate flips dominate the max-norm (up to
                       1.2e-1), so they assert the Frobenius norm: 3e-2 [7.1e-3]; both norms are printed.
  5. whole encoder:    the randomly initialised 53-convolution trunk with two 4-stage decoders amplifies last-bit differences:
                       'simt' (exact fp32) outputs and running statistics 1.5e-3 [3.3e-4], gradients 0.5 [1.1e-1]; bench (N = 4, 16)
                       outputs 0.6 [1.5e-1], gradients 3 [7.9e-1] -- this case guards against gross errors only; sections 1-4 carry
                       the precision.
"""
import contextlib
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False

DEV = 'cuda'
F64 = torch.float64
U32 = 2.0 ** -24                                        # unit round-off of fp32
TF32C_SCALE = float(np.float32(1.000705))
BN_TOL, BN_RUN_TOL = 1e-6, 6e-7
STATS_TOL = 1e-6
CONV_TOL = {'tf32c': 5e-5, 'tf32rn': 5e-5, 'tf32': 5e-5, 'tf32x3': 1.5e-4}
BLOCK_TOL = {'simt': 1e-5, 'tf32x3': 1.2e-4, 'bench': 1.5e-3}
GATED_BLOCKS, GATED_FROB_TOL = ('layer1[0]', 'layer2[0]', 'identity layer1[1]', 'layer4[-1]', 'resnet18 basic'), 3e-2
NET_TOL = {('simt', 4): (1.5e-3, 0.5), ('bench', 4): (0.6, 3.0), ('bench', 16): (0.6, 3.0)}     # (outputs and running statistics, gradients)
ARITH = {'simt': ('simt', 'simt'), 'tf32x3': ('tf32x3', 'tf32x3'), 'bench': ('tf32c', 'tf32x3')}


def rel(a, b, scale=None):
    a, b = a.detach().to(F64), b.detach().to(F64)
    assert a.shape == b.shape, (a.shape, b.shape)
    s = b.abs().max() if scale is None else scale
    return float((a - b).abs().max() / torch.as_tensor(s, dtype=F64).clamp_min(1e-30))


def frob(a, b):
    a, b = a.detach().to(F64), b.detach().to(F64)
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def report(tag, errs, tol):
    """Print every measured error, then fail on the ones at or above the tolerance."""
    print('%s: %s' % (tag, ', '.join('%s %.2e' % kv for kv in errs.items())))
    bad = {k: '%.2e' % e for k, e in errs.items() if not e < tol}
    assert not bad, '%s: over the tolerance %.1e: %s' % (tag, tol, bad)


def randn(*shape, gen, scale=1.0, grad=False):
    return (torch.randn(*shape, generator=gen) * scale).to(DEV).requires_grad_(grad)


def f64_leaf(t, grad=True):
    return t.detach().to(F64).requires_grad_(grad)


def nchw(rows, N, H, C=None):
    return rows.reshape(N, H, H, rows.shape[1] if C is None else C).permute(0, 3, 1, 2)


def rows_of(t):
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


@pytest.fixture(scope='module')
def ops():
    from renderih_b200 import ops as o
    return o


CAPPED = []          # streams this module capped with rih_set_stream_cta_limit


@pytest.fixture(autouse=True)
def _restore_globals(ops):
    """Every global a test here changes: GEMM arithmetic, FUSED switches, side-stream weight gradients, registered gradient targets, CTA
    limits, direct stride 2 and the launch trace."""
    from renderih_b200 import _lib
    mode, fused, wg = dict(ops.MODE), dict(ops.FUSED), ops._WG['enabled']
    try:
        yield
    finally:
        _lib.TRACE = None
        ops.set_gemm_mode(mode['conv'], mode['linear'])
        ops.FUSED.clear(); ops.FUSED.update(fused)
        ops._WG['enabled'] = wg
        ops.clear_grad_targets()
        while CAPPED:
            ops.call('rih_set_stream_cta_limit', CAPPED.pop().cuda_stream, 0)
        ops.call('rih_set_s2_direct', 1)


@contextlib.contextmanager
def arithmetic(ops, conv, linear=None):
    ops.set_gemm_mode(conv, linear or conv)
    try:
        yield
    finally:
        ops.set_gemm_mode('simt', 'simt')


def launch_counts(ops, reset=True):
    """(TMA-store tensor-core launches, per-thread-store tensor-core launches, SIMT launches, transposed dgrad launches) since the last reset"""
    out, t = (ctypes.c_longlong * 3)(), ctypes.c_longlong(0)
    ops.call('rih_gemm_launch_counts', out, int(reset))
    ops.call('rih_gemm_dgrad_t_launches', ctypes.byref(t), int(reset))
    return tuple(out) + (t.value,)


def flat_params(params, gen):
    """train.FlatParams over `params`, its gradient prefilled with random values -> (FlatParams, prefill)."""
    from renderih_b200.train import FlatParams
    fp = FlatParams(params)
    prefill = torch.randn(fp.numel, generator=gen).to(DEV)
    fp.grad.copy_(prefill)
    return fp, prefill


def flat_deltas(fp, prefill):
    """{param: gradient accumulated on top of the prefill}; also checks that every .grad is still its view of the flat buffer."""
    delta = fp.grad.to(F64) - prefill.to(F64)
    out = {}
    for p, off in zip(fp.params, fp.offsets):
        assert p.grad is not None and p.grad.data_ptr() == fp.grad.data_ptr() + 4 * off, 'gradient left the flat buffer'
        out[p] = torch.as_strided(delta, p.shape, p.stride(), off)
    return out


# ============================================================================ 0. fp64 reference with emulated TF32 operands
def tf32_operand(t, arith):
    """The fp32 value of `t` as a tensor core multiplies it in arithmetic `arith`, as fp64 ('exact': `t` itself)."""
    if arith == 'exact':
        return t.detach()
    t = t.detach().to(torch.float32).contiguous()
    if arith in ('tf32', 'tf32c'):
        t = (t.view(torch.int32) & -8192).view(torch.float32)               # & 0xFFFFE000: truncation
    elif arith == 'tf32rn':
        t = ((t.view(torch.int32) + 0x1000) & -8192).view(torch.float32)    # split_tf32: nearest, ties away from zero
    return t.to(F64)


def acc_scale(arith):
    return TF32C_SCALE if arith == 'tf32c' else 1.0


class EmulConv(torch.autograd.Function):
    """fp64 conv2d whose forward, input-gradient and weight-gradient products each take emulated operands (arith = per-pass arithmetic)."""

    @staticmethod
    def forward(ctx, x, w, b, stride, pad, arith):
        ctx.save_for_backward(x, w)
        ctx.cfg = (stride, pad, arith)
        y = F.conv2d(tf32_operand(x, arith[0]), tf32_operand(w, arith[0]), None, stride, pad) * acc_scale(arith[0])
        return y if b is None else y + b.view(1, -1, 1, 1)

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        stride, pad, arith = ctx.cfg
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = torch.nn.grad.conv2d_input(x.shape, tf32_operand(w, arith[1]), tf32_operand(dy, arith[1]), stride, pad) * acc_scale(arith[1])
        if ctx.needs_input_grad[1]:
            dw = torch.nn.grad.conv2d_weight(tf32_operand(x, arith[2]), w.shape, tf32_operand(dy, arith[2]), stride, pad) * acc_scale(arith[2])
        if ctx.needs_input_grad[2]:
            db = dy.sum((0, 2, 3))
        return dx, dw, db, None, None, None


def conv_on_tc(ops, mode, N, H, Cin, Cout, k, stride, pad, which, accumulate=False, img_grad=False):
    """True when pass `which` (0 fwd, 1 dgrad, 2 wgrad) of this convolution runs on the tensor cores in conv mode `mode`, False when it
    takes the SIMT kernel (the dispatch of csrc/gemm_api.cu)."""
    if mode == 'simt':
        return False
    if Cin == 3:            # the RGB stem: stem_conv / the im2col GEMM on the tensor cores, _conv_bn's SIMT convolution when the image needs a gradient
        return not img_grad
    if k == 1 and stride == 1 and pad == 0:    # dense GEMM: 16-byte aligned rows, and the weight gradient needs 16 output channels
        return Cin % 4 == 0 and (which == 0 or Cout % 4 == 0) and (which != 2 or Cout >= 16)
    if which == 1 and stride == 2 and accumulate:
        return False
    Ho = (H + 2 * pad - k) // stride + 1
    geom = (ctypes.c_int * 13)(N, H, H, Cin, Ho, Ho, Cout, k, k, stride, pad, Cin, Cout)
    sup = ctypes.c_int(0)
    prev = dict(ops.MODE)
    ops.set_gemm_mode('tf32', prev['linear'])
    try:
        ops.call('rih_conv2d_tc_supported', geom, which, ctypes.byref(sup))
    finally:
        ops.set_gemm_mode(prev['conv'], prev['linear'])
    return bool(sup.value)


def conv_arith(ops, mode, *geom, **kw):
    """Emulated arithmetic of that pass: `mode` on the tensor cores except 3xTF32 (fp32-faithful), 'exact' (plain fp64) otherwise."""
    return mode if mode not in ('simt', 'tf32x3') and conv_on_tc(ops, mode, *geom, **kw) else 'exact'


def make_conv(ops, mode, img_grad=False):
    """A drop-in for F.conv2d (the `conv=` argument of oracle.model_ref) computing in the emulated arithmetic of conv mode `mode`."""
    def conv(x, w, b=None, stride=1, padding=0):
        N, Cin, H, _ = x.shape
        Cout, k = w.shape[0], w.shape[-1]
        arith = tuple(conv_arith(ops, mode, N, H, Cin, Cout, k, stride, padding, which, img_grad=img_grad) for which in range(3))
        return EmulConv.apply(x, w, b, stride, padding, arith)
    return conv


# ============================================================================ 1. the BatchNorm node
def bn_case(ops, M, C, training=True, relu=True, res=True, mask_input=False, stats_in=False, tracked=True, param_acc=False, ld=None,
            x_grad=True, seed=0):
    """One forward + backward of ops.batchnorm and of fp64 F.batch_norm on the same values -> errors.  The ReLU gate of the reference's
    backward is the kernel's own (y > 0), so that gradients compare element by element."""
    gen = torch.Generator().manual_seed(seed + M + C)
    ld = ld or C
    xb = randn(M, ld, gen=gen, scale=1.5)
    xb = xb + randn(1, ld, gen=gen)                       # per-channel offsets
    if mask_input:                                        # Conv -> ReLU -> BN: x is a ReLU output
        xb = xb.clamp_min(0)
    x = xb[:, :C].detach().requires_grad_(x_grad) if ld == C else xb.detach().requires_grad_(x_grad)[:, :C]
    leaf_x = x if ld == C else x._base
    gamma = (1 + randn(C, gen=gen, scale=0.3)).requires_grad_(True)
    beta = randn(C, gen=gen, scale=0.3, grad=True)
    rm, rv = randn(C, gen=gen, scale=0.2), 0.5 + torch.rand(C, generator=gen).to(DEV)
    r = None
    if res:
        rb = randn(M, ld, gen=gen)
        r = rb[:, :C].detach().requires_grad_(True) if ld == C else rb.requires_grad_(True)[:, :C]
    trk = torch.tensor([5], dtype=torch.int64, device=DEV) if tracked else None
    stats = None
    if stats_in:
        xd = x.detach().to(F64)
        stats = torch.cat([xd.sum(0), (xd * xd).sum(0)])
    rm_d, rv_d = rm.to(F64), rv.to(F64)
    fp = None
    if param_acc:
        fp, prefill = flat_params([gamma, beta], gen)
    cot = randn(M, C, gen=gen)
    y = ops.batchnorm(x, gamma, beta, rm, rv, res=r, training=training, relu=relu, mask_input=mask_input, stats=stats, tracked=trk)
    (y * cot).sum().backward()
    ops.clear_grad_targets()

    xd, gd, bd = f64_leaf(x), f64_leaf(gamma), f64_leaf(beta)
    rd = f64_leaf(r) if res else None
    z = F.batch_norm(xd, rm_d, rv_d, gd, bd, training, 0.1, 1e-5)
    if res:
        z = z + rd
    errs = {'out': rel(y, z.clamp_min(0) if relu else z)}
    zg = z * (y.detach() > 0) if relu else z
    (zg * cot.to(F64)).sum().backward()
    if x_grad:
        dx_ref = xd.grad * (x.detach() > 0) if mask_input else xd.grad
        dxo = leaf_x.grad if ld == C else leaf_x.grad[:, :C]
        errs['dx'] = rel(dxo, dx_ref)
        if ld != C:
            assert float(leaf_x.grad[:, C:].abs().max()) == 0.0, 'gradient outside the strided view'
    else:
        assert leaf_x.grad is None
    if res:
        errs['dres'] = rel(r.grad if ld == C else r._base.grad[:, :C], rd.grad)
    if param_acc:
        dp = flat_deltas(fp, prefill)
        dg, db = dp[gamma], dp[beta]
    else:
        dg, db = gamma.grad, beta.grad
    errs['dgamma'], errs['dbeta'] = rel(dg, gd.grad), rel(db, bd.grad)
    run = {'running_mean': rel(rm, rm_d), 'running_var': rel(rv, rv_d)}
    if tracked:      # exactly +1 per training call: 0 when right, 1 when not
        run['num_batches_tracked'] = float(int(trk.item()) != (6 if training else 5))
    return errs, run


BN_FLAGS = [(tr, relu, res, mi, si, trk, pa) for tr in (True, False) for relu in (True, False) for res in (True, False)
            for mi in (True, False) for si in ((True, False) if tr else (False,)) for trk in (True, False) for pa in (True, False)]


@pytest.mark.parametrize('training,relu,res,mask_input,stats_in,tracked,param_acc', BN_FLAGS,
                         ids=['%s-relu%d-res%d-mask%d-stats%d-trk%d-acc%d' % ((('train' if f[0] else 'eval'),) + tuple(map(int, f[1:])))
                              for f in BN_FLAGS])
def test_batchnorm_node_flags(ops, training, relu, res, mask_input, stats_in, tracked, param_acc):
    """Every combination of the node's switches at M = 4097 (a partial block of rows), C = 100."""
    errs, run = bn_case(ops, 4097, 100, training, relu, res, mask_input, stats_in, tracked, param_acc)
    report('bn flags', errs, BN_TOL)
    report('bn flags running stats', run, BN_RUN_TOL)


BN_SHAPES = [(63, 4, None), (63, 36, None), (63, 2048, None), (192, 64, None), (192, 100, None), (192, 2048, None), (4097, 36, None),
             (4097, 2048, None), (64 ** 3, 4, None), (64 ** 3, 36, None), (64 ** 3, 64, None), (64 ** 3, 100, None),
             (4097, 100, 108), (64 ** 3, 64, 72)]


@pytest.mark.parametrize('M,C,ld', BN_SHAPES)
@pytest.mark.parametrize('training', [True, False], ids=['train', 'eval'])
def test_batchnorm_node_shapes(ops, M, C, ld, training):
    """The residual ReLU node of a bottleneck (and its eval form) at every shape; ld = a row stride wider than C (x and res)."""
    errs, run = bn_case(ops, M, C, training, ld=ld)
    report('bn M=%d C=%d ld=%s %s' % (M, C, ld, 'train' if training else 'eval'), errs, BN_TOL)
    report('bn running stats', run, BN_RUN_TOL)


@pytest.mark.parametrize('param_acc', [False, True])
@pytest.mark.parametrize('training', [True, False], ids=['train', 'eval'])
def test_batchnorm_residual_relu_gate_without_input_gradient(ops, training, param_acc):
    """A residual ReLU BatchNorm whose x needs no gradient (its convolution frozen) while res, gamma and beta do: the backward must gate
    with relu(bn(x) + res), not with relu(bn(x)).  Before the fix the gate was rebuilt from x alone (the mask was recorded only when x
    needed a gradient); dres measured 1.0 and dgamma / dbeta 0.2-0.5 relative errors."""
    errs, run = bn_case(ops, 4097, 64, training, param_acc=param_acc, x_grad=False)
    report('bn residual gate, x without gradient', errs, BN_TOL)


def test_batchnorm_large_mean_statistics_bound(ops):
    """Channels with |mean| / std up to 30, statistics from the fused GEMM epilogue (fp32 partial sums over 32 rows, fp64 across them).

    Bound: each column's sum of squares is a sum of fp32 products x^2 (error u) added in fp32 over 32 rows (5 levels, all terms positive):
    relative error <= 6u; the column sum likewise <= 5u (|mean| >> std: nearly all terms of one sign), so mean^2 <= 10u.  The variance
    E[x^2] - mean^2 is then off by <= 16u (mean^2 + var), i.e. 16u (1 + rho^2) relative, rho = |mean| / std; rstd by half of that.  The
    normalised output (x - mean) * rstd is off by 8u (1 + rho^2) |xhat| from rstd, 6u rho from the mean and its fp32 rounding, and a few
    u from the fp32 arithmetic of the normalisation: bound(rho) = 8u (1 + rho^2) + 6u rho + 8u relative to the channel's max |xhat|.
    dx = gamma rstd (g - mean(g) - xhat mean(g xhat)) carries rstd three times: 3 bound(rho).  Asserted per channel; the
    rih_bn_colstats path (fp64 per element) is held to the node tolerance."""
    M, C, K = 8192, 64, 32
    gen = torch.Generator().manual_seed(77)
    A = torch.cat([torch.randn(M, K - 1, generator=gen), torch.ones(M, 1)], 1).to(DEV)
    W = torch.randn(C, K, generator=gen) * (K - 1) ** -0.5
    rho = torch.linspace(0, 30, C)
    W[:, K - 1] = rho * W[:, :K - 1].norm(dim=1) * torch.where(torch.arange(C) % 2 == 0, 1.0, -1.0)
    W = W.to(DEV)
    gamma, beta = torch.ones(C, device=DEV, requires_grad=True), torch.zeros(C, device=DEV, requires_grad=True)
    cot = randn(M, C, gen=gen)
    results = {}
    for path in ('fused', 'colstats'):
        stats = torch.empty(2 * C, device=DEV, dtype=F64)
        with arithmetic(ops, 'tf32x3'):
            launch_counts(ops)
            y = ops.linear(A, W, None, stats=stats if path == 'fused' else None, as_conv=True)
            n = launch_counts(ops)
        assert n[0] == 1 and n[1] == n[2] == 0, n
        x = y.detach().requires_grad_(True)
        rm, rv = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)
        out = ops.batchnorm(x, gamma, beta, rm, rv, training=True, stats=stats if path == 'fused' else None)
        (out * cot).sum().backward()
        xd = f64_leaf(x)
        ref = F.batch_norm(xd, None, None, gamma.detach().to(F64), beta.detach().to(F64), True, 0.1, 1e-5)
        (ref * cot.to(F64)).sum().backward()
        e_out = (out.detach().to(F64) - ref.detach()).abs().max(0).values / ref.detach().abs().max(0).values
        e_dx = (x.grad.to(F64) - xd.grad).abs().max(0).values / xd.grad.abs().max(0).values
        results[path] = (e_out, e_dx)
        gamma.grad = beta.grad = None
    xs = y.detach().to(F64)
    rho_m = (xs.mean(0).abs() / xs.std(0)).cpu()
    bound = (8 * U32 * (1 + rho_m ** 2) + 6 * U32 * rho_m + 8 * U32)
    e_out, e_dx = (t.cpu() for t in results['fused'])
    print('bn |mean|/std up to %.1f, fused statistics: worst out error / bound %.2f (out %.2e at rho %.1f, bound %.2e), '
          'worst dx error / 3 bound %.2f (dx %.2e)' % (float(rho_m.max()), float((e_out / bound).max()), float(e_out.max()),
                                                      float(rho_m[e_out.argmax()]), float(bound[e_out.argmax()]),
                                                      float((e_dx / (3 * bound)).max()), float(e_dx.max())))
    assert bool((e_out <= bound).all()), ('out over the derived bound', (e_out / bound).max())
    assert bool((e_dx <= 3 * bound).all()), ('dx over the derived bound', (e_dx / (3 * bound)).max())
    report('bn |mean|/std up to 30, rih_bn_colstats', {'out': float(results['colstats'][0].max()), 'dx': float(results['colstats'][1].max())},
           BN_TOL)


# ============================================================================ 2. fused BatchNorm statistics of every producer
def weight(gen, Cout, Cin, k):
    return randn(Cout, Cin, k, k, gen=gen, scale=(Cin * k * k) ** -0.5).contiguous(memory_format=torch.channels_last)


# name: (producer, expected route in a tensor-core mode: 'fused' = statistics in the TMA-store epilogue, 'per_thread' = per-thread-store
# epilogue + rih_bn_colstats, 'simt' = SIMT kernel + rih_bn_colstats)
STATS_CASES = {
    'conv1x1 64->64 M=675': 'fused',                     # partial last row tile
    'conv1x1 64->160 M=1922 capped 2 CTAs': 'fused',      # partial tile, two column blocks walked by each of 2 persistent CTAs
    'conv3x3 64->160 M=768': 'fused',
    'conv3x3/2 64->64 direct': 'fused',
    'conv3x3/2 64->64 copy-based': 'fused',
    'conv1x1/2 1024->2048 M=128': 'fused',
    'conv1x1/2 1024->2048 M=192': 'simt',                # M % 128 != 0: the implicit GEMM does not take it
    'conv1x1 64->42': 'per_thread',                      # rows of 42 floats: no TMA store
    'stem_conv': 'fused',
    'im2col stem M=1922': 'fused',
}


def stats_producer(ops, name, gen):
    """-> (y [rows, C] as stored, fp64 statistics the producer wrote)."""
    def conv(N, H, Cin, Cout, k, stride):
        x = randn(N * H * H, Cin, gen=gen)
        stats = torch.full((2 * Cout,), 7.0, device=DEV, dtype=F64)
        y = ops.conv2d(x, weight(gen, Cout, Cin, k), None, N, H, H, stride=stride, pad=k // 2, stats=stats)
        return y, stats
    if name == 'conv1x1 64->64 M=675':
        return conv(3, 15, 64, 64, 1, 1)
    if name == 'conv1x1 64->160 M=1922 capped 2 CTAs':
        st = torch.cuda.Stream()
        CAPPED.append(st)
        ops.call('rih_set_stream_cta_limit', st.cuda_stream, 2)
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            out = conv(2, 31, 64, 160, 1, 1)
        torch.cuda.current_stream().wait_stream(st)
        return out
    if name == 'conv3x3 64->160 M=768':
        return conv(3, 16, 64, 160, 3, 1)
    if name.startswith('conv3x3/2'):
        ops.call('rih_set_s2_direct', int('direct' in name))
        return conv(2, 32, 64, 64, 3, 2)
    if name == 'conv1x1/2 1024->2048 M=128':
        return conv(2, 16, 1024, 2048, 1, 2)
    if name == 'conv1x1/2 1024->2048 M=192':
        return conv(3, 16, 1024, 2048, 1, 2)
    if name == 'conv1x1 64->42':
        return conv(2, 16, 64, 42, 1, 1)
    if name == 'stem_conv':
        stats = torch.full((128,), 7.0, device=DEV, dtype=F64)
        img = randn(2, 3, 256, 256, gen=gen)
        return ops.stem_conv(img, weight(gen, 64, 3, 7), stats), stats
    # ResNetSimple._stem: im2col to 160-wide rows, then a dense GEMM in the convolution arithmetic
    N, H = 2, 62
    img = randn(N, 3, H, H, gen=gen)
    A = ops.im2col(ops.nchw_to_nhwc(img), N, H, H, 7, 7, 2, 3, 160)
    w2d = F.pad(weight(gen, 64, 3, 7).permute(0, 2, 3, 1).reshape(64, 147), (0, 13))
    stats = torch.full((128,), 7.0, device=DEV, dtype=F64)
    return ops.linear(A, w2d, None, stats=stats, as_conv=True), stats


@pytest.mark.parametrize('mode', ['simt', 'tf32', 'tf32rn', 'tf32c', 'tf32x3'])
@pytest.mark.parametrize('name', list(STATS_CASES))
def test_fused_batchnorm_statistics(ops, name, mode):
    """The statistics a producer hands the following BatchNorm against fp64 column sums and sums of squares of the output it stored:
    |error| <= 1e-6 of sum |y| and of sum y^2 per column.  Asserts the route (fused epilogue / fall-back pass) through the launch counts."""
    if name == 'stem_conv' and mode == 'simt':
        pytest.skip('stem_conv needs a tensor-core convolution mode')
    gen = torch.Generator().manual_seed(len(name))
    with arithmetic(ops, mode):
        launch_counts(ops)
        y, stats = stats_producer(ops, name, gen)
        n = launch_counts(ops)
    torch.cuda.synchronize()
    route = 'simt' if mode == 'simt' else STATS_CASES[name]
    if route == 'fused':
        assert n[0] >= 1 and n[1] == 0 and n[2] == 0, n
    elif route == 'per_thread':
        assert n[1] >= 1 and n[2] == 0, n
    else:
        assert n[2] >= 1 and n[0] == n[1] == 0, n
    yd = y.detach().to(F64)
    C = yd.shape[1]
    errs = {'sum': float(((stats[:C] - yd.sum(0)).abs() / yd.abs().sum(0).clamp_min(1e-30)).max()),
            'sum of squares': float(((stats[C:] - (yd * yd).sum(0)).abs() / (yd * yd).sum(0).clamp_min(1e-30)).max())}
    report('stats %s %s' % (name, mode), errs, STATS_TOL)


# ============================================================================ 3. convolution products in the emulated arithmetic
# (name, Cin, Cout, H, k, stride): the encoder's geometries; 'up' = the aux decoder's 3x3 after bilinear2x (input H, convolved at 2H)
CONV_CASES = [('1x1 256->64', 256, 64, 64, 1, 1), ('1x1 64->256', 64, 256, 64, 1, 1), ('1x1/2 1024->2048', 1024, 2048, 16, 1, 2),
              ('3x3 64', 64, 64, 64, 3, 1), ('3x3/2 128', 128, 128, 64, 3, 2), ('3x3/2 512', 512, 512, 16, 3, 2),
              ('3x3 256', 256, 256, 16, 3, 1), ('up 3x3 128', 128, 128, 8, 3, 1)]


def conv_product_case(ops, mode, ref_mode, name, Cin, Cout, H, k, stride, N, variant):
    """Forward, dgrad and wgrad of ops.conv2d in conv mode `mode` against the section-0 reference in `ref_mode`.  variant 'alias_flat':
    the input is also consumed through the alias output (dgrad accumulates onto that gradient) and the weight gradient goes to a
    registered flat target with side-stream weight gradients.  -> (errors, launch counts fwd, launch counts bwd, predicted arithmetic)"""
    gen = torch.Generator().manual_seed(Cin + Cout + H + N)
    up = name.startswith('up')
    x0 = randn(N * H * H, Cin, gen=gen, grad=True)
    w = weight(gen, Cout, Cin, k).requires_grad_(True)
    alias = variant == 'alias_flat'
    fp = None
    if alias:
        fp, prefill = flat_params([w], gen)
    Hc = 2 * H if up else H
    Ho = (Hc + 2 * (k // 2) - k) // stride + 1
    cot = randn(N * Ho * Ho, Cout, gen=gen)
    cot_a = randn(N * Hc * Hc, Cin, gen=gen) if alias else None
    with arithmetic(ops, mode, 'simt'):
        launch_counts(ops)
        xin = ops.bilinear2x(x0, N, H, H) if up else x0
        y = ops.conv2d(xin, w, None, N, Hc, Hc, stride=stride, pad=k // 2, alias_input=alias)
        if alias:
            y, xa = y
        n_fwd = launch_counts(ops)
        loss = (y * cot).sum() + ((xa * cot_a).sum() if alias else 0)
        loss.backward()
        n_bwd = launch_counts(ops)
    ops.clear_grad_targets()
    tc = tuple(conv_on_tc(ops, mode, N, Hc, Cin, Cout, k, stride, k // 2, which, accumulate=alias) for which in range(3))
    arith = tuple(conv_arith(ops, ref_mode, N, Hc, Cin, Cout, k, stride, k // 2, which, accumulate=alias) for which in range(3))
    xd, wd = f64_leaf(x0), f64_leaf(w)
    xr = nchw(xd, N, H)
    if up:      # the product's operand is the bilinear2x output the kernel multiplied (its gradient flows through F.interpolate): a last-bit
        xr = F.interpolate(xr, scale_factor=2, mode='bilinear', align_corners=True)     # difference would move the TF32 rounding of it
        xr = xr + (nchw(xin.detach().to(F64), N, Hc) - xr).detach()
    yd = EmulConv.apply(xr, wd, None, stride, k // 2, arith)
    loss_d = (rows_of(yd) * cot.to(F64)).sum()
    if alias:
        loss_d = loss_d + (rows_of(xr) * cot_a.to(F64)).sum()
    loss_d.backward()
    errs = {'y': rel(y, rows_of(yd)), 'dx': rel(x0.grad, xd.grad),
            'dw': rel(flat_deltas(fp, prefill)[w] if alias else w.grad, wd.grad)}
    return errs, route_mismatch(n_fwd, n_bwd, tc, Cin), arith


def route_mismatch(n_fwd, n_bwd, tc, Cin):
    """'' when the tensor-core / SIMT route of every pass is the one the reference assumed (one SIMT launch per SIMT pass, transposed
    input gradients dX^T = W^T dY^T exactly when a tensor-core dgrad has at least 128 input channels), else what differs."""
    ok = (n_fwd[2] == 0 and n_fwd[0] + n_fwd[1] >= 1) if tc[0] else (n_fwd[2] == 1 and n_fwd[0] + n_fwd[1] == 0)
    ok = ok and n_bwd[2] == sum(not t for t in tc[1:])
    if tc[1]:
        ok = ok and (n_bwd[3] > 0) == (Cin >= 128)
    return '' if ok else 'launches fwd %s bwd %s, expected tensor cores %s' % (n_fwd, n_bwd, tc)


@pytest.mark.parametrize('variant', ['plain', 'alias_flat'])
@pytest.mark.parametrize('N', [3, 64])
@pytest.mark.parametrize('name,Cin,Cout,H,k,stride', CONV_CASES, ids=[c[0] for c in CONV_CASES])
@pytest.mark.parametrize('mode', ['tf32c', 'tf32rn', 'tf32x3'])
def test_conv_products_match_emulated_fp64(ops, mode, name, Cin, Cout, H, k, stride, N, variant):
    errs, routes, arith = conv_product_case(ops, mode, mode, name, Cin, Cout, H, k, stride, N, variant)
    if routes:
        print('conv %s %s N=%d %s: %s' % (name, mode, N, variant, routes))
    report('conv %s %s N=%d %s [%s]' % (name, mode, N, variant, '/'.join(arith)), errs, CONV_TOL[mode])
    assert not routes, routes


@pytest.mark.parametrize('name,Cin,Cout,H,k,stride', [CONV_CASES[0], CONV_CASES[3]], ids=[CONV_CASES[0][0], CONV_CASES[3][0]])
def test_conv_products_negative_control(ops, name, Cin, Cout, H, k, stride):
    """'tf32' kernels (truncation, no compensation) match the 'tf32' emulation to the tolerance but miss the 'tf32c' emulation by more
    than 5x it: the comparison sees a missing 1.000705."""
    errs, routes, arith = conv_product_case(ops, 'tf32', 'tf32', name, Cin, Cout, H, k, stride, 3, 'plain')
    assert not routes and arith == ('tf32',) * 3, (routes, arith)
    report('conv %s tf32 vs tf32 emulation' % name, errs, CONV_TOL['tf32'])
    errs, _, _ = conv_product_case(ops, 'tf32', 'tf32c', name, Cin, Cout, H, k, stride, 3, 'plain')
    print('conv %s tf32 kernels vs tf32c emulation: %s' % (name, ', '.join('%s %.2e' % kv for kv in errs.items())))
    assert all(e > 5 * CONV_TOL['tf32c'] for e in errs.values()), errs


@pytest.mark.parametrize('N', [3, 64])
@pytest.mark.parametrize('mode', ['tf32c', 'tf32rn', 'tf32x3'])
def test_stem_conv_products_match_emulated_fp64(ops, mode, N):
    """stem_conv (implicit GEMM, 7x7 / 2 over the 256 x 256 image) forward and rih_stem_conv_wgrad; the image has no gradient."""
    gen = torch.Generator().manual_seed(N)
    img = randn(N, 3, 256, 256, gen=gen)
    w = weight(gen, 64, 3, 7).requires_grad_(True)
    cot = randn(N * 128 * 128, 64, gen=gen)
    with arithmetic(ops, mode):
        assert ops.stem_supported(256, 256)
        with launch_trace() as calls:
            y = ops.stem_conv(img, w)
            (y * cot).sum().backward()
    names = [c for c, _ in calls]
    assert 'rih_stem_conv_fwd' in names and 'rih_stem_conv_wgrad' in names, names
    wd = f64_leaf(w)
    ar = 'exact' if mode == 'tf32x3' else mode
    yd = EmulConv.apply(img.to(F64), wd, None, 2, 3, (ar, ar, ar))
    (rows_of(yd) * cot.to(F64)).sum().backward()
    report('stem_conv %s N=%d' % (mode, N), {'y': rel(y, rows_of(yd)), 'dw': rel(w.grad, wd.grad)}, CONV_TOL[mode])


@contextlib.contextmanager
def launch_trace():
    from renderih_b200 import _lib
    _lib.TRACE = []
    calls = []
    try:
        yield calls
    finally:
        calls.extend((n, a) for n, a, _, _ in _lib.TRACE)
        _lib.TRACE = None


# ============================================================================ 4. blocks in train mode
def encoder(model_type='resnet50', seed=0):
    """A ResNetSimple with seeded weights, BatchNorm affine parameters and running statistics away from their defaults, train mode."""
    from renderih_b200.model import ResNetSimple
    torch.manual_seed(seed)
    enc = ResNetSimple(model_type, aux_heads=(model_type == 'resnet50'))
    gen = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for m in enc.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.weight.copy_(1 + 0.2 * torch.randn(m.num_features, generator=gen))
                m.bias.copy_(0.2 * torch.randn(m.num_features, generator=gen))
                m.running_mean.copy_(0.1 * torch.randn(m.num_features, generator=gen))
                m.running_var.copy_(0.5 + torch.rand(m.num_features, generator=gen))
    return enc.to(DEV).train()


@pytest.fixture(scope='module')
def enc50():
    return encoder('resnet50')


@pytest.fixture(scope='module')
def enc18():
    return encoder('resnet18')


def f64_state(module, prefix):
    """The module's parameters (fp64 leaves) and buffers (fp64 copies; running statistics are updated in place by the reference)."""
    sd = {}
    for k, v in module.state_dict().items():
        if not v.is_floating_point():
            continue
        sd[prefix + k] = v.detach().to(F64).clone()
    for k, p in module.named_parameters():
        sd[prefix + k].requires_grad_(True)
    return sd


def block_setup(ops, name, enc50, enc18, mode):
    """-> (module, input [rows or NCHW image], ours(x) -> rows, ref(x64, sd, conv) -> NCHW, N, Hout, sd prefix, needs the input in NCHW)"""
    from oracle import model_ref
    gen = torch.Generator().manual_seed(len(name))
    if name.startswith('stem'):
        form = name.split()[1]
        H = 128 if form == 'im2col' else 256
        N = 3
        img = randn(N, 3, H, H, gen=gen)
        r = torch.nn.ModuleDict({'conv1': enc50.resnet.conv1, 'bn1': enc50.resnet.bn1})

        def ref(x, sd, conv):
            y = F.relu(model_ref._bn(conv(x, sd['b.conv1.weight'], stride=2, padding=3), sd, 'b.bn1', True))
            return F.max_pool2d(y, 3, 2, 1)
        return r, img, lambda x: enc50.stem(x)[0], ref, N, H // 4, form == 'conv_bn'
    if name in ('layer1[0]', 'layer2[0]', 'identity layer1[1]', 'layer4[-1]'):
        r = enc50.resnet
        blk, N, H, stride, ds = {'layer1[0]': (r.layer1[0], 4, 64, 1, True), 'layer2[0]': (r.layer2[0], 4, 64, 2, True),
                                 'identity layer1[1]': (r.layer1[1], 4, 64, 1, False), 'layer4[-1]': (r.layer4[2], 3, 8, 1, False)}[name]
        x = randn(N * H * H, blk.conv1.in_channels, gen=gen, scale=0.7).clamp_min(0)     # a block input is a ReLU output
        return blk, x, lambda x: enc50._bottleneck(blk, x, N, H)[0], \
            lambda x, sd, conv: model_ref._bottleneck(x, sd, 'b', stride, ds, True, conv=conv), N, H // stride, False
    if name == 'resnet18 basic':
        blk, N, H = enc18.resnet.layer1[0], 4, 64
        x = randn(N * H * H, 64, gen=gen, scale=0.7).clamp_min(0)
        return blk, x, lambda x: enc18._basic(blk, x, N, H)[0], \
            lambda x, sd, conv: model_ref._basic_block(x, sd, 'b', True, conv=conv), N, H, False
    if name.startswith('decoder'):
        dec = enc50.hms_decoder
        i, H, Cin = (0, 8, 2048) if 'flat' in name else (1, 8, 128)
        N = 4
        x = randn(N * H * H, Cin, gen=gen, scale=0.7).clamp_min(0)
        seq = dec.models[i]
        cname, bname, pad = ('b.0', 'b.2', 0) if i == 0 else ('b.1', 'b.3', 1)

        def ref(x, sd, conv):
            if i:
                x = F.interpolate(x, scale_factor=2, mode='bilinear', align_corners=True)
            return model_ref._bn(F.relu(conv(x, sd[cname + '.weight'], padding=pad)), sd, bname, True)
        return seq, x, lambda x: dec.stage(i, x, N, H)[0], ref, N, H * (2 if i else 1), False
    # resnet_mid level 1: cat(hms fmap 128, dp fmap 128, trunk feature 1024) at 16 x 16 -> 1x1 -> ReLU -> BN
    from renderih_b200.model import resnet_mid
    torch.manual_seed(5)
    mid = resnet_mid('resnet50', in_fmapDim=(128, 128, 128, 128)).to(DEV).train()
    N, H = 4, 16
    parts = [randn(N * H * H, c, gen=gen, scale=0.7).clamp_min(0) for c in (128, 128, 1024)]
    x = torch.cat(parts, 1)

    def ours(x):
        hms, dp, img = x[:, :128], x[:, 128:256], x[:, 256:]
        return mid.level(1, [None, (img, H)], (hms, H), (dp, H), N)[0]
    seq = mid.convs[1]

    def ref(x, sd, conv):
        return model_ref._bn(F.relu(conv(x, sd['b.0.weight'])), sd, 'b.2', True)
    return seq, x, ours, ref, N, H, False


BLOCKS = ['stem igemm', 'stem im2col', 'stem conv_bn', 'layer1[0]', 'layer2[0]', 'identity layer1[1]', 'layer4[-1]', 'resnet18 basic',
          'decoder flat', 'decoder up', 'mid level']


@pytest.mark.parametrize('variant', ['input_grad', 'no_input_grad_flat'])
@pytest.mark.parametrize('arith', ['simt', 'tf32x3', 'bench'])
@pytest.mark.parametrize('name', BLOCKS)
def test_block_train_mode_matches_emulated_fp64(ops, enc50, enc18, name, arith, variant):
    """Output, input gradient, every parameter gradient and the running statistics of one block, train mode, against the fp64 reference
    with the block's convolutions emulated in the arithmetic that ran.  'input_grad': the input needs a gradient (alias outputs on);
    'no_input_grad_flat': it does not, and the block's parameters are re-homed into a FlatParams (direct weight-gradient targets)."""
    conv_mode = ARITH[arith][0]
    if name == 'stem igemm' and conv_mode == 'simt':
        pytest.skip('the implicit-GEMM stem needs a tensor-core convolution mode')
    if name == 'stem conv_bn' and variant != 'input_grad' or name in ('stem igemm', 'stem im2col') and variant == 'input_grad':
        pytest.skip('the stem form is chosen by whether the image needs a gradient')
    mod, x, ours, ref, N, Hout, img_grad = block_setup(ops, name, enc50, enc18, conv_mode)
    x = x.detach().requires_grad_(variant == 'input_grad')
    for p in mod.parameters():
        p.grad = None
    sd = f64_state(mod, 'b.')
    bufs0 = {k: v.detach().clone() for k, v in mod.state_dict().items() if 'running' in k or 'num_batches' in k}
    gen = torch.Generator().manual_seed(99)
    fp = None
    params = [p for p in mod.parameters()]
    if variant != 'input_grad':
        fp, prefill = flat_params(params, gen)
    with arithmetic(ops, *ARITH[arith]):
        if name == 'stem im2col':
            assert not ops.stem_supported(x.shape[-1], x.shape[-1])
        y = ours(x)
        cot = randn(*y.shape, gen=gen)
        (y * cot).sum().backward()
    ops.clear_grad_targets()
    conv = make_conv(ops, conv_mode, img_grad=img_grad)
    if x.dim() == 4:
        xd = f64_leaf(x, grad=x.requires_grad)
        yd = ref(xd, sd, conv)
    else:
        xd = f64_leaf(x, grad=x.requires_grad)
        yd = ref(nchw(xd, N, int(round((x.shape[0] / N) ** 0.5))), sd, conv)
    (rows_of(yd) * cot.to(F64)).sum().backward()
    errs, fro = {'out': rel(y, rows_of(yd))}, {'out': frob(y, rows_of(yd))}
    if x.requires_grad:
        errs['dx'], fro['dx'] = rel(x.grad, xd.grad), frob(x.grad, xd.grad)
    grads = flat_deltas(fp, prefill) if fp is not None else {p: p.grad for p in params}
    for k, p in mod.named_parameters():
        errs['d ' + k], fro['d ' + k] = rel(grads[p], sd['b.' + k].grad), frob(grads[p], sd['b.' + k].grad)
    cur = mod.state_dict()
    for k in bufs0:
        if 'num_batches' in k:      # exactly +1: 0 when right, 1 when not
            errs[k] = float(int(cur[k]) != int(bufs0[k]) + 1)
        else:
            errs[k] = rel(cur[k], sd['b.' + k])
        cur[k].copy_(bufs0[k])      # leave the shared module as it was
    if name in GATED_BLOCKS and arith != 'simt' or name == 'identity layer1[1]':
        # ReLU gates between the block's convolutions: a pre-activation within the arithmetics' difference of zero flips, and its O(1)
        # gradient change spreads through the next convolution, so the max-norm sees single flips; compare in the Frobenius norm
        print('block %s %s %s max-norm: %s' % (name, arith, variant, ', '.join('%s %.2e' % kv for kv in errs.items())))
        report('block %s %s %s Frobenius' % (name, arith, variant), fro, GATED_FROB_TOL)
        return
    print('block %s %s %s Frobenius: %s' % (name, arith, variant, ', '.join('%s %.2e' % kv for kv in fro.items())))
    report('block %s %s %s max-norm' % (name, arith, variant), errs, BLOCK_TOL[arith])


# ============================================================================ 5. the whole ResNetSimple
@pytest.mark.parametrize('arith,N', [('simt', 4), ('bench', 4), ('bench', 16)])
def test_whole_encoder_train_mode_matches_emulated_fp64(ops, arith, N):
    """ResNetSimple (trunk + heat-map and dense-pose decoders), train mode, bench arithmetic, against oracle.model_ref.encoder_forward in
    fp64 with the emulated convolutions: every output and every encoder parameter gradient under a random linear functional of all
    outputs, printed as a per-tensor table."""
    from oracle import model_ref
    enc = encoder('resnet50', seed=3)
    gen = torch.Generator().manual_seed(N)
    img = randn(N, 3, 256, 256, gen=gen)
    sd = f64_state(enc, 'encoder.')
    torch.cuda.reset_peak_memory_stats()
    with arithmetic(ops, *ARITH[arith]):
        hms, mask, dp, fm, hf, df = enc(img)
        outs = {'hms': hms, 'mask': mask, 'dp': dp}
        outs.update({'img_fmaps[%d]' % i: nchw(r, N, H) for i, (r, H) in enumerate(fm)})
        outs.update({'hms_fmaps[%d]' % i: nchw(r, N, H) for i, (r, H) in enumerate(hf)})
        outs.update({'dp_fmaps[%d]' % i: nchw(r, N, H) for i, (r, H) in enumerate(df)})
        cots = {k: randn(*v.shape, gen=gen) for k, v in outs.items()}
        sum((v * cots[k]).sum() for k, v in outs.items()).backward()
    torch.cuda.synchronize()
    conv = make_conv(ops, ARITH[arith][0])
    hms_d, mask_d, dp_d, fm_d, hf_d, df_d = model_ref.encoder_forward(sd, img.to(F64), True, conv=conv)
    refs = {'hms': hms_d, 'mask': mask_d, 'dp': dp_d}
    refs.update({'img_fmaps[%d]' % i: t for i, t in enumerate(fm_d)})
    refs.update({'hms_fmaps[%d]' % i: t for i, t in enumerate(hf_d)})
    refs.update({'dp_fmaps[%d]' % i: t for i, t in enumerate(df_d)})
    sum((v * cots[k].to(F64)).sum() for k, v in refs.items()).backward()
    errs, fro = {}, {}
    for k, v in outs.items():
        errs['out ' + k], fro['out ' + k] = rel(v, refs[k]), frob(v, refs[k])
    for k, p in enc.named_parameters():
        r = sd['encoder.' + k].grad
        if r is None:
            assert p.grad is None or float(p.grad.abs().max()) == 0.0, k
            continue
        errs['d ' + k], fro['d ' + k] = rel(p.grad, r), frob(p.grad, r)
    for k, v in enc.state_dict().items():
        if 'running' in k:
            errs[k], fro[k] = rel(v, sd['encoder.' + k]), frob(v, sd['encoder.' + k])
    print('whole encoder %s N=%d: %d tensors, peak %.2f GB' % (arith, N, len(errs), torch.cuda.max_memory_allocated() / 2 ** 30))
    for k in errs:
        print('  %-60s max %.2e  frob %.2e' % (k, errs[k], fro[k]))
    for cat in ('out ', 'd ', 'running'):
        es = [e for k, e in errs.items() if k.startswith(cat) or (cat == 'running' and 'running' in k)]
        print('  %-8s worst max-norm %.2e over %d tensors' % (cat, max(es), len(es)))
    tol_out, tol_grad = NET_TOL[arith, N]
    bad = {k: '%.2e' % e for k, e in errs.items() if not e < (tol_grad if k.startswith('d ') else tol_out)}
    assert not bad, 'whole encoder %s N=%d over the tolerances %s: %s' % (arith, N, NET_TOL[arith, N], bad)
