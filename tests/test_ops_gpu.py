"""Per-kernel parity (forward AND backward) of every C-ABI operator against the same op written in plain torch fp32
on the same device.  Tolerances are fp32 round-off (different summation order), stated per test."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# the torch side of every comparison must be true fp32 (cuDNN / cuBLAS default to TF32 convolutions on sm_100)
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False

DEV = 'cuda'


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-20))


def check(a, b, tol, what):
    assert a.shape == b.shape, (what, a.shape, b.shape)
    e = rel(a, b)
    assert e < tol, '%s: rel err %.3e (tol %.1e)' % (what, e, tol)


def grads(outs, ins, seed=0):
    g = torch.Generator(device='cpu').manual_seed(seed)
    outs = outs if isinstance(outs, (tuple, list)) else [outs]
    loss = 0
    for o in outs:
        w = torch.randn(o.shape, generator=g).to(o.device)
        loss = loss + (o * w).sum()
    return torch.autograd.grad(loss, ins, allow_unused=True)


def T(*shape, scale=1.0, seed=0, grad=True):
    g = torch.Generator().manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(DEV).requires_grad_(grad)


@pytest.fixture(scope='module')
def ops():
    from renderih_b200 import ops as o
    return o


@pytest.mark.parametrize('M,N,K', [(130, 64, 64), (4032, 256, 1024), (16128, 64, 128), (64, 509, 2048), (1000, 3, 64), (8128, 256, 256), (7, 5, 9)])
def test_linear(ops, M, N, K):
    x, w, b = T(M, K), T(N, K, scale=K ** -0.5, seed=1), T(N, seed=2)
    y = ops.linear(x, w, b)
    yr = F.linear(x, w, b)
    check(y, yr, 2e-5, 'linear fwd')
    for a, r, n in zip(grads(y, [x, w, b]), grads(yr, [x, w, b]), 'xwb'):
        check(a, r, 5e-5, 'linear d' + n)


def test_linear_relu_residual_strided(ops):
    M, N, K = 500, 128, 96
    big = T(M, K + 32)
    x = big[:, 16:16 + K]
    w, b, res = T(N, K, scale=0.1, seed=1), T(N, seed=2), T(M, N, seed=3)
    y = ops.linear(x, w, b, relu=True)
    yr = F.relu(F.linear(x, w, b))
    check(y, yr, 2e-5, 'linear relu fwd')
    for a, r in zip(grads(y, [big, w, b]), grads(yr, [big, w, b])):
        check(a, r, 5e-5, 'linear relu bwd')
    y = ops.linear(x, w, b, res=res)
    yr = F.linear(x, w, b) + res
    check(y, yr, 2e-5, 'linear res fwd')
    for a, r in zip(grads(y, [big, w, b, res]), grads(yr, [big, w, b, res])):
        check(a, r, 5e-5, 'linear res bwd')


def test_linear_dropout_is_consistent(ops):
    M, N, K = 300, 64, 64
    x, w, b = T(M, K), T(N, K, scale=0.2, seed=1), T(N, seed=2)
    ops.seed_state.manual_seed(1234, torch.device('cuda', torch.cuda.current_device()))
    ops.seed_state.begin_forward()
    y = ops.linear(x, w, b, p_drop=0.25)
    y0 = F.linear(x, w, b)
    keep = (y != 0)
    frac = float(keep.float().mean())
    assert 0.70 < frac < 0.80, frac
    check(y[keep], (y0 / 0.75)[keep], 2e-5, 'dropout scaling')
    gx, = grads(y, [x])
    gxr, = grads(y0 * keep / 0.75, [x])
    check(gx, gxr, 5e-5, 'dropout bwd uses the same mask')


@pytest.mark.parametrize('N,H,Cin,Cout,k,stride,pad,bias', [
    (2, 16, 64, 128, 3, 1, 1, False), (2, 16, 128, 128, 3, 2, 1, False), (2, 32, 256, 64, 1, 1, 0, False),
    (2, 32, 64, 128, 1, 2, 0, False), (2, 64, 3, 64, 7, 2, 3, False), (3, 16, 256, 64, 2, 2, 0, True),
    (2, 32, 256, 64, 4, 4, 0, True), (2, 16, 128, 42, 1, 1, 0, True), (1, 9, 8, 12, 3, 1, 1, True)])
def test_conv2d(ops, N, H, Cin, Cout, k, stride, pad, bias):
    x = T(N, Cin, H, H)
    w = (torch.randn(Cout, Cin, k, k) * (Cin * k * k) ** -0.5).to(DEV).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    b = T(Cout, seed=5) if bias else None
    xr = x.permute(0, 2, 3, 1).contiguous().reshape(N * H * H, Cin)
    y = ops.conv2d(xr, w, b, N, H, H, stride=stride, pad=pad)
    yr = F.conv2d(x, w, b, stride=stride, padding=pad)
    Ho = yr.shape[2]
    yr2 = yr.permute(0, 2, 3, 1).reshape(N * Ho * Ho, Cout)
    check(y, yr2, 3e-5, 'conv fwd')
    ins = [x, w] + ([b] if bias else [])
    for a, r, n in zip(grads(y, ins), grads(yr2, ins), 'xwb'):
        check(a, r, 1e-4, 'conv d' + n)


def test_conv_relu_bn_order(ops):
    """Conv -> ReLU -> BN (training) with the ReLU mask applied inside the BN backward."""
    N, H, C, Co = 4, 8, 64, 128
    x = T(N, C, H, H)
    w = (torch.randn(Co, C, 3, 3) * 0.05).to(DEV).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    gamma, beta = T(Co, seed=1), T(Co, seed=2)
    rm, rv = torch.zeros(Co, device=DEV), torch.ones(Co, device=DEV)
    rm2, rv2 = rm.clone(), rv.clone()
    xr = x.permute(0, 2, 3, 1).contiguous().reshape(-1, C)
    y = ops.conv2d(xr, w, None, N, H, H, stride=1, pad=1, relu=True, relu_masked_by_consumer=True)
    y = ops.batchnorm(y, gamma, beta, rm, rv, training=True, mask_input=True)
    yr = F.batch_norm(F.relu(F.conv2d(x, w, padding=1)), rm2, rv2, gamma, beta, True, 0.1, 1e-5)
    yr = yr.permute(0, 2, 3, 1).reshape(-1, Co)
    check(y, yr, 3e-5, 'conv-relu-bn fwd')
    check(rm, rm2, 1e-5, 'running mean'); check(rv, rv2, 1e-5, 'running var')
    for a, r, n in zip(grads(y, [x, w, gamma, beta]), grads(yr, [x, w, gamma, beta]), ['x', 'w', 'gamma', 'beta']):
        check(a, r, 2e-4, 'conv-relu-bn d' + n)


@pytest.mark.parametrize('mode', ['simt', 'tf32x3'])
def test_conv_bn_fused_statistics(ops, mode):
    """BatchNorm batch statistics accumulated inside the convolution's epilogue == statistics of a separate pass."""
    N, H, C, Co = 3, 16, 64, 160      # 768 pixels (6 row tiles), Cout not a multiple of the 128-wide tile
    x = T(N, C, H, H, grad=False)
    w = (torch.randn(Co, C, 1, 1) * 0.1).to(DEV).contiguous(memory_format=torch.channels_last)
    xr = x.permute(0, 2, 3, 1).contiguous().reshape(-1, C)
    stats = torch.full((2 * Co,), 7.0, device=DEV, dtype=torch.float64)
    ops.set_gemm_mode(mode, mode)
    try:
        y = ops.conv2d(xr, w, None, N, H, H, relu=True, relu_masked_by_consumer=True, stats=stats)
    finally:
        ops.set_gemm_mode('simt', 'simt')
    torch.cuda.synchronize()
    check(stats[:Co].float(), y.double().sum(0).float(), 1e-5, 'fused column sums')
    check(stats[Co:].float(), (y.double() ** 2).sum(0).float(), 1e-5, 'fused column sums of squares')


@pytest.mark.parametrize('training', [True, False])
def test_batchnorm_residual_relu(ops, training):
    M, C = 2048, 256
    x, res, gamma, beta = T(M, C), T(M, C, seed=1), T(C, seed=2), T(C, seed=3)
    rm, rv = torch.randn(C, device=DEV) * 0.1, torch.rand(C, device=DEV) + 0.5
    rm2, rv2 = rm.clone(), rv.clone()
    y = ops.batchnorm(x, gamma, beta, rm, rv, res=res, training=training, relu=True)
    yr = F.relu(F.batch_norm(x, rm2, rv2, gamma, beta, training, 0.1, 1e-5) + res)
    check(y, yr, 2e-5, 'bn fwd')
    check(rm, rm2, 1e-5, 'running mean'); check(rv, rv2, 1e-5, 'running var')
    for a, r, n in zip(grads(y, [x, res, gamma, beta]), grads(yr, [x, res, gamma, beta]), ['x', 'res', 'gamma', 'beta']):
        check(a, r, 1e-4, 'bn d' + n)


@pytest.mark.parametrize('F_', [64, 256, 509, 512])
def test_layernorm(ops, F_):
    M = 777
    a, b, g, be = T(M, F_), T(M, F_, seed=1), T(F_, seed=2), T(F_, seed=3)
    y = ops.layernorm(a, g, be, b=b, relu=True)
    yr = F.relu(F.layer_norm(a + b, (F_,), g, be, 1e-6))
    check(y, yr, 1e-5, 'ln fwd')
    for u, r, n in zip(grads(y, [a, b, g, be]), grads(yr, [a, b, g, be]), ['a', 'b', 'gamma', 'beta']):
        check(u, r, 1e-4, 'ln d' + n)
    y = ops.layernorm(a, g, be)
    yr = F.layer_norm(a, (F_,), g, be, 1e-6)
    check(y, yr, 1e-5, 'ln fwd plain')
    for u, r in zip(grads(y, [a, g, be]), grads(yr, [a, g, be])):
        check(u, r, 1e-4, 'ln plain bwd')


def test_cheb(ops):
    from renderih_b200 import assets
    from renderih_b200.model import GraphCSR
    L = assets.synthetic_assets(3)['left_graph']['coarsen_graphs_L'][2]   # 252
    g = GraphCSR(L).to(torch.device(DEV))
    Ld = g.dense().to(DEV)
    B, V, Fin = 5, 252, 64
    x = T(B * V, Fin)
    y = ops.cheb(x, g, B, V)
    x3 = x.view(B, V, Fin)
    yr = torch.stack([x3, torch.einsum('vu,buf->bvf', Ld, x3)], -1).reshape(B * V, 2 * Fin)
    check(y, yr, 1e-5, 'cheb fwd')
    check(grads(y, [x])[0], grads(yr, [x])[0], 1e-5, 'cheb bwd')


@pytest.mark.parametrize('B,H,Sq,Sk,d', [(3, 4, 63, 63, 64), (2, 4, 252, 316, 16), (2, 4, 126, 190, 32), (2, 4, 64, 64, 16), (1, 2, 5, 7, 8)])
def test_attention(ops, B, H, Sq, Sk, d):
    q, k, v = T(B * Sq, H * d), T(B * Sk, H * d, seed=1), T(B * Sk, H * d, seed=2)
    o = ops.attention(q, k, v, B, H, Sq, Sk)
    qh = q.view(B, Sq, H, d).transpose(1, 2); kh = k.view(B, Sk, H, d).transpose(1, 2); vh = v.view(B, Sk, H, d).transpose(1, 2)
    a = F.softmax(torch.matmul(qh, kh.transpose(-1, -2)) / d ** 0.5, -1)
    orf = torch.matmul(a, vh).transpose(1, 2).reshape(B * Sq, H * d)
    check(o, orf, 1e-5, 'attn fwd')
    for u, r, n in zip(grads(o, [q, k, v]), grads(orf, [q, k, v]), 'qkv'):
        check(u, r, 1e-4, 'attn d' + n)


@pytest.mark.parametrize('B,H,Sq,Sk,d', [(3, 4, 63, 63, 64), (2, 4, 252, 316, 16), (2, 4, 126, 190, 32), (2, 4, 64, 64, 16), (5, 4, 63, 127, 64),
                                          (1, 2, 5, 7, 8), (2, 3, 130, 70, 32)])
@pytest.mark.parametrize('nsplit_mode', ['tf32x3', 'tf32'])
def test_attention_tensor_core(ops, B, H, Sq, Sk, d, nsplit_mode):
    """wgmma attention core (batched per-head GEMMs over 4-D TMA maps + warp-per-row softmax), forward and backward, against plain
    torch fp32.  Stated tolerance: 3xTF32 5e-5 relative to each tensor's max (fp32-faithful), single-pass TF32 5e-3."""
    tol = 5e-5 if nsplit_mode == 'tf32x3' else 5e-3
    q, k, v = T(B * Sq, H * d, seed=1), T(B * Sk, H * d, seed=2), T(B * Sk, H * d, seed=3)
    ops.set_gemm_mode('simt', nsplit_mode)
    try:
        o = ops.attention(q, k, v, B, H, Sq, Sk, impl='tc')
        g_ours = grads(o, [q, k, v])
    finally:
        ops.set_gemm_mode('simt', 'simt')
    qh, kh, vh = (t.view(B, -1, H, d).transpose(1, 2) for t in (q, k, v))
    ref = torch.matmul(F.softmax(torch.matmul(qh, kh.transpose(-1, -2)) / d ** 0.5, -1), vh).transpose(1, 2).reshape(B * Sq, H * d)
    check(o, ref, tol, 'attn tc fwd')
    for a, r, n in zip(g_ours, grads(ref, [q, k, v]), 'qkv'):
        check(a, r, tol, 'attn tc d' + n)


def test_attention_tensor_core_dropout_matches_simt_statistics(ops):
    """Dropout on the tensor-core path: forward / backward stay consistent (same regenerated mask), the kept fraction is 1 - p and the
    expectation is preserved; with p = 0 the result equals the SIMT kernel's to fp32 round-off."""
    B, H, S, d = 4, 4, 126, 32
    q, k, v = T(B * S, H * d, seed=4), T(B * S, H * d, seed=5), T(B * S, H * d, seed=6)
    ops.seed_state.manual_seed(1234, q.device)
    ops.seed_state.begin_forward()
    ops.set_gemm_mode('simt', 'tf32x3')
    try:
        o0 = ops.attention(q, k, v, B, H, S, S, p_drop=0.0, impl='tc')
        o1 = ops.attention(q, k, v, B, H, S, S, p_drop=0.3, impl='tc')
        gq, gk, gv = grads(o1, [q, k, v])
    finally:
        ops.set_gemm_mode('simt', 'simt')
    os_ = ops.attention(q, k, v, B, H, S, S, p_drop=0.0, impl='simt')
    check(o0, os_, 5e-5, 'tc vs simt (no dropout)')
    assert torch.isfinite(o1).all() and torch.isfinite(gq).all() and torch.isfinite(gk).all() and torch.isfinite(gv).all()
    assert rel(o1.mean(0), o0.mean(0)) < 0.5            # same expectation (loose: one draw)
    # finite-difference check of the dropout path through V (linear in V, so exact up to round-off): <dO, dV-direction>
    dvdir = torch.randn_like(v)
    ops.seed_state.begin_forward()
    ops.set_gemm_mode('simt', 'tf32x3')
    try:
        _ = ops.attention(q, k, v, B, H, S, S, p_drop=0.0, impl='tc')           # consume site 0 like above
        o2 = ops.attention(q, k, (v + dvdir).detach(), B, H, S, S, p_drop=0.3, impl='tc')
    finally:
        ops.set_gemm_mode('simt', 'simt')
    w = torch.randn(o1.shape, generator=torch.Generator(device='cpu').manual_seed(0)).to(o1.device)     # the cotangent grads() used
    lhs = float(((o2 - o1) * w).sum())
    rhs = float((gv * dvdir).sum())
    assert abs(lhs - rhs) / (abs(rhs) + 1e-6) < 1e-3, (lhs, rhs)


def test_attention_strided_qkv(ops):
    B, H, S, d = 2, 4, 63, 16
    qkv = T(B * S, 3 * H * d)
    q, k, v = qkv[:, :H * d], qkv[:, H * d:2 * H * d], qkv[:, 2 * H * d:]
    o = ops.attention(q, k, v, B, H, S, S)
    qh, kh, vh = (t.reshape(B, S, H, d).transpose(1, 2) for t in (q, k, v))
    orf = torch.matmul(F.softmax(torch.matmul(qh, kh.transpose(-1, -2)) / d ** 0.5, -1), vh).transpose(1, 2).reshape(B * S, H * d)
    check(o, orf, 1e-5, 'attn strided fwd')
    check(grads(o, [qkv])[0], grads(orf, [qkv])[0], 1e-4, 'attn strided bwd')


def test_posemb_upsample(ops):
    B, V, F_ = 3, 63, 128
    x, emb = T(B * V, F_), T(2 * V, F_, seed=1)
    y = ops.posemb(x, emb, B, 2 * V, 2)
    yr = (x.view(B, V, F_).repeat_interleave(2, dim=1) + emb[None]).reshape(B * 2 * V, F_)
    check(y, yr, 1e-6, 'posemb fwd')
    for u, r in zip(grads(y, [x, emb]), grads(yr, [x, emb])):
        check(u, r, 1e-5, 'posemb bwd')


def test_gf_broadcast(ops):
    B, V, G = 4, 63, 509
    g, emb = T(B, G), T(V, G + 3, seed=1)
    pe = torch.randn(V, 3, device=DEV)
    y = ops.gf_broadcast(g, pe, emb, B, V)
    yr = (torch.cat([g[:, None].repeat(1, V, 1), pe[None].repeat(B, 1, 1)], -1) + emb[None]).reshape(B * V, G + 3)
    check(y, yr, 1e-6, 'gf fwd')
    for u, r in zip(grads(y, [g, emb]), grads(yr, [g, emb])):
        check(u, r, 1e-5, 'gf bwd')


def test_decoder_tail(ops):
    B, V, F_, Nv = 3, 252, 64, 778
    Lf = T(B * V, F_)
    aw, ab, pw, pb, cw, cb = T(V, scale=0.05, seed=1), T(1, seed=2), T(3, F_, scale=0.1, seed=3), T(3, seed=4), T(3, F_, scale=0.1, seed=5), T(3, seed=6)
    U = T(Nv, V, scale=0.05, seed=7)
    outs = ops.decoder_tail(Lf, aw, ab, pw, pb, cw, cb, U, B, V, 256.0)
    L3 = Lf.view(B, V, F_)
    t = F.linear(F.linear(L3.transpose(1, 2), aw[None], ab)[..., 0], pw, pb)
    scale, trans = t[:, 0], t[:, 1:]
    v3c = F.linear(L3, cw, cb)
    proj = lambda v: (scale * 256)[:, None, None] * v[..., :2] + (trans * 128 + 128)[:, None]
    v3 = F.linear(v3c.transpose(1, 2), U).transpose(1, 2)
    refs = (scale, trans, v3c, proj(v3c), v3, proj(v3))
    for o, r, n in zip(outs, refs, ['scale', 'trans', 'v3c', 'v2c', 'v3', 'v2']):
        check(o, r, 2e-5, 'tail ' + n)
    ins = [Lf, aw, ab, pw, pb, cw, cb, U]
    for u, r, n in zip(grads(list(outs), ins), grads(list(refs), ins), ['Lf', 'aw', 'ab', 'pw', 'pb', 'cw', 'cb', 'U']):
        check(u, r, 2e-4, 'tail d' + n)


def test_maxpool_bilinear_gap_layout(ops):
    N, C, H = 2, 64, 16
    x = T(N, C, H, H)
    xr = ops.nchw_to_nhwc(x)
    check(xr, x.permute(0, 2, 3, 1).reshape(-1, C), 1e-7, 'nchw->nhwc')
    y = ops.maxpool3x3s2(F.relu(xr), N, H, H)
    yr = F.max_pool2d(F.relu(x), 3, 2, 1).permute(0, 2, 3, 1).reshape(-1, C)
    check(y, yr, 1e-7, 'maxpool fwd')
    check(grads(y, [x])[0], grads(yr, [x])[0], 1e-6, 'maxpool bwd')
    y = ops.bilinear2x(xr, N, H, H)
    yr = F.interpolate(x, scale_factor=2, mode='bilinear', align_corners=True).permute(0, 2, 3, 1).reshape(-1, C)
    check(y, yr, 1e-5, 'bilinear fwd')
    check(grads(y, [x])[0], grads(yr, [x])[0], 1e-5, 'bilinear bwd')
    y = ops.global_avgpool(xr, N, H * H)
    yr = x.mean(dim=(2, 3))
    check(y, yr, 1e-5, 'gap fwd')
    check(grads(y, [x])[0], grads(yr, [x])[0], 1e-5, 'gap bwd')
    y = ops.nhwc_to_nchw(xr, N, H, H, 8, 16)
    check(y, x[:, 8:24], 1e-7, 'nhwc->nchw slice')
    check(grads(y, [x])[0], grads(x[:, 8:24], [x])[0], 1e-7, 'nhwc->nchw bwd')
    y = ops.concat_channels([xr, xr[:, :32] * 2])
    yr = torch.cat([xr, xr[:, :32] * 2], 1)
    check(y, yr, 1e-7, 'concat')
    check(grads(y, [x])[0], grads(yr, [x])[0], 1e-6, 'concat bwd')
    a, b = T(3 * 5, 8), T(3 * 2, 8, seed=1)
    y = ops.concat_rows(a, b, 3, 5, 2)
    yr = torch.cat([a.view(3, 5, 8), b.view(3, 2, 8)], 1).reshape(21, 8)
    check(y, yr, 1e-7, 'concat rows')
    for u, r in zip(grads(y, [a, b]), grads(yr, [a, b])):
        check(u, r, 1e-7, 'concat rows bwd')
    idx = torch.randint(0, 4 * 12, (30,), device=DEV, dtype=torch.int32)
    z = T(2, 12, 3)
    y = ops.gather_rows(z, idx, 4)
    yr = z[:, (idx // 4).long()]
    check(y, yr, 1e-7, 'gather rows')
    check(grads(y, [z])[0], grads(yr, [z])[0], 1e-6, 'gather rows bwd')


def test_no_cpu_fallback(ops):
    with pytest.raises(RuntimeError):
        ops.linear(torch.randn(4, 4), torch.randn(4, 4))


# ----------------------------------------------------------------------------- wgmma tensor-core GEMM (TF32 multiplicands)
def _tf32_trunc(t):
    return (t.view(torch.int32) & -8192).view(torch.float32)


@pytest.mark.parametrize('M,N,K', [(128, 128, 32), (128, 128, 256), (256, 64, 64), (4032, 256, 1024), (1000, 200, 72), (16128, 64, 128), (300, 509, 2048)])
def test_gemm_tf32_kmajor(M, N, K):
    from renderih_b200._lib import call
    a, b = T(M, K, grad=False), T(N, K, seed=1, grad=False)
    c = torch.full((M, N), float('nan'), device=DEV)
    call('rih_gemm_tf32', a.data_ptr(), K, 0, b.data_ptr(), K, 0, c.data_ptr(), N, M, N, K, None, 0, 0, 0, 1, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    ref = _tf32_trunc(a).double() @ _tf32_trunc(b).double().t()
    ref_rn = a.double() @ b.double().t()
    e_trunc, e_full = rel(c, ref), rel(c, ref_rn)
    print('tf32 gemm %dx%dx%d: err vs truncated-input fp64 %.2e, vs exact %.2e' % (M, N, K, e_trunc, e_full))
    assert e_full < 5e-3, (e_trunc, e_full)


@pytest.mark.parametrize('a_mn,b_mn', [(0, 1), (1, 1)])
def test_gemm_tf32_mn_major(a_mn, b_mn):
    from renderih_b200._lib import call
    M, N, K = 384, 256, 160
    a = T(K, M, grad=False) if a_mn else T(M, K, grad=False)
    b = T(K, N, seed=1, grad=False) if b_mn else T(N, K, seed=1, grad=False)
    c = torch.full((M, N), float('nan'), device=DEV)
    call('rih_gemm_tf32', a.data_ptr(), a.shape[1], a_mn, b.data_ptr(), b.shape[1], b_mn, c.data_ptr(), N, M, N, K, None, 0, 0, 0, 1,
         torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    A = a.t() if a_mn else a
    Bm = b.t() if b_mn else b
    e = rel(c, A.double() @ Bm.double().t())
    print('tf32 gemm a_mn=%d b_mn=%d: rel err %.2e' % (a_mn, b_mn, e))
    assert e < 5e-3, e


def test_gemm_tf32_splitk_bias_relu():
    from renderih_b200._lib import call
    M, N, K = 256, 128, 8192
    a, b = T(K, M, grad=False), T(K, N, seed=1, grad=False)
    c = torch.full((M, N), float('nan'), device=DEV)
    call('rih_gemm_tf32', a.data_ptr(), M, 1, b.data_ptr(), N, 1, c.data_ptr(), N, M, N, K, None, 0, 0, 1, 1, torch.cuda.current_stream().cuda_stream)
    e = rel(c, a.double().t() @ b.double())
    assert e < 5e-3, e
    a2, b2, bias = T(500, 96, grad=False), T(70, 96, seed=1, grad=False), T(70, seed=2, grad=False)
    c2 = torch.empty((500, 70), device=DEV)
    call('rih_gemm_tf32', a2.data_ptr(), 96, 0, b2.data_ptr(), 96, 0, c2.data_ptr(), 70, 500, 70, 96, bias.data_ptr(), 1, 0, 0, 1, torch.cuda.current_stream().cuda_stream)
    e = rel(c2, F.relu(a2.double() @ b2.double().t() + bias.double()))
    assert e < 5e-3, e


@pytest.mark.parametrize('N,H,Cin,Cout,k', [(2, 64, 128, 128, 3), (4, 32, 128, 128, 3), (8, 16, 256, 256, 3), (4, 8, 512, 512, 3), (2, 64, 64, 64, 3),
                                             (2, 32, 512, 128, 1), (4, 16, 1024, 256, 1), (2, 64, 256, 64, 1)])
def test_conv2d_tensor_core_tf32(ops, N, H, Cin, Cout, k):
    """wgmma implicit-GEMM convolution (fwd, dgrad, wgrad) against fp32 torch; tolerance = single-pass TF32."""
    x = T(N, Cin, H, H)
    w = (torch.randn(Cout, Cin, k, k) * (Cin * k * k) ** -0.5).to(DEV).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    xr = x.permute(0, 2, 3, 1).contiguous().reshape(N * H * H, Cin)
    ops.set_gemm_mode('tf32', 'tf32')
    try:
        y = ops.conv2d(xr, w, None, N, H, H, stride=1, pad=k // 2)
        g_ours = grads(y, [x, w])
    finally:
        ops.set_gemm_mode('simt', 'simt')
    yr = F.conv2d(x, w, None, stride=1, padding=k // 2).permute(0, 2, 3, 1).reshape(N * H * H, Cout)
    e = rel(y, yr)
    print('tc conv %dx%d %d->%d @%d: fwd rel err %.2e' % (k, k, Cin, Cout, H, e))
    assert e < 3e-3, e
    for a, r, n in zip(g_ours, grads(yr, [x, w]), 'xw'):
        e = rel(a, r)
        print('   d%s rel err %.2e' % (n, e))
        assert e < 3e-3, (n, e)


@pytest.mark.parametrize('N,H,Cin,Cout,k', [(4, 64, 128, 128, 3), (4, 32, 256, 256, 3), (8, 16, 512, 512, 3), (4, 64, 256, 512, 1), (4, 16, 1024, 2048, 1)])
@pytest.mark.parametrize('mode', ['tf32', 'tf32x3'])
@pytest.mark.parametrize('direct', [1, 0])
def test_conv2d_stride2_tensor_core(ops, N, H, Cin, Cout, k, mode, direct):
    """stride-2 convolutions on the wgmma path.  direct = 1: the tensors are addressed in place through element-strided tensor maps (forward,
    weight gradient) and the input gradient runs as four parity-class GEMMs; direct = 0: parity-stacked input for fwd/wgrad, zero-inserted dY
    for dgrad (the copy-based formulation kept for comparison)."""
    from renderih_b200._lib import call
    call('rih_set_s2_direct', direct)
    x = T(N, Cin, H, H)
    w = (torch.randn(Cout, Cin, k, k) * (Cin * k * k) ** -0.5).to(DEV).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    xr = x.permute(0, 2, 3, 1).contiguous().reshape(N * H * H, Cin)
    ops.set_gemm_mode(mode, mode)
    try:
        y = ops.conv2d(xr, w, None, N, H, H, stride=2, pad=k // 2)
        g_ours = grads(y, [x, w])
    finally:
        ops.set_gemm_mode('simt', 'simt')
        call('rih_set_s2_direct', 1)
    yr = F.conv2d(x, w, None, stride=2, padding=k // 2).permute(0, 2, 3, 1).reshape(-1, Cout)
    tol = 3e-3 if mode == "tf32" else 1e-4
    assert rel(y, yr) < tol, rel(y, yr)
    for a, r, n in zip(g_ours, grads(yr, [x, w]), 'xw'):
        assert rel(a, r) < tol, (n, rel(a, r))


@pytest.mark.parametrize('N,H,Cin,Cout,k,stride', [
    (2, 64, 48, 48, 3, 1), (2, 32, 96, 96, 3, 1), (4, 16, 192, 192, 3, 1), (2, 8, 384, 384, 3, 1),      # HRNet-w48 branch blocks
    (2, 64, 256, 48, 3, 1), (2, 64, 48, 128, 3, 1), (2, 16, 80, 208, 3, 1),                              # transition1.0 / odd multiples of 16
    (2, 64, 48, 48, 3, 2), (2, 64, 48, 96, 3, 2), (4, 32, 96, 192, 3, 2), (2, 64, 256, 96, 3, 2), (4, 16, 192, 384, 3, 2)])   # fuse / transition chains
def test_conv2d_tensor_core_channels_multiple_of_16(ops, N, H, Cin, Cout, k, stride):
    """Channel counts that are multiples of 16 but not of 32 / 64 (HRNet-w48: 48, 96 ...) on the wgmma path: the K blocks / N chunks that
    stick out of the tensor are zero-filled (loads) and clipped (stores, 3-D dW map per tap) by the TMA unit.  3xTF32 so that any stray
    contribution would show: tolerance 1e-4 relative (fp32-faithful), forward, dgrad and wgrad; and the path must really be the tensor-core one."""
    import ctypes
    from renderih_b200._lib import call
    x = T(N, Cin, H, H)
    w = (torch.randn(Cout, Cin, k, k) * (Cin * k * k) ** -0.5).to(DEV).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    xr = x.permute(0, 2, 3, 1).contiguous().reshape(N * H * H, Cin)
    ops.set_gemm_mode('tf32x3', 'tf32x3')
    try:
        Ho = (H + 2 * (k // 2) - k) // stride + 1
        geom = (ctypes.c_int * 13)(N, H, H, Cin, Ho, Ho, Cout, k, k, stride, k // 2, Cin, Cout)
        for which in (0, 1, 2):
            flag = ctypes.c_int(0)
            call('rih_conv2d_tc_supported', geom, which, ctypes.byref(flag))
            assert flag.value == 1, ('not on the tensor-core path', which)
        y = ops.conv2d(xr, w, None, N, H, H, stride=stride, pad=k // 2)
        g_ours = grads(y, [x, w])
    finally:
        ops.set_gemm_mode('simt', 'simt')
    yr = F.conv2d(x, w, None, stride=stride, padding=k // 2).permute(0, 2, 3, 1).reshape(-1, Cout)
    assert rel(y, yr) < 1e-4, rel(y, yr)
    for a, r, n in zip(g_ours, grads(yr, [x, w]), 'xw'):
        assert rel(a, r) < 1e-4, (n, rel(a, r))


@pytest.mark.parametrize('H,p,C,Co', [(32, 4, 256, 64), (16, 2, 256, 128)])
def test_patchify_linear_equals_patch_conv(ops, H, p, C, Co):
    N = 3
    x = T(N, C, H, H)
    w = (torch.randn(Co, C, p, p) * 0.02).to(DEV).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    b = T(Co, seed=3)
    xr = x.permute(0, 2, 3, 1).contiguous().reshape(N * H * H, C)
    y = ops.linear(ops.patchify(xr, N, H, H, p), w.permute(0, 2, 3, 1).reshape(Co, -1), b, relu=True)
    yr = F.relu(F.conv2d(x, w, b, stride=p)).permute(0, 2, 3, 1).reshape(-1, Co)
    check(y, yr, 3e-5, 'patch conv fwd')
    for a, r, n in zip(grads(y, [x, w, b]), grads(yr, [x, w, b]), 'xwb'):
        check(a, r, 1e-4, 'patch conv d' + n)


@pytest.mark.parametrize('M,N,K', [(4032, 256, 512), (16128, 64, 128), (8128, 256, 256)])
def test_linear_tensor_core_tf32(ops, M, N, K):
    x, w, b = T(M, K), T(N, K, scale=K ** -0.5, seed=1), T(N, seed=2)
    ops.set_gemm_mode('tf32', 'tf32')
    try:
        y = ops.linear(x, w, b)          # (no ReLU here: a TF32-perturbed mask would dominate the gradient comparison)
        g_ours = grads(y, [x, w, b])
    finally:
        ops.set_gemm_mode('simt', 'simt')
    yr = F.linear(x, w, b)
    assert rel(y, yr) < 3e-3
    for a, r, n in zip(g_ours, grads(yr, [x, w, b]), 'xwb'):
        assert rel(a, r) < 3e-3, (n, rel(a, r))


@pytest.mark.parametrize('M,N,K,a_mn,b_mn', [(4032, 256, 1024, 0, 0), (1000, 200, 72, 0, 0), (384, 256, 160, 0, 1), (384, 256, 160, 1, 1), (256, 128, 8192, 1, 1)])
def test_gemm_3xtf32_is_fp32_faithful(M, N, K, a_mn, b_mn):
    """Error-compensated 3xTF32 (hi/lo split in shared memory): fp32-level accuracy from the tensor cores."""
    from renderih_b200._lib import call
    a = T(K, M, grad=False) if a_mn else T(M, K, grad=False)
    b = T(K, N, seed=1, grad=False) if b_mn else T(N, K, seed=1, grad=False)
    c = torch.full((M, N), float('nan'), device=DEV)
    call('rih_gemm_tf32', a.data_ptr(), a.shape[1], a_mn, b.data_ptr(), b.shape[1], b_mn, c.data_ptr(), N, M, N, K, None, 0, 0, int(K >= 4096), 3,
         torch.cuda.current_stream().cuda_stream)
    A_ = a.t() if a_mn else a
    B_ = b.t() if b_mn else b
    ref = A_.double() @ B_.double().t()
    e = rel(c, ref)
    e32 = rel(A_ @ B_.t(), ref)
    print('3xtf32 gemm %dx%dx%d (a_mn=%d b_mn=%d): rel err %.2e   (torch fp32 matmul: %.2e)' % (M, N, K, a_mn, b_mn, e, e32))
    assert e < 2e-5, e   # limited by the tensor core's internal (truncating) accumulation over K, not by the operand split


def test_gemm_tf32_round_to_nearest_is_unbiased():
    """NSPLIT=2: operands rounded to nearest TF32 in shared memory (cuDNN/cuBLAS convention) -> smaller, unbiased error
    than the hardware's truncation."""
    from renderih_b200._lib import call
    M, N, K = 2048, 256, 1024
    a, b = (T(M, K, grad=False).abs() + 0.1), (T(N, K, seed=1, grad=False).abs() + 0.1)     # all-positive: truncation bias shows
    ref = a.double() @ b.double().t()
    errs = {}
    for ns in (1, 2):
        c = torch.empty((M, N), device=DEV)
        call('rih_gemm_tf32', a.data_ptr(), K, 0, b.data_ptr(), K, 0, c.data_ptr(), N, M, N, K, None, 0, 0, 0, ns, torch.cuda.current_stream().cuda_stream)
        errs[ns] = float(((c.double() - ref) / ref).mean())
    print('mean signed relative error: truncating %.2e, round-to-nearest %.2e' % (errs[1], errs[2]))
    assert abs(errs[2]) < 2e-5 and abs(errs[1]) > 1e-4


@pytest.mark.parametrize('nsplit', [1, 3])
def test_gemm_bias_relu_many_tiles(nsplit):
    """Bias + ReLU epilogue over many 128x128 output tiles (N % 256 == 0) against fp64."""
    from renderih_b200._lib import call
    M, N, K = 16384, 512, 192
    a, b, bias = T(M, K, grad=False), T(N, K, seed=1, grad=False), T(N, seed=2, grad=False)
    c = torch.empty((M, N), device=DEV)
    call('rih_gemm_tf32', a.data_ptr(), K, 0, b.data_ptr(), K, 0, c.data_ptr(), N, M, N, K, bias.data_ptr(), 1, 0, 0, nsplit, torch.cuda.current_stream().cuda_stream)
    ref = F.relu(a.double() @ b.double().t() + bias.double())
    assert rel(c, ref) < (3e-3 if nsplit == 1 else 2e-5)


def test_preprocess_u8_matches_reference_loader_ops():
    """GPU input kernel against the exact host ops of core/loader.py:151-152,178-181 (cv.flip, cv.cvtColor BGR2RGB, /255, permute,
    torchvision Normalize): bit-identical."""
    import numpy as np
    import cv2 as cv
    from torchvision import transforms
    from renderih_b200.input import preprocess_u8
    rng = np.random.RandomState(0)
    imgs = rng.randint(0, 256, size=(5, 64, 48, 3), dtype=np.uint8)
    flips = [False, True, False, True, True]
    norm = transforms.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])
    ref = []
    for img, f in zip(imgs, flips):
        if f:
            img = cv.flip(img, 1)
        t = torch.tensor(cv.cvtColor(img, cv.COLOR_BGR2RGB), dtype=torch.float32) / 255
        ref.append(norm(t.permute(2, 0, 1)))
    ref = torch.stack(ref)
    out = preprocess_u8(torch.from_numpy(imgs).cuda(), flip=torch.tensor(flips))
    assert out.shape == ref.shape and torch.equal(out.cpu(), ref)
    out2 = preprocess_u8(torch.from_numpy(imgs).cuda())
    assert torch.equal(out2[0].cpu(), ref[0]) and not torch.equal(out2[1].cpu(), ref[1])
    with pytest.raises(RuntimeError):
        preprocess_u8(torch.from_numpy(imgs))


@pytest.mark.parametrize('mode', ['tf32', 'tf32x3'])
def test_stem_conv_implicit_gemm(ops, mode):
    """torchvision conv1 (7x7 / stride 2 / pad 3, 3 -> 64) as the wgmma implicit GEMM over the zero-bordered NHWC4 image (overlapping-stride
    tensor map, no im2col buffer): forward, fused BatchNorm column statistics and the weight gradient against F.conv2d."""
    N, H = 2, 256
    g = torch.Generator().manual_seed(3)
    img = torch.randn(N, 3, H, H, generator=g).to(DEV)
    w = (torch.randn(64, 3, 7, 7, generator=g) * 147 ** -0.5).to(DEV).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    ops.set_gemm_mode(mode, mode)
    try:
        assert ops.stem_supported(H, H)
        stats = torch.empty(128, device=DEV, dtype=torch.float64)
        y = ops.stem_conv(img, w, stats)
        gw = grads(y, [w])[0]
    finally:
        ops.set_gemm_mode('simt', 'simt')
    wr = w.detach().clone().requires_grad_(True)
    yr = F.conv2d(img, wr, None, stride=2, padding=3).permute(0, 2, 3, 1).reshape(-1, 64)
    tol = 3e-3 if mode == 'tf32' else 1e-4
    assert y.shape == yr.shape
    assert rel(y, yr) < tol, rel(y, yr)
    assert rel(gw, grads(yr, [wr])[0]) < tol, rel(gw, grads(yr, [wr])[0])
    ref_s = torch.cat([y.double().sum(0), (y.double() ** 2).sum(0)])
    assert rel(stats, ref_s) < 1e-6, rel(stats, ref_s)


def test_bottleneck_with_stride2_shortcut_tensor_core_matches_exact(ops):
    """A ResNet bottleneck whose shortcut is a 1x1 / stride-2 convolution (layer2[0]), train mode: the tensor-core path (3xTF32; direct stride-2
    convolutions, the shortcut's input gradient accumulated by conv1's dgrad epilogue (TMA reduce-add), ReLU bitmask
    of the residual BatchNorm, multi-tap wgrad tiles) against the exact-fp32 kernels -- output, input gradient and every parameter gradient."""
    from renderih_b200.model import ResNetSimple
    torch.manual_seed(0)
    enc = ResNetSimple('resnet50', aux_heads=False).to(DEV).train()
    blk = enc.resnet.layer2[0]
    N, H = 4, 64
    x0 = (torch.randn(N * H * H, 256, device=DEV) * 0.5)
    res = {}
    for mode in ('simt', 'tf32x3'):
        for p in blk.parameters():
            p.grad = None
        for m in blk.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.reset_running_stats()
        x = x0.clone().requires_grad_(True)
        ops.set_gemm_mode(mode, mode)
        try:
            y, Ho = enc._bottleneck(blk, x, N, H)
            g = torch.Generator(device='cpu').manual_seed(1)
            wgt = torch.randn(y.shape, generator=g).to(DEV)
            (y * wgt).sum().backward()
        finally:
            ops.set_gemm_mode('simt', 'simt')
        res[mode] = (y.detach().clone(), x.grad.clone(), {k: p.grad.clone() for k, p in blk.named_parameters()})
    assert Ho == 32
    assert rel(res['tf32x3'][0], res['simt'][0]) < 2e-4, rel(res['tf32x3'][0], res['simt'][0])

    # Gradients: the two arithmetics differ by ~1e-6, which flips the ReLU gate of the handful of pre-activations that sit that close to zero
    # (16 M activations in the block); a flipped gate changes that element's gradient by O(1), so the max-norm sees single flips (9e-2 here,
    # identical with every kernel switch) and a 3x3 convolution spreads it over the neighbouring pixels.  Compare in the Frobenius norm.
    def l2(a, b):
        a, b = a.double(), b.double()
        return float((a - b).norm() / b.norm().clamp_min(1e-30))

    # measured (tools/debug_bottleneck.py, torch fp32 as the third opinion): exact-fp32 kernels 4e-7 from torch in every tensor; 3xTF32 path y 3.7e-6,
    # dx 1.7e-3, parameter gradients 5e-4 ... 2.6e-3 -- identical for direct / copy-based stride 2 and with / without the alias accumulation
    dx, dxr = res['tf32x3'][1], res['simt'][1]
    assert l2(dx, dxr) < 5e-3, l2(dx, dxr)
    for k, gref in res['simt'][2].items():
        e = l2(res['tf32x3'][2][k], gref)
        assert e < 5e-3, (k, e)


@pytest.mark.parametrize('N,H,Cin,Cout,k,stride', [(4, 32, 256, 64, 1, 1), (4, 32, 64, 64, 3, 1), (4, 32, 64, 256, 1, 1), (2, 32, 128, 128, 3, 2),
                                                    (2, 32, 256, 512, 1, 2), (2, 16, 48, 96, 3, 1)])
@pytest.mark.parametrize('mode', ['simt', 'tf32x3'])
@pytest.mark.parametrize('order,with_res', [(0, False), (0, True), (1, False)])
def test_conv2d_with_folded_eval_batchnorm(ops, N, H, Cin, Cout, k, stride, mode, order, with_res):
    """rih_conv2d_bn_eval_fwd (eval-mode BatchNorm, residual and final ReLU in the convolution's epilogue; scale / shift from rih_bn_fold) against
    torch: order 0 = Conv -> BN -> (+res) -> ReLU (torchvision Bottleneck.forward), order 1 = Conv -> ReLU -> BN (models/encoder.py:52-54)."""
    torch.manual_seed(Cin + Cout + k)
    conv = torch.nn.Conv2d(Cin, Cout, k, stride, k // 2, bias=False).to(DEV)
    conv.weight.data = conv.weight.data.contiguous(memory_format=torch.channels_last)
    bn = torch.nn.BatchNorm2d(Cout).to(DEV).eval()
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5); bn.bias.normal_(); bn.running_mean.normal_(); bn.running_var.uniform_(0.5, 2.0)
    holder = torch.nn.Sequential(conv, bn)
    x = T(N, Cin, H, H, grad=False)
    Ho = (H + 2 * (k // 2) - k) // stride + 1
    res = T(N, Cout, Ho, Ho, seed=3, grad=False) if with_res else None
    rows = lambda t: t.permute(0, 2, 3, 1).contiguous().reshape(-1, t.shape[1])
    with torch.no_grad():
        assert ops.bn_fold_refresh(holder)
        ops.set_gemm_mode(mode, mode)
        try:
            y = ops.conv2d_bn_eval(rows(x), conv.weight, N, H, H, stride, k // 2, bn._rih_fold, order=order, relu=True,
                                   res=rows(res) if with_res else None)
        finally:
            ops.set_gemm_mode('simt', 'simt')
        c = F.conv2d(x.double(), conv.weight.double(), None, stride, k // 2)
        bnd = lambda t: F.batch_norm(t, bn.running_mean.double(), bn.running_var.double(), bn.weight.double(), bn.bias.double(), False, 0.0, bn.eps)
        if order == 0:
            r = bnd(c)
            if with_res:
                r = r + res.double()
            r = F.relu(r)
        else:
            r = bnd(F.relu(c))
    assert rel(y, rows(r).float()) < 2e-5, rel(y, rows(r).float())


def test_bn_fold_tracks_live_running_statistics(ops):
    """The fold table reads the BatchNorm storage at every refresh: changing the running statistics in place (what training does between two
    evaluations) changes the folded vectors without rebuilding anything."""
    bn = torch.nn.BatchNorm2d(64).to(DEV).eval()
    root = torch.nn.Sequential(bn, torch.nn.BatchNorm2d(48).to(DEV).eval())
    with torch.no_grad():
        assert ops.bn_fold_refresh(root)
        s0 = bn._rih_fold[0].clone()
        bn.running_var.mul_(4.0)
        root[1].bias.add_(1.0)
        assert ops.bn_fold_refresh(root)
        assert rel(bn._rih_fold[0], s0 * ((bn.running_var / 4 + bn.eps) / (bn.running_var + bn.eps)).sqrt()) < 1e-6
        b1 = root[1]
        ref_shift = b1.bias - b1.running_mean * b1.weight / (b1.running_var + b1.eps).sqrt()
        assert rel(b1._rih_fold[1], ref_shift) < 1e-6
    assert not ops.bn_fold_refresh(root)          # gradients enabled: the folded inference path is off


@pytest.mark.parametrize('opt', [0, 1, 2, 3, 7])
@pytest.mark.parametrize('M,N,K,mode', [(8064, 256, 256, 'tf32x3'), (4032, 128, 256, 'tf32x3'), (1000, 64, 64, 'tf32x3'), (16384, 256, 64, 'tf32')])
def test_epilogue_options_linear_with_bias_and_residual(ops, opt, M, N, K, mode):
    """rih_set_epilogue_opt: residual prefetch (bit 0), column vectors in shared memory (bit 1) and warp-wide TMA issue (bit 2) are pure
    re-schedulings of the same arithmetic: y = x W^T + b + res must not depend on them (ragged M: 1000 rows)."""
    from renderih_b200._lib import call
    x, w, b, res = T(M, K, grad=False), T(N, K, scale=K ** -0.5, seed=1, grad=False), T(N, seed=2, grad=False), T(M, N, seed=3, grad=False)
    call('rih_set_epilogue_opt', opt)
    ops.set_gemm_mode(mode, mode)
    try:
        with torch.no_grad():
            y = ops.linear(x, w, b, res=res)
    finally:
        ops.set_gemm_mode('simt', 'simt')
        call('rih_set_epilogue_opt', 7)
    ref = (x.double() @ w.double().t() + b.double() + res.double()).float()
    tol = 2e-5 if mode == 'tf32x3' else 3e-3
    assert rel(y, ref) < tol, rel(y, ref)


@pytest.mark.parametrize('opt', [0, 3])
def test_epilogue_options_folded_conv_with_residual(ops, opt):
    """conv3 + bn3 + identity + ReLU of a layer1 bottleneck (1x1, 64 -> 256) with every epilogue option off / on."""
    from renderih_b200._lib import call
    N, H, Cin, Cout = 2, 64, 64, 256
    conv = torch.nn.Conv2d(Cin, Cout, 1, bias=False).to(DEV)
    conv.weight.data = conv.weight.data.contiguous(memory_format=torch.channels_last)
    bn = torch.nn.BatchNorm2d(Cout).to(DEV).eval()
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5); bn.bias.normal_(); bn.running_mean.normal_(); bn.running_var.uniform_(0.5, 2.0)
    x, res = T(N, Cin, H, H, grad=False), T(N, Cout, H, H, seed=5, grad=False)
    rows = lambda t: t.permute(0, 2, 3, 1).contiguous().reshape(-1, t.shape[1])
    call('rih_set_epilogue_opt', opt)
    ops.set_gemm_mode('tf32x3', 'tf32x3')
    try:
        with torch.no_grad():
            assert ops.bn_fold_refresh(torch.nn.Sequential(bn))
            y = ops.conv2d_bn_eval(rows(x), conv.weight, N, H, H, 1, 0, bn._rih_fold, order=0, relu=True, res=rows(res))
    finally:
        ops.set_gemm_mode('simt', 'simt')
        call('rih_set_epilogue_opt', 7)
    with torch.no_grad():
        r = F.relu(F.batch_norm(F.conv2d(x.double(), conv.weight.double()), bn.running_mean.double(), bn.running_var.double(), bn.weight.double(),
                                bn.bias.double(), False, 0.0, bn.eps) + res.double())
    assert rel(y, rows(r).float()) < 2e-5, rel(y, rows(r).float())


@pytest.mark.parametrize('opt', [3, 7])
@pytest.mark.parametrize('N,H,Cin,Cout,k,stride', [(4, 64, 64, 64, 3, 1), (4, 32, 128, 128, 3, 2), (2, 64, 48, 48, 3, 1), (4, 32, 256, 64, 1, 1)])
def test_warp_wide_tma_issue_conv_forward_and_gradients(ops, opt, N, H, Cin, Cout, k, stride):
    """rih_set_epilogue_opt bit 2: every lane of the producer warp issues its share of a k-block's TMA boxes (forward: A + B box from two
    lanes; dgrad: 1 + BN / 32 boxes; wgrad: 4 + BN / 32 four-KB boxes with per-chunk tap coordinates) -- same results as single-thread issue."""
    from renderih_b200._lib import call
    x = T(N, Cin, H, H)
    w = (torch.randn(Cout, Cin, k, k) * (Cin * k * k) ** -0.5).to(DEV).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    xr = x.permute(0, 2, 3, 1).contiguous().reshape(N * H * H, Cin)
    call('rih_set_epilogue_opt', opt)
    ops.set_gemm_mode('tf32x3', 'tf32x3')
    try:
        y = ops.conv2d(xr, w, None, N, H, H, stride=stride, pad=k // 2)
        g_ours = grads(y, [x, w])
    finally:
        ops.set_gemm_mode('simt', 'simt')
        call('rih_set_epilogue_opt', 7)
    yr = F.conv2d(x, w, None, stride=stride, padding=k // 2).permute(0, 2, 3, 1).reshape(-1, Cout)
    assert rel(y, yr) < 1e-4, rel(y, yr)
    for a, r, n in zip(g_ours, grads(yr, [x, w]), 'xw'):
        assert rel(a, r) < 1e-4, (n, rel(a, r))
