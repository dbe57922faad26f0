"""Backward of the token decoder in the arithmetic bench.py runs (3xTF32 Linears and attention contractions) against plain fp64 torch.

The decoder has no BatchNorm, and its Linears and attention contractions run 3xTF32 in the bench arithmetic, so the autograd plumbing
only that arithmetic runs can be held to fp32-faithful tolerances op by op:

  1. the fused projection + attention node (ops.attention_proj / AttnProjFn): q, k, v as column slices of one buffer, one dgrad / wgrad GEMM
     over the stacked weights, self / cross (Sk = V + 64) / inter attention (two nodes sharing one set of weights), adjacent, separate and
     flat-buffer weights, the longest key sequence, and dropout whose mask backward regenerates from (seed, site).  The launches are
     recorded, so each case also asserts the branch that ran (GEMM widths, row strides, split count, dq / dk / dv slices);
  2. alias outputs (layernorm / cheb / conv2d with alias_input=True): the residual branch's gradient accumulated in place by the backward
     kernel when it arrives contiguous, added after it otherwise;
  3. direct flat-gradient targets (train.FlatParams): every backward with a `_gt` branch accumulates into the prefilled flat buffer, with the
     side-stream weight gradients on and off, read on the caller's stream without a synchronize;
  4. the whole decoder (model.decoder, train mode, dropout 0) against oracle.model_ref.decoder_forward in fp64, plain autograd and with the
     FlatParams targets TrainStep installs.

Every error is max |ours - fp64| / max |fp64| per tensor; the gradient of w_ks.bias is mathematically zero (softmax shift invariance) and is
measured against the largest bias gradient of the same projection instead.  Tolerances are about 4x the worst error measured on an H100
80GB HBM3 (700 W power limit), given in brackets:

  attention_proj (section 1):  'simt' 4e-6 [8.3e-7], 'tf32x3' 3e-5 [7.2e-6], single-pass 'tf32' 1.5e-2 [4.0e-3];
                               fused vs unfused (FUSED['qkv'] off) 1e-5 [2.7e-6]; dropout directional derivative 5e-6 [1.2e-6]
  alias outputs (section 2):   2e-5 [5.0e-6]; blocks with FUSED['alias'] on vs off 3e-6 [5.9e-7; outputs bit-identical]
  flat targets (section 3):    4e-5 [1.0e-5] in 3xTF32
  whole decoder (section 4):   outputs agree to 4e-6 in 'simt'; the gradients of this randomly initialised 3-level decoder are ill-conditioned
                               and worsen with the batch: plain torch fp32 (TF32 off) itself is 7.2e-5 (B=2) and 1.7e-2 (B=64) off fp64.
                               'simt'   B=2 1e-3 [2.4e-4], B=64 1e-1 [3.0e-2]
                               'tf32x3' (all GEMMs 3xTF32) B=2 3e-2 [8.6e-3], B=64 1e-1 [2.7e-2]; single-pass TF32 Linears and attention
                                        instead measure 2.4e-1 (B=2) and 4.4e-1 (B=64)
                               bench    ('tf32c' convolutions + 3xTF32 Linears) B=2 5e-1 [1.5e-1], B=64 4e-1 [1.1e-1]: the level-0 patch
                                        projection (8 px feature map, 8 x 8 grid: kernel = stride = 1) is not patchified into a Linear but
                                        runs as a convolution, in single-pass TF32, and dominates; this case guards against gross errors only
"""
import contextlib

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False

DEV = 'cuda'
F64 = torch.float64
H = 4                                                   # attention heads of every decoder attention
ATTN_TOL = {'simt': 4e-6, 'tf32x3': 3e-5, 'tf32': 1.5e-2}
UNFUSED_TOL, DROPOUT_TOL = 1e-5, 5e-6
ALIAS_TOL, BLOCK_TOL, DIRECT_TOL = 2e-5, 3e-6, 4e-5
DECODER_TOL = {('simt', 2): 1e-3, ('simt', 64): 1e-1, ('tf32x3', 2): 3e-2, ('tf32x3', 64): 1e-1, ('bench', 2): 5e-1, ('bench', 64): 4e-1}
DECODER_ARITH = {'simt': ('simt', 'simt'), 'tf32x3': ('tf32x3', 'tf32x3'), 'bench': ('tf32c', 'tf32x3')}
# (B, V, HD): the three decoder levels (63 / 126 / 252 vertices, HD = 256 / 128 / 64, so d = 64 / 32 / 16) at batch 2, 1 and 64
ATTN_SHAPES = [(2, 63, 256), (1, 126, 128), (64, 252, 64)]
GRID = 64                                               # image-grid tokens: the cross attention of img_attn has Sk = V + 64


def rel(a, b, scale=None):
    a, b = a.detach().to(F64), b.detach().to(F64)
    assert a.shape == b.shape, (a.shape, b.shape)
    s = b.abs().max() if scale is None else scale
    return float((a - b).abs().max() / torch.as_tensor(s, dtype=F64).clamp_min(1e-30))


def report(tag, errs, tol):
    """Print every measured error, then fail on the ones at or above the tolerance."""
    print('%s: %s' % (tag, ', '.join('%s %.2e' % kv for kv in errs.items())))
    bad = {k: '%.2e' % e for k, e in errs.items() if not e < tol}
    assert not bad, '%s: over the tolerance %.1e: %s' % (tag, tol, bad)


def randn(*shape, gen, scale=1.0, grad=False):
    return (torch.randn(*shape, generator=gen) * scale).to(DEV).requires_grad_(grad)


def f64_leaf(t):
    return t.detach().to(F64).requires_grad_(True)


@pytest.fixture(scope='module')
def ops():
    from renderih_b200 import ops as o
    return o


@pytest.fixture(autouse=True)
def _restore_globals(ops):
    """Every global a test here changes: GEMM arithmetic, A/B switches, side-stream weight gradients, registered flat-gradient targets,
    the launch trace and the device-resident dropout seed."""
    from renderih_b200 import _lib
    mode, fused, wg = dict(ops.MODE), dict(ops.FUSED), ops._WG['enabled']
    seeds, site = {k: t.clone() for k, t in ops.seed_state.tensors.items()}, ops.seed_state.site
    try:
        yield
    finally:
        _lib.TRACE = None
        ops.set_gemm_mode(mode['conv'], mode['linear'])
        ops.FUSED.clear(); ops.FUSED.update(fused)
        ops._WG['enabled'] = wg
        ops.clear_grad_targets()
        for k in list(ops.seed_state.tensors):
            if k in seeds:
                ops.seed_state.tensors[k].copy_(seeds[k])
            else:
                del ops.seed_state.tensors[k]
        ops.seed_state.site = site


@contextlib.contextmanager
def launch_trace():
    """(name, args) of every kernel-launching call issued inside the block."""
    from renderih_b200 import _lib
    _lib.TRACE = []
    calls = []
    try:
        yield calls
    finally:
        calls.extend((n, a) for n, a, _, _ in _lib.TRACE)
        _lib.TRACE = None


def flat_params(params, groups, gen):
    """train.FlatParams over `params` (TrainStep's grouping), its gradient prefilled with random values -> (FlatParams, prefill)."""
    from renderih_b200.train import FlatParams
    fp = FlatParams(params, groups=groups)
    prefill = torch.randn(fp.numel, generator=gen).to(DEV)
    fp.grad.copy_(prefill)
    return fp, prefill


def flat_deltas(fp, prefill):
    """{param: gradient accumulated on top of the prefill}, computed on the current stream (no synchronize: the autograd-engine callback
    that joins the side streams is what orders it); also checks that every .grad is still its view of the flat buffer."""
    delta = fp.grad.to(F64) - prefill.to(F64)
    out = {}
    for p, off in zip(fp.params, fp.offsets):
        assert p.grad is not None and p.grad.data_ptr() == fp.grad.data_ptr() + 4 * off, 'gradient left the flat buffer'
        out[p] = torch.as_strided(delta, p.shape, p.stride(), off)
    return out


def scatter_storage(params):
    """Give every tensor its own place with a gap after it, so that no two of them are adjacent in memory."""
    buf = torch.zeros(sum(p.numel() + 64 for p in params), device=DEV)
    off = 0
    with torch.no_grad():
        for p in params:
            v = buf[off:off + p.numel()].view(p.shape)
            v.copy_(p.data)
            p.data = v
            off += p.numel() + 64


# ============================================================================ 1. fused projections + attention core
def ref_attention(xq, xkv, W, b, B, Sq):
    q, k, v = F.linear(xq, W[0], b[0]), F.linear(xkv, W[1], b[1]), F.linear(xkv, W[2], b[2])
    HD = q.shape[1]
    d = HD // H
    qh, kh, vh = (t.view(B, -1, H, d).transpose(1, 2) for t in (q, k, v))
    a = F.softmax(torch.matmul(qh, kh.transpose(-1, -2)) / d ** 0.5, -1)
    return torch.matmul(a, vh).transpose(1, 2).reshape(B * Sq, HD)


def attn_module(kind, HD, seed):
    from renderih_b200.model import SelfAttn, inter_attn
    torch.manual_seed(seed)
    m = inter_attn(HD, n_heads=H, dropout=0.0) if kind == 'inter' else SelfAttn(HD, n_heads=H, dropout=0.0)
    return m.to(DEV).train()


def run_proj(ops, kind, xs, lins, B, V, Sk, p_drop=0.0):
    """The decoder's calls: SelfAttn.forward (self), SelfAttn.forward_query_subset (cross), inter_attn.forward (both directions)."""
    if kind == 'self':
        return [ops.attention_proj(xs[0], None, *lins, B, H, V, V, p_drop=p_drop)]
    if kind == 'cross':
        return [ops.attention_proj(xs[0], xs[1], *lins, B, H, V, Sk, p_drop=p_drop)]
    return [ops.attention_proj(xs[0], xs[1], *lins, B, H, V, V, p_drop=p_drop),
            ops.attention_proj(xs[1], xs[0], *lins, B, H, V, V, p_drop=p_drop)]


def proj_case(ops, monkeypatch, mode, kind, layout, B, V, HD, Sk=None, seed=0):
    """One forward + backward of the fused node(s) and of its fp64 restatement -> (errors, fp64 reference scale, launch trace)."""
    Sk = Sk or (V + GRID if kind == 'cross' else V)
    m = attn_module(kind, HD, seed=V + HD + seed)
    lins = (m.w_qs, m.w_ks, m.w_vs)
    params = [t for lin in lins for t in (lin.weight, lin.bias)]          # the module's parameter order (what TrainStep hands FlatParams)
    gen = torch.Generator().manual_seed(HD + seed)
    xs = [randn(B * V, HD, gen=gen, grad=True)]
    if kind != 'self':
        xs.append(randn(B * Sk, HD, gen=gen, grad=True))
    cots = [randn(B * V, HD, gen=gen) for _ in range(2 if kind == 'inter' else 1)]
    fp = None
    if layout == 'separate':
        scatter_storage(params)
        monkeypatch.setattr(ops, 'fuse_storage', lambda ps: False)
    elif layout == 'flat':
        fp, prefill = flat_params(params, m.fused_param_groups(), gen)
    ops.set_gemm_mode('simt', mode)
    with launch_trace() as calls:
        outs = run_proj(ops, kind, xs, lins, B, V, Sk)
        sum((o * w).sum() for o, w in zip(outs, cots)).backward()
    ops.set_gemm_mode('simt', 'simt')
    if layout == 'flat':
        dp = flat_deltas(fp, prefill)
        grads = [dp[t] for t in params]
    else:
        grads = [t.grad for t in params]
    if layout == 'adjacent':
        assert ops.adjacent([m.w_ks.weight, m.w_vs.weight]) and (kind != 'self' or ops.adjacent([l.weight for l in lins]))
    elif layout == 'separate':
        assert not ops.adjacent([m.w_ks.weight, m.w_vs.weight]) and not ops.adjacent([m.w_ks.bias, m.w_vs.bias])

    Wd = [f64_leaf(l.weight) for l in lins]
    bd = [f64_leaf(l.bias) for l in lins]
    xd = [f64_leaf(x) for x in xs]
    if kind == 'self':
        refs = [ref_attention(xd[0], xd[0], Wd, bd, B, V)]
    elif kind == 'cross':
        refs = [ref_attention(xd[0], xd[1], Wd, bd, B, V)]
    else:
        refs = [ref_attention(xd[0], xd[1], Wd, bd, B, V), ref_attention(xd[1], xd[0], Wd, bd, B, V)]
    sum((o * w.to(F64)).sum() for o, w in zip(refs, cots)).backward()

    errs = {}
    for i, (o, r) in enumerate(zip(outs, refs)):
        errs['o%d' % i] = rel(o, r)
    for i, (x, r) in enumerate(zip(xs, xd)):
        errs['dx%d' % i] = rel(x.grad, r.grad)
    for n, g, r in zip(('dWq', 'dbq', 'dWk', 'dbk', 'dWv', 'dbv'), grads, [t.grad for wb in zip(Wd, bd) for t in wb]):
        if n == 'dbk':      # mathematically zero: absolute, against the scale of the other bias gradients
            errs[n] = rel(g, r, scale=max(bd[0].grad.abs().max(), bd[2].grad.abs().max()))
        else:
            errs[n] = rel(g, r)
    return errs, calls


def check_attention_launches(calls, kind, layout, mode, HD, fallback=False):
    """The branch that ran: projection GEMM widths, the attention kernels and their row strides / split count, and the dq / dk / dv slices
    of the one gradient buffer."""
    n_nodes = 2 if kind == 'inter' else 1
    names = [n for n, _ in calls]
    widths = lambda name, idx: sorted(a[idx] for n, a in calls if n == name)
    if kind == 'self':
        proj = [3 * HD] if layout != 'separate' else [HD] * 3
    else:
        proj = sorted(([HD, 2 * HD] if layout != 'separate' else [HD] * 3) * n_nodes)
    assert widths('rih_linear_fwd', 8) == proj, widths('rih_linear_fwd', 8)
    assert widths('rih_linear_dgrad', 7) == proj, widths('rih_linear_dgrad', 7)
    assert widths('rih_linear_wgrad', 7) == ([3 * HD] if (kind == 'self' and layout != 'separate') else [HD] * 3 * n_nodes)
    if mode == 'simt' or fallback:
        assert names.count('rih_attn_fwd') == names.count('rih_attn_bwd') == n_nodes and 'rih_attn_tc_fwd' not in names
        return
    nsplit = {'tf32x3': 3, 'tf32': 1}[mode]
    ldq, ldkv = (3 * HD, 3 * HD) if kind == 'self' else (HD, 2 * HD)
    fwd = [a for n, a in calls if n == 'rih_attn_tc_fwd']
    bwd = [a for n, a in calls if n == 'rih_attn_tc_bwd']
    assert len(fwd) == len(bwd) == n_nodes and 'rih_attn_fwd' not in names
    for a in fwd:
        assert (a[1], a[3], a[5], a[20]) == (ldq, ldkv, ldkv, nsplit), (a[1], a[3], a[5], a[20])
        assert a[4] - a[2] == 4 * HD and (kind != 'self' or a[2] - a[0] == 4 * HD), 'q / k / v are not slices of one buffer'
    for a in bwd:
        assert (a[1], a[3], a[5], a[13], a[15], a[17], a[27]) == (ldq, ldkv, ldkv, ldq, ldkv, ldkv, nsplit)
        assert a[16] - a[14] == 4 * HD and (kind != 'self' or a[14] - a[12] == 4 * HD), 'dk / dv are not the k / v slices of the gradient'


@pytest.mark.parametrize('B,V,HD', ATTN_SHAPES)
@pytest.mark.parametrize('layout', ['adjacent', 'separate', 'flat'])
@pytest.mark.parametrize('kind', ['self', 'cross', 'inter'])
@pytest.mark.parametrize('mode', ['simt', 'tf32x3', 'tf32'])
def test_attention_proj_matches_fp64(ops, monkeypatch, mode, kind, layout, B, V, HD):
    """Output, input gradients and every weight / bias gradient of the fused node against fp64 (tolerances in the module docstring).
    'flat' = the parameters in a FlatParams laid out by the module's fused_param_groups(), side-stream weight gradients on."""
    errs, calls = proj_case(ops, monkeypatch, mode, kind, layout, B, V, HD)
    check_attention_launches(calls, kind, layout, mode, HD)
    report('attention_proj %s %s %s B=%d V=%d HD=%d' % (mode, kind, layout, B, V, HD), errs, ATTN_TOL[mode])


def test_attention_proj_longest_key_sequence(ops, monkeypatch):
    """Sk = 512 is the longest key sequence of the tensor-core core: the fused node still takes it and matches fp64.  Above it the node
    falls back to the SIMT core, which stops at 512 keys as well: Sk = 520 must fail loudly, in either arithmetic, rather than compute."""
    errs, calls = proj_case(ops, monkeypatch, 'tf32x3', 'cross', 'adjacent', 2, 63, 64, Sk=512)
    check_attention_launches(calls, 'cross', 'adjacent', 'tf32x3', 64)
    report('attention_proj cross Sk=512', errs, ATTN_TOL['tf32x3'])
    for mode in ('simt', 'tf32x3'):
        with pytest.raises(RuntimeError, match='unsupported'):
            proj_case(ops, monkeypatch, mode, 'cross', 'adjacent', 2, 63, 64, Sk=520)
        ops.set_gemm_mode('simt', 'simt')


@pytest.mark.parametrize('B,V,HD', [(2, 63, 256), (64, 252, 64)])
@pytest.mark.parametrize('kind', ['self', 'cross', 'inter'])
@pytest.mark.parametrize('mode', ['simt', 'tf32x3'])
def test_attention_proj_matches_unfused_projections(ops, mode, kind, B, V, HD):
    """FUSED['qkv'] off (separate ops.linear projections + ops.attention) and on agree to fp32 reordering."""
    Sk = V + GRID if kind == 'cross' else V
    res = {}
    for fused in (True, False):
        m = attn_module(kind, HD, seed=7)
        gen = torch.Generator().manual_seed(11)
        xs = [randn(B * V, HD, gen=gen, grad=True)] + ([randn(B * Sk, HD, gen=gen, grad=True)] if kind != 'self' else [])
        cots = [randn(B * V, HD, gen=gen) for _ in range(2)]
        ops.FUSED['qkv'] = fused
        ops.set_gemm_mode('simt', mode)
        outs = run_proj(ops, kind, xs, (m.w_qs, m.w_ks, m.w_vs), B, V, Sk)
        sum((o * w).sum() for o, w in zip(outs, cots)).backward()
        ops.set_gemm_mode('simt', 'simt')
        res[fused] = [o.detach() for o in outs] + [x.grad for x in xs] + \
                     [t.grad for l in (m.w_qs, m.w_ks, m.w_vs) for t in (l.weight, l.bias)]
    names = ['o%d' % i for i in range(2 if kind == 'inter' else 1)] + ['dx%d' % i for i in range(1 if kind == 'self' else 2)] + \
            ['dWq', 'dbq', 'dWk', 'dbk', 'dWv', 'dbv']
    errs = {n: rel(a, b, scale=(res[False][-1].abs().max() if n == 'dbk' else None))
            for n, a, b in zip(names, res[True], res[False])}
    report('attention_proj fused vs unfused %s %s B=%d V=%d' % (mode, kind, B, V), errs, UNFUSED_TOL)


@pytest.mark.parametrize('kind', ['self', 'cross'])
@pytest.mark.parametrize('mode', ['simt', 'tf32x3'])
def test_attention_proj_dropout_backward_regenerates_forward_mask(ops, mode, kind):
    """Probability dropout p = 0.05 (the training configuration): for a fixed (seed, site) the output is linear in Wv and bv, so
    <cotangent, o(Wv + D, bv + e) - o(Wv, bv)> must equal the directional derivative <dL/dWv, D> + <dL/dbv, e> that backward computed.
    A backward that drew another mask than forward (or read it through the wrong slice) misses by about p; stated tolerance 1e-4."""
    B, V, HD, p = 2, 126, 128, 0.05
    Sk = V + GRID if kind == 'cross' else V
    dev = torch.device(DEV, torch.cuda.current_device())
    m = attn_module(kind, HD, seed=3)
    lins = (m.w_qs, m.w_ks, m.w_vs)
    gen = torch.Generator().manual_seed(5)
    xs = [randn(B * V, HD, gen=gen)] + ([randn(B * Sk, HD, gen=gen)] if kind != 'self' else [])
    cot = randn(B * V, HD, gen=gen).to(F64)
    D = randn(HD, HD, gen=gen, scale=float(m.w_vs.weight.detach().std()))
    e = randn(HD, gen=gen, scale=float(m.w_vs.bias.detach().std()))
    ops.seed_state.manual_seed(4321, dev)

    def forward(p_drop):
        ops.seed_state.begin_forward()
        ops.set_gemm_mode('simt', mode)
        try:
            return run_proj(ops, kind, xs, lins, B, V, Sk, p_drop=p_drop)[0]
        finally:
            ops.set_gemm_mode('simt', 'simt')
    o1 = forward(p)
    (o1.to(F64) * cot).sum().backward()
    with torch.no_grad():
        o0 = forward(0.0)
        w0, b0 = m.w_vs.weight.detach().clone(), m.w_vs.bias.detach().clone()
        m.w_vs.weight.add_(D); m.w_vs.bias.add_(e)
        o2 = forward(p)
        m.w_vs.weight.copy_(w0); m.w_vs.bias.copy_(b0)
    assert rel(o1, o0) > 1e-2, 'dropout did not change the output'
    lhs = float(((o2.to(F64) - o1.detach().to(F64)) * cot).sum())
    rhs = float((m.w_vs.weight.grad.to(F64) * D).sum() + (m.w_vs.bias.grad.to(F64) * e).sum())
    report('attention_proj dropout %s %s' % (mode, kind), {'directional derivative': abs(lhs - rhs) / abs(rhs)}, DROPOUT_TOL)


# ============================================================================ 2. alias outputs
def alias_case(ops, op, mode, use):
    """-> (our leaves, our loss, fp64 leaves, fp64 loss).  `use` is how the alias output is consumed: 'contiguous' = by a Linear /
    convolution whose input gradient arrives dense (accumulated in place by the backward kernel), 'transposed' / 'expanded' = by a view
    whose gradient arrives non-contiguous (added afterwards), 'unused'."""
    gen = torch.Generator().manual_seed(23)

    def alias_term(alias, alias_d, consumer, consumer_d):
        if use == 'contiguous':
            y = consumer(alias)
            w = randn(*y.shape, gen=gen)
            return (y * w).sum(), (consumer_d(alias_d) * w.to(F64)).sum()
        if use == 'transposed':
            w = randn(alias.shape[1], alias.shape[0], gen=gen)
            return (alias.t() * w).sum(), (alias_d.t() * w.to(F64)).sum()
        if use == 'expanded':
            w = randn(alias.shape[1], gen=gen)
            return (alias.sum(0) * w).sum(), (alias_d.sum(0) * w.to(F64)).sum()
        return 0.0, 0.0

    if op == 'layernorm':            # pre-LN block: h, x = LN(x) ; y = fc(h) + x
        M, Fd = 64 * 63, 256
        x = randn(M, Fd, gen=gen, grad=True)
        gam, bet = randn(Fd, gen=gen, scale=0.5, grad=True), randn(Fd, gen=gen, scale=0.5, grad=True)
        W, b = randn(Fd, Fd, gen=gen, scale=Fd ** -0.5, grad=True), randn(Fd, gen=gen, grad=True)
        leaves = [x, gam, bet, W, b]
        h, xa = ops.layernorm(x, gam, bet, alias_input=True)
        y = ops.linear(h, W, b, res=xa if use == 'contiguous' else None)
        d = [f64_leaf(t) for t in leaves]
        yd = F.linear(F.layer_norm(d[0], (Fd,), d[1], d[2], 1e-6), d[3], d[4]) + (d[0] if use == 'contiguous' else 0)
        w = randn(M, Fd, gen=gen)
        t, td = alias_term(xa, d[0], None, None) if use != 'contiguous' else (0.0, 0.0)
        return leaves, (y * w).sum() + t, d, (yd * w.to(F64)).sum() + td
    if op == 'cheb':                 # GCN_ResBlock: c, x = cheb(x) ; fc1(c) ... + shortcut(x)
        from renderih_b200 import assets
        from renderih_b200.model import GraphCSR
        g = GraphCSR(assets.synthetic_assets(3)['left_graph']['coarsen_graphs_L'][2]).to(torch.device(DEV))     # 252 vertices
        Ld = g.dense().to(DEV, F64)
        B, V, Fd, Fo = 4, 252, 64, 64
        x = randn(B * V, Fd, gen=gen, grad=True)
        W1, b1 = randn(Fo, 2 * Fd, gen=gen, scale=(2 * Fd) ** -0.5, grad=True), randn(Fo, gen=gen, grad=True)
        Ws, bs = randn(Fo, Fd, gen=gen, scale=Fd ** -0.5, grad=True), randn(Fo, gen=gen, grad=True)
        leaves = [x, W1, b1, Ws, bs]
        c, xa = ops.cheb(x, g, B, V, alias_input=True)
        y = ops.linear(c, W1, b1)
        d = [f64_leaf(t) for t in leaves]
        x3 = d[0].view(B, V, Fd)
        cd = torch.stack([x3, torch.einsum('vu,buf->bvf', Ld, x3)], -1).reshape(B * V, 2 * Fd)
        yd = F.linear(cd, d[1], d[2])
        w = randn(B * V, Fo, gen=gen)
        t, td = alias_term(xa, d[0], lambda a: ops.linear(a, Ws, bs), lambda a: F.linear(a, d[3], d[4]))
        return leaves, (y * w).sum() + t, d, (yd * w.to(F64)).sum() + td
    # conv2d: Bottleneck conv1 with the downsample shortcut on the alias: y = conv1(x), x = alias ; downsample(x)
    N, Hh, Cin, Cout, Cds = 2, 16, 64, 64, 256
    x = randn(N * Hh * Hh, Cin, gen=gen, grad=True)
    w1 = randn(Cout, Cin, 1, 1, gen=gen, scale=Cin ** -0.5).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    wd = randn(Cds, Cin, 1, 1, gen=gen, scale=Cin ** -0.5).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    leaves = [x, w1, wd]
    y, xa = ops.conv2d(x, w1, None, N, Hh, Hh, alias_input=True)
    d = [f64_leaf(t) for t in leaves]
    nchw = lambda r: r.view(N, Hh, Hh, -1).permute(0, 3, 1, 2)
    rows = lambda t: t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])
    yd = rows(F.conv2d(nchw(d[0]), d[1]))
    w = randn(N * Hh * Hh, Cout, gen=gen)
    t, td = alias_term(xa, d[0], lambda a: ops.conv2d(a, wd, None, N, Hh, Hh), lambda a: rows(F.conv2d(nchw(a), d[2])))
    return leaves, (y * w).sum() + t, d, (yd * w.to(F64)).sum() + td


@pytest.mark.parametrize('use', ['contiguous', 'transposed', 'expanded', 'unused'])
@pytest.mark.parametrize('mode', ['simt', 'tf32x3'])
@pytest.mark.parametrize('op', ['layernorm', 'cheb', 'conv2d'])
def test_alias_output_gradients_match_fp64(ops, op, mode, use):
    """Input and parameter gradients through an alias output against fp64, for each way its gradient can arrive."""
    ops.set_gemm_mode(mode, mode)
    try:
        leaves, loss, d, loss_d = alias_case(ops, op, mode, use)
        loss.backward()
    finally:
        ops.set_gemm_mode('simt', 'simt')
    loss_d.backward()
    errs = {}
    for i, (a, r) in enumerate(zip(leaves, d)):
        if r.grad is None:          # the shortcut's parameters when the alias output is not consumed by it
            assert a.grad is None, i
        else:
            errs['d%d' % i] = rel(a.grad, r.grad)
    report('alias %s %s %s' % (op, mode, use), errs, ALIAS_TOL)


def block_case(block, seed):
    """-> (module, inputs, forward) at the decoder's shapes, dropout 0."""
    from renderih_b200 import assets
    from renderih_b200.model import GCN_ResBlock, GraphCSR, MLP_res_block, SelfAttn, inter_attn
    torch.manual_seed(seed)
    gen = torch.Generator().manual_seed(seed)
    if block == 'GCN_ResBlock':
        g = GraphCSR(assets.synthetic_assets(3)['left_graph']['coarsen_graphs_L'][2])
        m = GCN_ResBlock(64, 64, 64, g, 2, 0.0)
        xs = [randn(4 * 252, 64, gen=gen, grad=True)]
        fwd = lambda m, xs: [m(xs[0], 4, 252, relu_out=True)]
    elif block == 'MLP_res_block':
        m = MLP_res_block(256, 256, 0.0)
        xs = [randn(8 * 63, 256, gen=gen, grad=True)]
        fwd = lambda m, xs: [m(xs[0])]
    elif block == 'SelfAttn':
        m = SelfAttn(128, hid_dim=128, n_heads=H, dropout=0.0)
        xs = [randn(2 * 126, 128, gen=gen, grad=True)]
        fwd = lambda m, xs: [m(xs[0], 2, 126)]
    else:
        m = inter_attn(256, n_heads=H, dropout=0.0)
        xs = [randn(2 * 63, 256, gen=gen, grad=True), randn(2 * 63, 256, gen=gen, grad=True)]
        fwd = lambda m, xs: list(m(xs[0], xs[1], 2, 63))
    return m.to(DEV).train(), xs, fwd


@pytest.mark.parametrize('mode', ['simt', 'tf32x3'])
@pytest.mark.parametrize('block', ['GCN_ResBlock', 'MLP_res_block', 'SelfAttn', 'inter_attn'])
def test_block_gradients_with_and_without_alias_outputs_agree(ops, block, mode):
    """The decoder blocks with FUSED['alias'] on (residual gradients summed inside the backward kernels) and off (autograd adds):
    outputs, input and parameter gradients agree to fp32 reordering."""
    res = {}
    for alias in (True, False):
        m, xs, fwd = block_case(block, seed=17)
        ops.FUSED['alias'] = alias
        ops.set_gemm_mode(mode, mode)
        try:
            outs = fwd(m, xs)
            gen = torch.Generator().manual_seed(3)
            sum((o * randn(*o.shape, gen=gen)).sum() for o in outs).backward()
        finally:
            ops.set_gemm_mode('simt', 'simt')
        res[alias] = {'out%d' % i: o.detach() for i, o in enumerate(outs)}
        res[alias].update({'dx%d' % i: x.grad for i, x in enumerate(xs)})
        res[alias].update({'d' + n: p.grad for n, p in m.named_parameters() if p.grad is not None})
    assert res[True].keys() == res[False].keys()
    errs = {k: rel(res[True][k], v, scale=(res[False][k.replace('w_ks', 'w_qs')].abs().max() if k.endswith('w_ks.bias') else None))
            for k, v in res[False].items()}
    report('%s %s alias on vs off' % (block, mode), errs, BLOCK_TOL)


# ============================================================================ 3. direct flat-gradient targets
def direct_case(ops, fn, gen):
    """-> (parameters, other leaves, forward(), fp64 forward(fp64 parameters, fp64 leaves, our output))."""
    if fn.startswith('linear'):
        M, K, N = 1000, 256, 128
        W, b = randn(N, K, gen=gen, scale=K ** -0.5, grad=True), randn(N, gen=gen, grad=True)
        x = randn(M, K, gen=gen, grad=True)
        if fn == 'linear_res':      # the pre-LN block: LayerNorm-backward adds the residual gradient in place into the dy LinearFn returned
            gam, bet = randn(K, gen=gen, scale=0.5, grad=True), randn(K, gen=gen, grad=True)
            W, b = randn(K, K, gen=gen, scale=K ** -0.5, grad=True), randn(K, gen=gen, grad=True)

            def ours():
                h, xa = ops.layernorm(x, gam, bet, alias_input=True)
                return ops.linear(h, W, b, res=xa)
            return [W, b, gam, bet], [x], ours, lambda P, X, y: F.linear(F.layer_norm(X[0], (K,), P[2], P[3], 1e-6), P[0], P[1]) + X[0]
        if fn == 'linear_relu':
            return [W, b], [x], lambda: ops.linear(x, W, b, relu=True), lambda P, X, y: F.linear(X[0], P[0], P[1]) * (y > 0)
        if fn == 'linear_dropout':
            def ours():
                ops.seed_state.manual_seed(99, torch.device(DEV, torch.cuda.current_device()))
                ops.seed_state.begin_forward()
                return ops.linear(x, W, b, p_drop=0.25)
            return [W, b], [x], ours, lambda P, X, y: F.linear(X[0], P[0], P[1]) * (y != 0) / 0.75
        return [W, b], [x], lambda: ops.linear(x, W, b), lambda P, X, y: F.linear(X[0], P[0], P[1])
    if fn == 'layernorm':            # norm3 of GCN_ResBlock: LN(a + b), relu
        M, Fd = 2 * 252, 64
        a, b2 = randn(M, Fd, gen=gen, grad=True), randn(M, Fd, gen=gen, grad=True)
        gam, bet = randn(Fd, gen=gen, scale=0.5, grad=True), randn(Fd, gen=gen, grad=True)
        return [gam, bet], [a, b2], lambda: ops.layernorm(a, gam, bet, b=b2, relu=True), \
            lambda P, X, y: F.layer_norm(X[0] + X[1], (Fd,), P[0], P[1], 1e-6) * (y > 0)
    if fn == 'posemb':               # graph_upsample(x, 2) + the next level's position embeddings
        B, U, Fd = 3, 126, 128
        x = randn(B * U // 2, Fd, gen=gen, grad=True)
        emb = randn(U, Fd, gen=gen, grad=True)
        return [emb], [x], lambda: ops.posemb(x, emb, B, U, 2), \
            lambda P, X, y: (X[0].view(B, U // 2, Fd).repeat_interleave(2, dim=1) + P[0]).reshape(B * U, Fd)
    if fn == 'conv2d':
        N, Hh, Cin, Cout = 2, 16, 64, 128
        x = randn(N * Hh * Hh, Cin, gen=gen, grad=True)
        w = randn(Cout, Cin, 3, 3, gen=gen, scale=(9 * Cin) ** -0.5).contiguous(memory_format=torch.channels_last).requires_grad_(True)
        b = randn(Cout, gen=gen, grad=True)
        nchw = lambda r: r.view(N, Hh, Hh, -1).permute(0, 3, 1, 2)
        return [w, b], [x], lambda: ops.conv2d(x, w, b, N, Hh, Hh, stride=1, pad=1), \
            lambda P, X, y: F.conv2d(nchw(X[0]), P[0], P[1], padding=1).permute(0, 2, 3, 1).reshape(-1, Cout)
    # batchnorm: training statistics, + residual, relu (the end of a Bottleneck)
    M, C = 2048, 128
    x, r = randn(M, C, gen=gen, grad=True), randn(M, C, gen=gen, grad=True)
    gam, bet = randn(C, gen=gen, scale=0.5, grad=True), randn(C, gen=gen, grad=True)
    rm, rv = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)
    return [gam, bet], [x, r], lambda: ops.batchnorm(x, gam, bet, rm, rv, res=r, training=True, relu=True), \
        lambda P, X, y: (F.batch_norm(X[0], None, None, P[0], P[1], True, 0.1, 1e-5) + X[1]) * (y > 0)


@pytest.mark.parametrize('wg', [True, False], ids=['side_stream', 'same_stream'])
@pytest.mark.parametrize('fn', ['linear', 'linear_relu', 'linear_res', 'linear_dropout', 'layernorm', 'posemb', 'conv2d', 'batchnorm'])
def test_direct_flat_gradient_targets_accumulate_onto_prefill(ops, fn, wg):
    """Parameters re-homed into a FlatParams whose gradient is prefilled with random values: one backward must leave prefill + the fp64
    gradient in the buffer (an overwrite loses the prefill, an extra autograd accumulation doubles the gradient) and the fp64 input
    gradients in the leaves.  3xTF32 arithmetic."""
    gen = torch.Generator().manual_seed(31)
    params, leaves, ours, ref = direct_case(ops, fn, gen)
    fp, prefill = flat_params(params, (), gen)
    ops._WG['enabled'] = wg
    ops.set_gemm_mode('tf32x3', 'tf32x3')
    try:
        y = ours()
        w = randn(*y.shape, gen=gen)
        (y * w).sum().backward()
    finally:
        ops.set_gemm_mode('simt', 'simt')
    dp = flat_deltas(fp, prefill)
    P, X = [f64_leaf(p) for p in params], [f64_leaf(x) for x in leaves]
    (ref(P, X, y.detach()) * w.to(F64)).sum().backward()
    errs = {'dparam%d' % i: rel(dp[p], r.grad) for i, (p, r) in enumerate(zip(params, P))}
    errs.update({'dx%d' % i: rel(x.grad, r.grad) for i, (x, r) in enumerate(zip(leaves, X))})
    report('flat targets %s %s' % (fn, 'side stream' if wg else 'same stream'), errs, DIRECT_TOL)


@pytest.mark.parametrize('wg', [True, False], ids=['side_stream', 'same_stream'])
@pytest.mark.parametrize('kind', ['self', 'inter'])
def test_direct_flat_gradient_targets_attention_proj(ops, monkeypatch, kind, wg):
    """The fused node's direct branch: one N = 3 HD weight-gradient GEMM into the grouped targets (self) and two nodes accumulating into
    the same targets (inter), side-stream weight gradients on and off."""
    ops._WG['enabled'] = wg
    errs, calls = proj_case(ops, monkeypatch, 'tf32x3', kind, 'flat', 64, 63, 256, seed=1)
    check_attention_launches(calls, kind, 'flat', 'tf32x3', 256)
    assert all(a[9] == 1 for n, a in calls if n == 'rih_linear_wgrad'), 'a direct weight gradient does not accumulate'
    report('flat targets attention_proj %s %s' % (kind, 'side stream' if wg else 'same stream'), errs, DIRECT_TOL)


# ============================================================================ 4. the whole decoder
def decoder_outputs(out):
    result, params, hlist, other = out
    d = {}
    for s in ('left', 'right'):
        d['verts3d_' + s], d['verts2d_' + s] = result['verts3d'][s], result['verts2d'][s]
        d['scale_' + s], d['trans2d_' + s] = params['scale'][s], params['trans2d'][s]
        d['v3c_' + s], d['v2c_' + s] = hlist[0]['verts3d'][s], hlist[0]['verts2d'][s]
        d['v3list_' + s], d['v2list_' + s] = other['verts3d_MANO_list'][s][0], other['verts2d_MANO_list'][s][0]
    return d


@pytest.fixture(scope='module')
def decoder_setup():
    """The model's decoder with seeded weights in train mode, dropout 0, unsample_layer frozen (as the end-to-end tests run it), and a
    cache of fp64 reference results per batch size."""
    from oracle import fixtures, model_ref
    from renderih_b200 import assets
    from renderih_b200.config import load_cfg
    from renderih_b200.model import load_model
    a = assets.synthetic_assets(0)
    model = load_model(load_cfg(), assets=a)
    sd = fixtures.init_state_dict(model.state_dict())
    model.load_state_dict(sd)
    dec = model.decoder.to(DEV).train()
    for m in dec.modules():
        if hasattr(m, 'p'):
            m.p = 0.0
    dec.unsample_layer.weight.requires_grad_(False)
    dims = [(l.img_ex_left.encoder.proj.weight.shape[1], l.img_ex_left.encoder.img_size) for l in dec.dual_gcn.layers]
    return {'dec': dec, 'sd': sd, 'A': model_ref.prepare_assets(a), 'dims': dims, 'ref': {}}


def decoder_inputs(setup, B):
    """gf [B, gf_dim] and the three used feature maps as NHWC rows (+ the unused last level), seeded; the cotangents of every output."""
    gen = torch.Generator().manual_seed(1000 + B)
    gf = torch.randn(B, setup['dec'].gf_dim, generator=gen)
    fm = [torch.randn(B * Hh * Hh, C, generator=gen) for C, Hh in setup['dims']]
    return gf, fm, gen


def decoder_reference(setup, B):
    from oracle import model_ref
    if B in setup['ref']:
        return setup['ref'][B]
    gf, fm, gen = decoder_inputs(setup, B)
    sd = {k: v.to(DEV, F64) if v.is_floating_point() else v.to(DEV) for k, v in setup['sd'].items() if k.startswith('decoder.')}
    for k, v in sd.items():
        if v.is_floating_point() and k not in ('decoder.dense_coor', 'decoder.unsample_layer.weight'):
            v.requires_grad_(True)
    A = {s: dict(setup['A'][s], L=[L.to(DEV, F64) for L in setup['A'][s]['L']]) for s in ('left', 'right')}
    gfd = gf.to(DEV, F64).requires_grad_(True)
    fmd = [r.to(DEV, F64).requires_grad_(True) for r in fm]
    nchw = [r.view(B, Hh, Hh, C).permute(0, 3, 1, 2) for r, (C, Hh) in zip(fmd, setup['dims'])]
    outs = decoder_outputs(model_ref.decoder_forward(sd, A, gfd, nchw + [None], 0.0, True))
    cots = {k: torch.randn(v.shape, generator=gen, dtype=F64).to(DEV) for k, v in outs.items()}
    sum((v * cots[k]).sum() for k, v in outs.items()).backward()
    ref = {'out': {k: v.detach() for k, v in outs.items()}, 'cot': cots, 'dgf': gfd.grad, 'dfm': [r.grad for r in fmd],
           'dparam': {k[len('decoder.'):]: v.grad for k, v in sd.items() if v.requires_grad and v.grad is not None}}
    setup['ref'][B] = ref
    return ref


@pytest.mark.parametrize('B', [2, 64])
@pytest.mark.parametrize('variant', ['autograd', 'flat'])
@pytest.mark.parametrize('arith', ['simt', 'tf32x3', 'bench'])
def test_decoder_backward_matches_fp64(ops, decoder_setup, arith, variant, B):
    """model.decoder against oracle.model_ref.decoder_forward in fp64 on the same weights: every output, d(gf), d(fmaps[i]) and every
    decoder parameter gradient under a fixed random linear functional of all outputs.  'bench' = tf32c convolutions + 3xTF32 Linears and
    attention (what bench.py runs); 'flat' = the parameters re-homed into the FlatParams TrainStep installs (grouped Q/K/V, side-stream
    weight gradients), read without a synchronize.  Tolerances and measured errors in the module docstring."""
    from renderih_b200.train import FlatParams
    setup = decoder_setup
    dec = setup['dec']
    ref = decoder_reference(setup, B)
    gf, fm, _ = decoder_inputs(setup, B)
    gf = gf.to(DEV).requires_grad_(True)
    fm = [r.to(DEV).requires_grad_(True) for r in fm]
    named = dict(dec.named_parameters())
    for p in dec.parameters():
        p.grad = None
    fp = None
    if variant == 'flat':
        groups = [g for m in dec.modules() if hasattr(m, 'fused_param_groups') for g in m.fused_param_groups()]
        fp = FlatParams([named[k] for k in ref['dparam']], groups=groups)
    ops.set_gemm_mode(*DECODER_ARITH[arith])
    try:
        ops.seed_state.begin_forward()
        outs = decoder_outputs(dec(gf, [(r, Hh) for r, (C, Hh) in zip(fm, setup['dims'])] + [None]))
        sum((v * ref['cot'][k].float()).sum() for k, v in outs.items()).backward()
    finally:
        ops.set_gemm_mode('simt', 'simt')
        ops.clear_grad_targets()
    errs = {'out:' + k: rel(v, ref['out'][k]) for k, v in outs.items()}
    errs['d gf'] = rel(gf.grad, ref['dgf'])
    errs.update({'d fmaps[%d]' % i: rel(r.grad, rd) for i, (r, rd) in enumerate(zip(fm, ref['dfm']))})
    for k, p in named.items():
        if k not in ref['dparam']:
            assert p.grad is None or float(p.grad.abs().max()) == 0.0, ('gradient where the reference has none', k)
            continue
        r = ref['dparam'][k]
        if k.endswith('w_ks.bias'):
            errs['d ' + k] = rel(p.grad, r, scale=ref['dparam'][k.replace('w_ks', 'w_qs')].abs().max())
        else:
            errs['d ' + k] = rel(p.grad, r)
    if fp is not None:
        assert all(p.grad.data_ptr() == fp.grad.data_ptr() + 4 * off for p, off in zip(fp.params, fp.offsets))
    worst = sorted(errs.items(), key=lambda kv: -kv[1])
    tol = DECODER_TOL[arith, B]
    print('decoder %s %s B=%d: %d comparisons, worst: %s' % (arith, variant, B, len(errs), ', '.join('%s %.2e' % kv for kv in worst[:6])))
    for cat in ('out:', 'd gf', 'd fmaps', 'd '):
        es = [e for k, e in errs.items() if k.startswith(cat)]
        print('  %-8s max %.2e over %d tensors' % (cat, max(es), len(es)))
    bad = {k: '%.2e' % e for k, e in worst if not e < tol}
    assert not bad, 'decoder %s %s B=%d over the tolerance %.1e: %s' % (arith, variant, B, tol, bad)
