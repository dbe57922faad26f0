"""Autograd operators over the C-ABI CUDA kernels (raw pointers + current CUDA stream).

Every operator here launches hand-written sm_90a kernels from librih_b200.so; torch is used only for
memory (caching allocator), autograd bookkeeping and streams.  There is no CPU / eager fallback: tensors
must be fp32 CUDA tensors, otherwise a RuntimeError is raised.
"""
import ctypes

import torch
from torch.autograd import Function

from . import _lib

call = _lib.call


GROUP_FLOPS = {}      # entry point -> f(args) = algorithmic flops of one call (measurement metadata for bench.py's class roofline)
GEMM_MODES = {'simt': 0, 'tf32': 1, 'tf32x3': 2, 'tf32rn': 3, 'tf32c': 4}
_ATTN = {'nsplit': 0}


MODE = {'conv': 'simt', 'linear': 'simt'}


def set_gemm_mode(conv='simt', linear='simt'):
    """Arithmetic of the GEMM-class kernels: 'simt' = exact fp32 CUDA-core path, 'tf32' = wgmma tensor cores with TF32
    multiplicands and fp32 accumulation (what the reference's cuDNN convolutions use by default on this GPU),
    'tf32c' = truncating TF32 whose mean shrinkage (7.05e-4) is compensated in the epilogue (RN-equivalent error statistics),
    'tf32rn' = TF32 with the operands rounded to nearest in shared memory before the MMA (unbiased; the cuDNN convention),
    'tf32x3' = the same tensor-core kernels with an in-kernel hi/lo operand split and 3 MMAs per step (fp32-faithful)."""
    call('rih_set_gemm_mode', GEMM_MODES[conv], GEMM_MODES[linear])
    MODE['conv'], MODE['linear'] = conv, linear
    # the attention contractions follow the nn.Linear arithmetic (the reference runs both as fp32 torch.matmul / addmm):
    # 0 = fused SIMT kernel (exact fp32), 1 = wgmma TF32, 3 = wgmma 3xTF32
    _ATTN['nsplit'] = {'simt': 0, 'tf32x3': 3}.get(linear, 1)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return None if t is None else t.data_ptr()


def _check(t, name='tensor'):
    if not (t.is_cuda and t.dtype == torch.float32):
        raise RuntimeError('renderih_b200: %s must be a float32 CUDA tensor (got %s on %s); there is no CPU fallback'
                           % (name, t.dtype, t.device))
    return t


def _rows(t):
    """2-D row-major view contract: [rows, C], unit column stride, row stride = ld."""
    _check(t)
    if t.dim() != 2 or (t.shape[1] > 1 and t.stride(1) != 1):
        raise RuntimeError('renderih_b200: expected a [rows, C] tensor with unit column stride, got shape %s strides %s'
                           % (tuple(t.shape), t.stride()))
    return t


def _ld(t):
    return t.stride(0) if t.shape[0] > 1 else max(t.shape[1], t.stride(0))


# ----------------------------------------------------------------------------- direct parameter-gradient accumulation
# train.FlatParams registers every trainable tensor's gradient view here (keyed by the parameter's data pointer).  A backward
# that finds its weight registered accumulates straight into that buffer (kernels have accumulate flags / atomics) and
# returns None to autograd, which removes one torch add kernel (AccumulateGrad) per parameter per step.
GRAD_TARGETS = {}


def register_grad_target(param, grad):
    import weakref
    GRAD_TARGETS[param.data_ptr()] = (grad, weakref.ref(param))


def clear_grad_targets():
    GRAD_TARGETS.clear()


def _gt(t):
    """Registered flat-gradient view for the parameter whose storage starts where `t` does (t may be a 2-D view of it)."""
    if t is None:
        return None
    e = GRAD_TARGETS.get(t.data_ptr())
    if e is None:
        return None
    grad, ref = e
    p = ref()
    if p is None or p.data_ptr() != t.data_ptr() or p.grad is None or p.grad.data_ptr() != grad.data_ptr() or p.numel() != t.numel():
        GRAD_TARGETS.pop(t.data_ptr(), None)    # stale registration (owner gone or re-homed): fall back to autograd
        return None
    return grad


# ----------------------------------------------------------------------------- weight gradients on a side stream
# A weight-gradient GEMM (and the bias-gradient column sum) has no consumer until the optimizer: when it accumulates straight into the
# flat gradient buffer it is issued on a side stream that forks off the stream running backward, so the (latency-bound) chain
# dgrad -> previous layer's backward does not wait for it.  All side streams are joined into the caller's stream by an autograd-engine
# final callback when the backward pass ends (under CUDA-graph capture the fork / join become parallel graph branches).
# _WG['enabled'] = False keeps them on the backward stream.
_WG = {'streams': {}, 'armed': False, 'enabled': True}


def _wgrad_fork(*tensors):
    """-> side stream handle (int) to launch on, or None when disabled.  `tensors` are the operands the side-stream kernels read:
    they are registered with the caching allocator as in use on the side stream."""
    if not _WG['enabled']:
        return None
    cur = torch.cuda.current_stream()
    key = (cur.device.index, cur.cuda_stream)
    st = _WG['streams'].get(key)
    if st is None:
        st = torch.cuda.Stream(device=cur.device)
        _WG['streams'][key] = st
    st.wait_stream(cur)
    note_stream(st)
    _WG.setdefault('dirty', set()).add(key)
    for t in tensors:
        if t is not None:
            t.record_stream(st)
    if not _WG['armed']:
        _WG['armed'] = True
        torch.autograd.Variable._execution_engine.queue_callback(_wgrad_join)
    return st.cuda_stream


def _wgrad_join():
    """Join only the side streams that forked during THIS backward pass (a stream that belongs to no running capture must not be waited
    on from a capturing stream)."""
    _WG['armed'] = False
    dirty, _WG['dirty'] = _WG.get('dirty', set()), set()
    for key in dirty:
        torch.cuda.current_stream(key[0]).wait_stream(_WG['streams'][key])


# ----------------------------------------------------------------------------- backward-progress markers / streams of the current step
# The model marks tensors whose gradient completes a backward segment (e.g. a ResNet layer's output: its gradient is ready exactly when
# everything downstream has been back-propagated).  train.TrainStep installs a callback and starts the gradient all-reduce of the finished
# segment's parameters on a communication stream while the rest of backward runs.
MARKER_CALLBACK = [None]
STEP_STREAMS = {}          # cuda_stream handle -> torch stream: every side stream the current step has forked work onto


def note_stream(st):
    STEP_STREAMS[st.cuda_stream] = st


def backward_marker(t, name):
    if t.requires_grad and MARKER_CALLBACK[0] is not None:
        def hook(grad, name=name):
            cb = MARKER_CALLBACK[0]
            if cb is not None:
                cb(name)
            return None
        t.register_hook(hook)
    return t


# ----------------------------------------------------------------------------- dropout seed (device resident)
class _SeedState:
    """Device-resident base seed advanced once per step (so CUDA-graph replays draw fresh masks)."""
    def __init__(self):
        self.tensors = {}
        self.site = 0

    def ptr(self, device):
        key = device.index if device.index is not None else torch.cuda.current_device()
        if key not in self.tensors:
            self.tensors[key] = torch.tensor([0x243F6A8885A308D3 & 0x7FFFFFFFFFFFFFFF], dtype=torch.int64, device=device)
        return self.tensors[key].data_ptr()

    def manual_seed(self, seed, device):
        self.ptr(device)
        key = device.index if device.index is not None else torch.cuda.current_device()
        self.tensors[key].fill_(int(seed) & 0x7FFFFFFFFFFFFFFF)

    def advance(self, device):
        call('rih_seed_advance', self.ptr(device), _stream())

    def begin_forward(self):
        self.site = 0
        STEP_STREAMS.clear()
        _WG['armed'] = False      # a backward pass that raised may have left the join callback un-run
        _WG['dirty'] = set()

    def next_site(self):
        self.site += 1
        return self.site


seed_state = _SeedState()


# ----------------------------------------------------------------------------- Linear
class LinearFn(Function):
    """y = dropout(relu(x @ w^T + b)) + res  -- torch.nn.Linear call sites of models/model_attn/*.py, models/decoder.py"""

    @staticmethod
    def forward(ctx, x, w, b, relu, res, p_drop, site, stats=None, as_conv=False):
        x = _rows(x); _check(w, 'weight')
        M, K = x.shape
        N = w.shape[0]
        assert w.shape[1] == K and w.stride(1) == 1
        assert not (relu and res is not None)
        y = torch.empty((M, N), device=x.device, dtype=torch.float32)
        if res is not None:
            res = _rows(res)
        sp = seed_state.ptr(x.device) if p_drop > 0 else None
        call('rih_linear_fwd', _p(x), _ld(x), _p(w), w.stride(0), _p(b), _p(y), N, M, N, K, int(relu), 0,
             _p(res), _ld(res) if res is not None else 0, float(p_drop), sp, site, _p(stats), int(as_conv), _stream())
        ctx.save_for_backward(x, w, y if (relu or p_drop > 0) else None)
        ctx.meta = (relu, p_drop, site, b is not None, res is not None)
        ctx.as_conv = int(as_conv)
        ctx.bias_ref = b
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, y = ctx.saved_tensors
        relu, p_drop, site, has_b, has_res = ctx.meta
        dy = _rows(dy.contiguous() if dy.stride(-1) != 1 else dy)
        M, K = x.shape
        N = w.shape[0]
        s = _stream()
        g = dy
        if relu or p_drop > 0:
            g = torch.empty((M, N), device=dy.device, dtype=torch.float32)
            call('rih_epilogue_bwd', _p(dy), _ld(dy), _p(y), N, _p(g), N, M, N, int(relu), float(p_drop),
                 seed_state.ptr(dy.device) if p_drop > 0 else None, site, s)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty((M, K), device=dy.device, dtype=torch.float32)
            call('rih_linear_dgrad', _p(g), _ld(g), _p(w), w.stride(0), _p(dx), K, M, N, K, 0, ctx.as_conv, s)
        side = None
        # When g IS dy and dy is also handed back as the residual gradient, autograd may accumulate the other branch's gradient into it
        # in place on the main stream while a side stream still reads it (record_stream only guards the free): keep such launches in order.
        may_fork = not (has_res and g is dy)
        if ctx.needs_input_grad[1]:
            tgt = _gt(w)
            if tgt is not None:
                side = _wgrad_fork(g, x) if may_fork else None
                call('rih_linear_wgrad', _p(g), _ld(g), _p(x), _ld(x), _p(tgt), w.stride(0), M, N, K, 1, ctx.as_conv, side or s)
            else:
                dw = torch.empty((N, K), device=dy.device, dtype=torch.float32)
                call('rih_linear_wgrad', _p(g), _ld(g), _p(x), _ld(x), _p(dw), K, M, N, K, 0, ctx.as_conv, s)
        if has_b and ctx.needs_input_grad[2]:
            tgt = _gt(ctx.bias_ref)
            if tgt is not None:
                if side is None and may_fork:
                    side = _wgrad_fork(g)
                call('rih_colsum', _p(g), _ld(g), M, N, _p(tgt), 1, side or s)
            else:
                db = torch.empty((N,), device=dy.device, dtype=torch.float32)
                call('rih_colsum', _p(g), _ld(g), M, N, _p(db), 0, s)
        dres = dy if (has_res and ctx.needs_input_grad[4]) else None
        return dx, dw, db, None, dres, None, None, None, None


def linear(x, w, b=None, relu=False, res=None, p_drop=0.0, stats=None, as_conv=False):
    """stats: optional float64 [2*N] buffer receiving the output's column sums / sums of squares (fused BN statistics).
    as_conv: this GEMM is a convolution (im2col'ed stem): it follows the convolution arithmetic mode of set_gemm_mode."""
    site = seed_state.next_site() if p_drop > 0 else 0
    return LinearFn.apply(x, w, b, relu, res, p_drop, site, stats, as_conv)


# ----------------------------------------------------------------------------- LayerNorm
class LayerNormFn(Function):
    """y = LN(a (+ b)) (relu)  -- nn.LayerNorm(eps=1e-6) sites, e.g. models/model_attn/gcn.py:105,110"""

    @staticmethod
    def forward(ctx, a, b, gamma, beta, eps, relu, alias_input=False):
        a = _rows(a)
        if b is not None:
            b = _rows(b)
        M, F = a.shape
        y = torch.empty((M, F), device=a.device, dtype=torch.float32)
        mean = torch.empty((M,), device=a.device, dtype=torch.float32)
        rstd = torch.empty((M,), device=a.device, dtype=torch.float32)
        call('rih_layernorm_fwd', _p(a), _ld(a), _p(b), _ld(b) if b is not None else 0, _p(gamma), _p(beta), _p(y), F,
             _p(mean), _p(rstd), M, F, float(eps), int(relu), _stream())
        ctx.save_for_backward(a, b, gamma, beta, mean, rstd)
        ctx.relu = relu
        if alias_input:       # second output = the input itself: the residual branch of a pre-LN block hangs off it, so its gradient arrives
            assert b is None  # in backward as `d_alias` and the LN-backward kernel adds onto it (no autograd add pass)
            return y, a
        return y

    @staticmethod
    def backward(ctx, dy, d_alias=None):
        a, b, gamma, beta, mean, rstd = ctx.saved_tensors
        M, F = a.shape
        if dy is None:        # only the alias branch contributed (cannot happen in the models of this package; kept for completeness)
            return d_alias, None, None, None, None, None, None
        dy = _rows(dy.contiguous() if dy.stride(-1) != 1 else dy)
        acc = 0
        if d_alias is not None and d_alias.is_contiguous() and d_alias.shape == (M, F):
            dx, acc = d_alias, 1
        else:
            dx = torch.empty((M, F), device=dy.device, dtype=torch.float32)
        tg, tb = _gt(gamma), _gt(beta)
        direct = tg is not None and tb is not None
        dgamma = tg if direct else torch.zeros((F,), device=dy.device, dtype=torch.float32)
        dbeta = tb if direct else torch.zeros((F,), device=dy.device, dtype=torch.float32)
        call('rih_layernorm_bwd', _p(dy), _ld(dy), _p(a), _ld(a), _p(b), _ld(b) if b is not None else 0, _p(gamma), _p(beta),
             _p(mean), _p(rstd), _p(dx), F, acc, _p(dgamma), _p(dbeta), M, F, int(ctx.relu), _stream())
        if d_alias is not None and acc == 0:
            dx = dx + d_alias
        if direct:
            dgamma = dbeta = None
        return dx, (dx if b is not None else None), dgamma, dbeta, None, None, None


def layernorm(a, gamma, beta, b=None, eps=1e-6, relu=False, alias_input=False):
    """alias_input: also return `a` as a second output; route the block's residual use of `a` through it and the gradient of that branch
    is accumulated by the LayerNorm-backward kernel instead of a separate autograd add (pre-LN residual blocks, self_attn.py:24-33,66-85)."""
    return LayerNormFn.apply(a, b, gamma, beta, eps, relu, alias_input)


# ----------------------------------------------------------------------------- Chebyshev basis (K=2)
class ChebFn(Function):
    """[x, Lx] interleaved along features -- graph_conv_cheby, models/model_attn/gcn.py:34-69"""

    @staticmethod
    def forward(ctx, x, graph, B, V, alias_input=False):
        x = _rows(x)
        F = x.shape[1]
        assert x.shape[0] == B * V
        out = torch.empty((B * V, 2 * F), device=x.device, dtype=torch.float32)
        call('rih_cheb_fwd', _p(x), _ld(x), _p(graph.rowptr), _p(graph.col), _p(graph.val), _p(out), B, V, F, _stream())
        ctx.graph, ctx.dims = graph, (B, V, F)
        if alias_input:
            return out, x
        return out

    @staticmethod
    def backward(ctx, d, d_alias=None):
        B, V, F = ctx.dims
        g = ctx.graph
        d = d.contiguous()
        acc = 0
        if d_alias is not None and d_alias.is_contiguous() and d_alias.shape == (B * V, F):
            dx, acc = d_alias, 1         # the shortcut branch's gradient: the SpMM-transpose kernel adds onto it
        else:
            dx = torch.empty((B * V, F), device=d.device, dtype=torch.float32)
        call('rih_cheb_bwd', _p(d), _p(g.rowptr_t), _p(g.col_t), _p(g.val_t), _p(dx), F, acc, B, V, F, _stream())
        if d_alias is not None and acc == 0:
            dx = dx + d_alias
        return dx, None, None, None, None


def cheb(x, graph, B, V, alias_input=False):
    """alias_input: also return x as a second output for the block's shortcut branch (gcn.py:99-110): its gradient is accumulated by the
    backward SpMM kernel instead of an autograd add."""
    return ChebFn.apply(x, graph, B, V, alias_input)


# ----------------------------------------------------------------------------- position embedding (+ nearest vertex upsample)
class PosEmbFn(Function):
    """y[b,u] = x[b,u//p] + emb[u]  -- DualGraph.py:76-80 (+ graph_upsample :135-137), img_attn.py:57-63"""

    @staticmethod
    def forward(ctx, x, emb, B, U, p):
        x = _rows(x)
        F = x.shape[1]
        assert x.shape[0] == B * (U // p) and emb.shape == (U, F) and emb.is_contiguous()
        y = torch.empty((B * U, F), device=x.device, dtype=torch.float32)
        call('rih_posemb_fwd', _p(x), _ld(x), _p(emb), _p(y), F, B, U, F, p, _stream())
        ctx.dims = (B, U, F, p)
        ctx.emb_ref = emb
        return y

    @staticmethod
    def backward(ctx, dy):
        B, U, F, p = ctx.dims
        dy = _rows(dy.contiguous() if dy.stride(-1) != 1 else dy)
        dx = demb = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty((B * (U // p), F), device=dy.device, dtype=torch.float32)
        tgt = _gt(ctx.emb_ref)
        if ctx.needs_input_grad[1]:
            demb = tgt if tgt is not None else torch.zeros((U, F), device=dy.device, dtype=torch.float32)
        call('rih_posemb_bwd', _p(dy), _ld(dy), _p(dx), F, _p(demb), B, U, F, p, _stream())
        return dx, (None if tgt is not None else demb), None, None, None


def posemb(x, emb, B, U, p=1):
    return PosEmbFn.apply(x, emb, B, U, p)


# ----------------------------------------------------------------------------- attention core
class AttnFn(Function):
    """softmax(Q K^T / sqrt(d)) V with probability dropout -- self_attn.py:63-76, inter_attn.py:90-105"""

    @staticmethod
    def forward(ctx, q, k, v, B, H, Sq, Sk, p_drop, site):
        q, k, v = _rows(q), _rows(k), _rows(v)
        HD = q.shape[1]
        d = HD // H
        assert q.shape[0] == B * Sq and k.shape[0] == B * Sk and v.shape[0] == B * Sk
        o = torch.empty((B * Sq, HD), device=q.device, dtype=torch.float32)
        lse = torch.empty((B * H * Sq,), device=q.device, dtype=torch.float32)
        scale = 1.0 / (d ** 0.5)
        sp = seed_state.ptr(q.device) if p_drop > 0 else None
        call('rih_attn_fwd', _p(q), Sq * _ld(q), _ld(q), _p(k), Sk * _ld(k), _ld(k), _p(v), Sk * _ld(v), _ld(v),
             _p(o), Sq * HD, HD, _p(lse), B, H, Sq, Sk, d, scale, float(p_drop), sp, site, _stream())
        ctx.save_for_backward(q, k, v, o, lse)
        ctx.meta = (B, H, Sq, Sk, d, scale, p_drop, site)
        return o

    @staticmethod
    def backward(ctx, do):
        q, k, v, o, lse = ctx.saved_tensors
        B, H, Sq, Sk, d, scale, p_drop, site = ctx.meta
        do = _rows(do.contiguous() if do.stride(-1) != 1 else do)
        HD = H * d
        dq = torch.empty((B * Sq, HD), device=do.device, dtype=torch.float32)
        dk = torch.empty((B * Sk, HD), device=do.device, dtype=torch.float32)
        dv = torch.empty((B * Sk, HD), device=do.device, dtype=torch.float32)
        sp = seed_state.ptr(do.device) if p_drop > 0 else None
        call('rih_attn_bwd', _p(q), Sq * _ld(q), _ld(q), _p(k), Sk * _ld(k), _ld(k), _p(v), Sk * _ld(v), _ld(v),
             _p(o), Sq * HD, HD, _p(do), Sq * _ld(do), _ld(do), _p(lse),
             _p(dq), Sq * HD, HD, _p(dk), Sk * HD, HD, _p(dv), Sk * HD, HD,
             B, H, Sq, Sk, d, scale, float(p_drop), sp, site, _stream())
        return dq, dk, dv, None, None, None, None, None, None


class AttnTcFn(Function):
    """The same attention core on the tensor cores as fused flash-style kernels (rih_attn_tc_fwd / rih_attn_tc_bwd): no score matrix
    reaches global memory; the forward keeps O and two statistics per query row (row max, 1 / row sum) for the backward pass."""

    @staticmethod
    def forward(ctx, q, k, v, B, H, Sq, Sk, p_drop, site, nsplit):
        q, k, v = _rows(q), _rows(k), _rows(v)
        HD = q.shape[1]
        d = HD // H
        assert q.shape[0] == B * Sq and k.shape[0] == B * Sk and v.shape[0] == B * Sk
        o = torch.empty((B * Sq, HD), device=q.device, dtype=torch.float32)
        stats = torch.empty((B * H * Sq, 2), device=q.device, dtype=torch.float32)
        scale = 1.0 / (d ** 0.5)
        sp = seed_state.ptr(q.device) if p_drop > 0 else None
        call('rih_attn_tc_fwd', _p(q), _ld(q), _p(k), _ld(k), _p(v), _ld(v), _p(o), HD, _p(stats), None, 0,
             B, H, Sq, Sk, d, scale, float(p_drop), sp, site, nsplit, _stream())
        ctx.save_for_backward(q, k, v, o, stats)
        ctx.meta = (B, H, Sq, Sk, d, scale, p_drop, site, nsplit)
        return o

    @staticmethod
    def backward(ctx, do):
        q, k, v, o, stats = ctx.saved_tensors
        B, H, Sq, Sk, d, scale, p_drop, site, nsplit = ctx.meta
        do = _rows(do.contiguous() if do.stride(-1) != 1 else do)
        HD = H * d
        dq = torch.empty((B * Sq, HD), device=do.device, dtype=torch.float32)
        dk = torch.empty((B * Sk, HD), device=do.device, dtype=torch.float32)
        dv = torch.empty((B * Sk, HD), device=do.device, dtype=torch.float32)
        sp = seed_state.ptr(do.device) if p_drop > 0 else None
        call('rih_attn_tc_bwd', _p(q), _ld(q), _p(k), _ld(k), _p(v), _ld(v), _p(do), _ld(do), _p(stats), _p(o), None, HD,
             _p(dq), HD, _p(dk), HD, _p(dv), HD, B, H, Sq, Sk, d, scale, float(p_drop), sp, site, nsplit, _stream())
        return dq, dk, dv, None, None, None, None, None, None, None


def attention(q, k, v, B, H, Sq, Sk, p_drop=0.0, impl=None):
    """impl: None = follow set_gemm_mode (SIMT fused kernel in 'simt' mode, tensor-core fused kernels otherwise), 'simt' | 'tc' to force."""
    site = seed_state.next_site() if p_drop > 0 else 0
    nsplit = _ATTN['nsplit']
    if impl == 'simt':
        nsplit = 0
    elif impl == 'tc' and nsplit == 0:
        nsplit = 3
    d = q.shape[1] // H
    aligned = all(t.data_ptr() % 16 == 0 and _ld(t) % 4 == 0 for t in (q, k, v)) and d % 4 == 0
    if nsplit and aligned and B * H > 0 and Sq > 0 and Sk <= 512:
        return AttnTcFn.apply(q, k, v, B, H, Sq, Sk, p_drop, site, nsplit)
    return AttnFn.apply(q, k, v, B, H, Sq, Sk, p_drop, site)


# ----------------------------------------------------------------------------- fused projections + attention core
def adjacent(ts):
    """True when the tensors lie back to back in memory (each one dense): then [t0; t1; ...] is ONE row-major matrix / vector."""
    if any(t is None for t in ts):
        return False
    for a, b in zip(ts[:-1], ts[1:]):
        if not a.is_contiguous() or a.data_ptr() + a.numel() * a.element_size() != b.data_ptr():
            return False
    return ts[-1].is_contiguous()


def fuse_storage(params):
    """Make the given parameters adjacent in memory (one backing buffer, each `.data` a view of it) unless they already are, so that GEMMs can
    treat them as one stacked matrix.  Parameters that train.FlatParams has re-homed keep their place (FlatParams lays tagged groups out
    adjacently itself); returns True when the group is adjacent afterwards."""
    if adjacent([p.data for p in params]):
        return True
    if any(p.data_ptr() in GRAD_TARGETS for p in params) or torch.cuda.is_current_stream_capturing():
        return False
    with torch.no_grad():
        buf = torch.empty(sum(p.numel() for p in params), device=params[0].device, dtype=params[0].dtype)
        off = 0
        for p in params:
            v = buf[off:off + p.numel()].view(p.shape)
            v.copy_(p.data)
            p.data = v
            off += p.numel()
    return True


class AttnProjFn(Function):
    """Q / K / V projections + the attention core as ONE autograd node:
         q = xq Wq^T + bq ; [k | v] = xkv [Wk; Wv]^T + [bk; bv] ; o = softmax(q k^T / sqrt(d)) v  (probability dropout)
       -- self_attn.py:66-76, inter_attn.py:82-105.  With xq is xkv (plain self-attention) the three projections are ONE GEMM with N = 3 HD
       (the weights are adjacent in memory: fuse_storage / FlatParams groups); otherwise one GEMM for q and one for [k | v].  q, k, v live as
       column slices of one [rows, 3 HD] / [rows, 2 HD] buffer (the kernels take row strides), and in backward the attention kernels write
       dq / dk / dv into the slices of one gradient buffer, so the input gradient is ONE dgrad GEMM (K = 3 HD) and the weight gradient ONE
       wgrad GEMM -- instead of 3 + 3 + 3 launches and two autograd adds."""

    @staticmethod
    def forward(ctx, xq, xkv, wq, wk, wv, bq, bk, bv, B, H, Sq, Sk, p_drop, site, nsplit):
        same = xkv is None
        xq = _rows(xq)
        xkv = xq if same else _rows(xkv)
        HD, K = wq.shape
        d = HD // H
        assert xq.shape == (B * Sq, K) and xkv.shape == (B * Sk, K)
        Mq, Mk = xq.shape[0], xkv.shape[0]
        dev = xq.device
        s = _stream()
        w_adj = adjacent([wq, wk, wv]) and adjacent([bq, bk, bv])
        if same:
            qkv = torch.empty((Mq, 3 * HD), device=dev, dtype=torch.float32)
            if w_adj:
                call('rih_linear_fwd', _p(xq), _ld(xq), _p(wq), K, _p(bq), _p(qkv), 3 * HD, Mq, 3 * HD, K, 0, 0, None, 0, 0.0, None, 0, None, 0, s)
            else:
                for i, (w, b) in enumerate(((wq, bq), (wk, bk), (wv, bv))):
                    call('rih_linear_fwd', _p(xq), _ld(xq), _p(w), K, _p(b), qkv.data_ptr() + 4 * i * HD, 3 * HD, Mq, HD, K, 0, 0, None, 0, 0.0, None, 0, None, 0, s)
            q, k, v = qkv[:, :HD], qkv[:, HD:2 * HD], qkv[:, 2 * HD:]
            kvbuf = None
        else:
            qkv = torch.empty((Mq, HD), device=dev, dtype=torch.float32)
            kvbuf = torch.empty((Mk, 2 * HD), device=dev, dtype=torch.float32)
            call('rih_linear_fwd', _p(xq), _ld(xq), _p(wq), K, _p(bq), _p(qkv), HD, Mq, HD, K, 0, 0, None, 0, 0.0, None, 0, None, 0, s)
            if adjacent([wk, wv]) and adjacent([bk, bv]):
                call('rih_linear_fwd', _p(xkv), _ld(xkv), _p(wk), K, _p(bk), _p(kvbuf), 2 * HD, Mk, 2 * HD, K, 0, 0, None, 0, 0.0, None, 0, None, 0, s)
            else:
                for i, (w, b) in enumerate(((wk, bk), (wv, bv))):
                    call('rih_linear_fwd', _p(xkv), _ld(xkv), _p(w), K, _p(b), kvbuf.data_ptr() + 4 * i * HD, 2 * HD, Mk, HD, K, 0, 0, None, 0, 0.0, None, 0, None, 0, s)
            q, k, v = qkv, kvbuf[:, :HD], kvbuf[:, HD:]
        o = torch.empty((Mq, HD), device=dev, dtype=torch.float32)
        scale = 1.0 / (d ** 0.5)
        sp = seed_state.ptr(dev) if p_drop > 0 else None
        stats = lse = None
        if nsplit:
            stats = torch.empty((B * H * Sq, 2), device=dev, dtype=torch.float32)
            call('rih_attn_tc_fwd', _p(q), _ld(q), _p(k), _ld(k), _p(v), _ld(v), _p(o), HD, _p(stats), None, 0,
                 B, H, Sq, Sk, d, scale, float(p_drop), sp, site, nsplit, s)
        else:
            lse = torch.empty((B * H * Sq,), device=dev, dtype=torch.float32)
            call('rih_attn_fwd', _p(q), Sq * _ld(q), _ld(q), _p(k), Sk * _ld(k), _ld(k), _p(v), Sk * _ld(v), _ld(v),
                 _p(o), Sq * HD, HD, _p(lse), B, H, Sq, Sk, d, scale, float(p_drop), sp, site, s)
        ctx.save_for_backward(xq, None if same else xkv, wq, wk, wv, qkv, kvbuf, o, stats, lse)
        ctx.meta = (same, B, H, Sq, Sk, d, scale, p_drop, site, nsplit)
        ctx.refs = (bq, bk, bv)
        return o

    @staticmethod
    def backward(ctx, do):
        xq, xkv, wq, wk, wv, qkv, kvbuf, o, stats, lse = ctx.saved_tensors
        same, B, H, Sq, Sk, d, scale, p_drop, site, nsplit = ctx.meta
        bq, bk, bv = ctx.refs
        if same:
            xkv = xq
        do = _rows(do.contiguous() if do.stride(-1) != 1 else do)
        HD, K = wq.shape
        Mq, Mk = xq.shape[0], xkv.shape[0]
        dev = do.device
        s = _stream()
        if same:
            q, k, v = qkv[:, :HD], qkv[:, HD:2 * HD], qkv[:, 2 * HD:]
            dqkv = torch.empty((Mq, 3 * HD), device=dev, dtype=torch.float32)
            dq, dk, dv = dqkv[:, :HD], dqkv[:, HD:2 * HD], dqkv[:, 2 * HD:]
            dkv = None
        else:
            q, k, v = qkv, kvbuf[:, :HD], kvbuf[:, HD:]
            dqkv = torch.empty((Mq, HD), device=dev, dtype=torch.float32)
            dkv = torch.empty((Mk, 2 * HD), device=dev, dtype=torch.float32)
            dq, dk, dv = dqkv, dkv[:, :HD], dkv[:, HD:]
        sp = seed_state.ptr(dev) if p_drop > 0 else None
        if nsplit:
            call('rih_attn_tc_bwd', _p(q), _ld(q), _p(k), _ld(k), _p(v), _ld(v), _p(do), _ld(do), _p(stats), _p(o), None, HD,
                 _p(dq), _ld(dq), _p(dk), _ld(dk), _p(dv), _ld(dv), B, H, Sq, Sk, d, scale, float(p_drop), sp, site, nsplit, s)
        else:
            call('rih_attn_bwd', _p(q), Sq * _ld(q), _ld(q), _p(k), Sk * _ld(k), _ld(k), _p(v), Sk * _ld(v), _ld(v),
                 _p(o), Sq * HD, HD, _p(do), Sq * _ld(do), _ld(do), _p(lse),
                 _p(dq), Sq * _ld(dq), _ld(dq), _p(dk), Sk * _ld(dk), _ld(dk), _p(dv), Sk * _ld(dv), _ld(dv),
                 B, H, Sq, Sk, d, scale, float(p_drop), sp, site, s)
        ni = ctx.needs_input_grad
        dxq = dxkv = None
        w3 = adjacent([wq, wk, wv])
        w2 = adjacent([wk, wv])
        # ---- input gradients
        if same and ni[0]:
            dxq = torch.empty((Mq, K), device=dev, dtype=torch.float32)
            if w3:
                call('rih_linear_dgrad', _p(dqkv), 3 * HD, _p(wq), K, _p(dxq), K, Mq, 3 * HD, K, 0, 0, s)
            else:
                for i, w in enumerate((wq, wk, wv)):
                    call('rih_linear_dgrad', dqkv.data_ptr() + 4 * i * HD, 3 * HD, _p(w), K, _p(dxq), K, Mq, HD, K, int(i > 0), 0, s)
        elif not same:
            if ni[0]:
                dxq = torch.empty((Mq, K), device=dev, dtype=torch.float32)
                call('rih_linear_dgrad', _p(dqkv), HD, _p(wq), K, _p(dxq), K, Mq, HD, K, 0, 0, s)
            if ni[1]:
                dxkv = torch.empty((Mk, K), device=dev, dtype=torch.float32)
                if w2:
                    call('rih_linear_dgrad', _p(dkv), 2 * HD, _p(wk), K, _p(dxkv), K, Mk, 2 * HD, K, 0, 0, s)
                else:
                    for i, w in enumerate((wk, wv)):
                        call('rih_linear_dgrad', dkv.data_ptr() + 4 * i * HD, 2 * HD, _p(w), K, _p(dxkv), K, Mk, HD, K, int(i > 0), 0, s)
        # ---- parameter gradients: straight into the flat gradient buffer when registered (side stream), else returned to autograd
        tw = [_gt(w) for w in (wq, wk, wv)]
        tb = [_gt(b) for b in (bq, bk, bv)]
        direct = all(t is not None for t in tw + tb)
        if direct:
            side = _wgrad_fork(dqkv, dkv, xq, xkv) or s
            gw, gb = tw, tb
            acc = 1
        else:
            side = s
            gw = [torch.empty((HD, K), device=dev, dtype=torch.float32) for _ in range(3)] if not (same and w3) else None
            gb = [torch.empty((HD,), device=dev, dtype=torch.float32) for _ in range(3)]
            acc = 0
        if same and w3 and (not direct or (adjacent(tw) and adjacent(tb))):
            if direct:
                call('rih_linear_wgrad', _p(dqkv), 3 * HD, _p(xq), _ld(xq), _p(gw[0]), K, Mq, 3 * HD, K, 1, 0, side)
                call('rih_colsum', _p(dqkv), 3 * HD, Mq, 3 * HD, _p(gb[0]), 1, side)
            else:
                big = torch.empty((3 * HD, K), device=dev, dtype=torch.float32)
                bigb = torch.empty((3 * HD,), device=dev, dtype=torch.float32)
                call('rih_linear_wgrad', _p(dqkv), 3 * HD, _p(xq), _ld(xq), _p(big), K, Mq, 3 * HD, K, 0, 0, side)
                call('rih_colsum', _p(dqkv), 3 * HD, Mq, 3 * HD, _p(bigb), 0, side)
                gw = [big[i * HD:(i + 1) * HD] for i in range(3)]
                gb = [bigb[i * HD:(i + 1) * HD] for i in range(3)]
        else:
            if gw is None:
                gw = [torch.empty((HD, K), device=dev, dtype=torch.float32) for _ in range(3)]
            srcs = ((dqkv, 0, 3 * HD, xq, Mq), (dqkv, HD, 3 * HD, xq, Mq), (dqkv, 2 * HD, 3 * HD, xq, Mq)) if same else \
                   ((dqkv, 0, HD, xq, Mq), (dkv, 0, 2 * HD, xkv, Mk), (dkv, HD, 2 * HD, xkv, Mk))
            for i, (g, off, ld, x, M) in enumerate(srcs):
                call('rih_linear_wgrad', g.data_ptr() + 4 * off, ld, _p(x), _ld(x), _p(gw[i]), K, M, HD, K, acc, 0, side)
                call('rih_colsum', g.data_ptr() + 4 * off, ld, M, HD, _p(gb[i]), acc, side)
        if direct:
            gw = gb = [None, None, None]
        return (dxq, dxkv, gw[0], gw[1], gw[2], gb[0], gb[1], gb[2]) + (None,) * 7


FUSED = {'qkv': True,        # False = separate projection GEMMs + attention node
         'alias': True}      # False = residual-branch gradients summed by autograd adds


def attention_proj(xq, xkv, lin_q, lin_k, lin_v, B, H, Sq, Sk, p_drop=0.0):
    """o = Attention(xq Wq, xkv Wk, xkv Wv) -- see AttnProjFn.  lin_*: the nn.Linear parameter holders (self_attn.py:54-56); pass xkv=None
    for plain self-attention (queries, keys and values all from xq)."""
    if not FUSED['qkv']:
        xk = xq if xkv is None else xkv
        q = linear(xq, lin_q.weight, lin_q.bias)
        k = linear(xk, lin_k.weight, lin_k.bias)
        v = linear(xk, lin_v.weight, lin_v.bias)
        return attention(q, k, v, B, H, Sq, Sk, p_drop=p_drop)
    site = seed_state.next_site() if p_drop > 0 else 0
    nsplit = _ATTN['nsplit']
    HD = lin_q.weight.shape[0]
    d = HD // H
    if not (nsplit and d % 4 == 0 and B * H > 0 and Sq > 0 and Sk <= 512):
        nsplit = 0
    if xkv is None:
        fuse_storage([lin_q.weight, lin_k.weight, lin_v.weight])
        fuse_storage([lin_q.bias, lin_k.bias, lin_v.bias])
    else:
        fuse_storage([lin_k.weight, lin_v.weight])
        fuse_storage([lin_k.bias, lin_v.bias])
    return AttnProjFn.apply(xq, xkv, lin_q.weight, lin_k.weight, lin_v.weight, lin_q.bias, lin_k.bias, lin_v.bias, B, H, Sq, Sk, p_drop, site, nsplit)


# ----------------------------------------------------------------------------- dropout (stand-alone)
class DropoutFn(Function):
    @staticmethod
    def forward(ctx, x, p, site):
        x = _rows(x)
        M, C = x.shape
        y = torch.empty((M, C), device=x.device, dtype=torch.float32)
        call('rih_dropout', _p(x), _ld(x), _p(y), C, M, C, float(p), seed_state.ptr(x.device), site, _stream())
        ctx.meta = (p, site)
        return y

    @staticmethod
    def backward(ctx, dy):
        p, site = ctx.meta
        dy = _rows(dy.contiguous() if dy.stride(-1) != 1 else dy)
        M, C = dy.shape
        dx = torch.empty((M, C), device=dy.device, dtype=torch.float32)
        call('rih_dropout', _p(dy), _ld(dy), _p(dx), C, M, C, float(p), seed_state.ptr(dy.device), site, _stream())
        return dx, None, None


def dropout(x, p):
    if p <= 0:
        return x
    return DropoutFn.apply(x, p, seed_state.next_site())


# ----------------------------------------------------------------------------- decoder entry / tail
class GfBroadcastFn(Function):
    """Lf[b,v,:] = cat(g[b,:], pe[v,:]) + emb[v,:]  -- models/decoder.py:132-135 + DualGraph.py:76-80"""

    @staticmethod
    def forward(ctx, g, pe, emb, B, V):
        g = _check(g).contiguous()
        G = g.shape[1]
        y = torch.empty((B * V, G + 3), device=g.device, dtype=torch.float32)
        call('rih_gf_broadcast_fwd', _p(g), _p(pe), _p(emb), _p(y), B, V, G, _stream())
        ctx.dims = (B, V, G)
        return y

    @staticmethod
    def backward(ctx, dy):
        B, V, G = ctx.dims
        dy = dy.contiguous()
        dg = torch.empty((B, G), device=dy.device, dtype=torch.float32)
        demb = torch.zeros((V, G + 3), device=dy.device, dtype=torch.float32) if ctx.needs_input_grad[2] else None
        call('rih_gf_broadcast_bwd', _p(dy), _p(dg), _p(demb), B, V, G, _stream())
        return dg, None, demb, None, None


def gf_broadcast(g, pe, emb, B, V):
    return GfBroadcastFn.apply(g, pe, emb, B, V)


def _ptr_array(tensors):
    arr = (ctypes.c_void_p * len(tensors))()
    for i, t in enumerate(tensors):
        arr[i] = None if t is None else t.data_ptr()
    return arr


class TailFn(Function):
    """avg_head/params_head/coord_head/unsample_layer/projection_batch -- models/decoder.py:139-159"""

    @staticmethod
    def forward(ctx, Lf, avg_w, avg_b, par_w, par_b, coord_w, coord_b, U, B, V, img):
        Lf = _rows(Lf)
        F = Lf.shape[1]
        Nv = U.shape[0]
        dev = Lf.device
        prm = torch.empty((B, 3), device=dev); temp = torch.empty((B, F), device=dev)
        v3c = torch.empty((B, V, 3), device=dev); v2c = torch.empty((B, V, 2), device=dev)
        v3 = torch.empty((B, Nv, 3), device=dev); v2 = torch.empty((B, Nv, 2), device=dev)
        params = [avg_w, avg_b, par_w, par_b, coord_w, coord_b, U]
        for t in params:
            assert t.is_contiguous()
        call('rih_tail_fwd', _ptr_array(params), _p(Lf), _ld(Lf), B, V, F, Nv, float(img), _p(prm), _p(temp), _p(v3c), _p(v2c),
             _p(v3), _p(v2), _stream())
        ctx.save_for_backward(Lf, avg_w, avg_b, par_w, par_b, coord_w, coord_b, U, prm, temp, v3c, v3)
        ctx.dims = (B, V, F, Nv, img)
        scale = prm[:, 0]
        trans = prm[:, 1:]
        return scale, trans, v3c, v2c, v3, v2

    @staticmethod
    def backward(ctx, d_scale, d_trans, d_v3c, d_v2c, d_v3, d_v2):
        Lf, avg_w, avg_b, par_w, par_b, coord_w, coord_b, U, prm, temp, v3c, v3 = ctx.saved_tensors
        B, V, F, Nv, img = ctx.dims
        dev = Lf.device

        def c(t):
            return None if t is None else t.contiguous()
        d_scale, d_trans, d_v3c, d_v2c, d_v3, d_v2 = map(c, (d_scale, d_trans, d_v3c, d_v2c, d_v3, d_v2))
        params = [avg_w, avg_b, par_w, par_b, coord_w, coord_b, U]
        grads = []
        for i, t in enumerate(params):
            grads.append(torch.zeros_like(t) if ctx.needs_input_grad[1 + i] else None)
        dLf = torch.empty((B * V, F), device=dev, dtype=torch.float32)
        call('rih_tail_bwd', _ptr_array(params), _ptr_array(grads), _p(Lf), _ld(Lf), B, V, F, Nv, float(img), _p(prm), _p(temp),
             _p(v3c), _p(v3), _p(d_scale), _p(d_trans), _p(d_v3c), _p(d_v2c), _p(d_v3), _p(d_v2), _p(dLf), F, _stream())
        return (dLf,) + tuple(grads) + (None, None, None)


def decoder_tail(Lf, avg_w, avg_b, par_w, par_b, coord_w, coord_b, U, B, V, img):
    return TailFn.apply(Lf, avg_w, avg_b, par_w, par_b, coord_w, coord_b, U, B, V, img)


class GatherRowsFn(Function):
    """y[b,i,:] = x[b, idx[i]//div, :] -- graph_upsample(p) + GCN_to_vert, models/decoder.py:165-172"""

    @staticmethod
    def forward(ctx, x, idx, div):
        x = _check(x).contiguous()
        B, Vin, C = x.shape
        Vout = idx.numel()
        y = torch.empty((B, Vout, C), device=x.device, dtype=torch.float32)
        call('rih_gather_rows', _p(x), _p(idx), _p(y), B, Vin, Vout, C, div, _stream())
        ctx.idx, ctx.dims = idx, (B, Vin, Vout, C, div)
        return y

    @staticmethod
    def backward(ctx, dy):
        B, Vin, Vout, C, div = ctx.dims
        dy = dy.contiguous()
        dx = torch.zeros((B, Vin, C), device=dy.device, dtype=torch.float32)
        call('rih_scatter_rows_add', _p(dy), _p(ctx.idx), _p(dx), B, Vin, Vout, C, div, _stream())
        return dx, None, None


def gather_rows(x, idx, div=1):
    return GatherRowsFn.apply(x, idx, div)


# ----------------------------------------------------------------------------- image side (NHWC rows)
def _geom(N, H, W, Cin, Cout, R, S, stride, pad, ldx, ldy):
    Ho = (H + 2 * pad - R) // stride + 1
    Wo = (W + 2 * pad - S) // stride + 1
    return (ctypes.c_int * 13)(N, H, W, Cin, Ho, Wo, Cout, R, S, stride, pad, ldx, ldy), Ho, Wo


def _conv_ws(g, which, device):
    """Workspace the tensor-core path needs for this geometry (stride-2 parity stack / zero-inserted dY); None if none."""
    n = ctypes.c_longlong(0)
    call('rih_conv2d_workspace', g, which, ctypes.byref(n))
    return torch.empty(n.value, device=device, dtype=torch.float32) if n.value > 0 else None


def _w_phys(w):
    """Conv2d weight [Cout,Cin,R,S] must be channels_last so that memory is [Cout,R,S,Cin]."""
    if w.dim() != 4 or not w.permute(0, 2, 3, 1).is_contiguous():
        raise RuntimeError('renderih_b200: conv weight must be a channels_last [Cout,Cin,R,S] tensor')
    return w


class Conv2dFn(Function):
    """NHWC conv (+bias)(+relu) -- nn.Conv2d sites of models/encoder.py, torchvision resnet, img_attn.py:48"""

    @staticmethod
    def forward(ctx, x, w, b, N, H, W, stride, pad, relu, relu_masked_by_consumer, stats, alias_input=False):
        x = _rows(x); _w_phys(_check(w, 'weight'))
        ctx.alias_input = alias_input
        Cout, Cin, R, S = w.shape
        assert x.shape == (N * H * W, Cin), (x.shape, N, H, W, Cin)
        g, Ho, Wo = _geom(N, H, W, Cin, Cout, R, S, stride, pad, _ld(x), Cout)
        y = torch.empty((N * Ho * Wo, Cout), device=x.device, dtype=torch.float32)
        call('rih_conv2d_fwd', _p(x), _p(w), _p(b), _p(y), g, int(relu), _p(_conv_ws(g, 0, x.device)), _p(stats), _stream())
        need_y = relu and not relu_masked_by_consumer
        ctx.save_for_backward(x, w, y if need_y else None)
        ctx.meta = (N, H, W, stride, pad, need_y, b is not None)
        ctx.bias_ref = b
        if alias_input:      # second output = the input itself: a later consumer of x (the residual add, the downsample conv) hangs off it,
            return y, x      # so its gradient arrives HERE and the dgrad kernel accumulates onto it instead of autograd adding two tensors
        return y

    @staticmethod
    def backward(ctx, dy, d_alias=None):
        x, w, y = ctx.saved_tensors
        N, H, W, stride, pad, need_y, has_b = ctx.meta
        Cout, Cin, R, S = w.shape
        dy = _rows(dy.contiguous() if dy.stride(-1) != 1 else dy)
        s = _stream()
        if need_y:
            g_ = torch.empty_like(y)
            call('rih_relu_bwd', _p(dy), _ld(dy), _p(y), Cout, _p(g_), Cout, y.shape[0], Cout, s)
            dy = g_
        g, Ho, Wo = _geom(N, H, W, Cin, Cout, R, S, stride, pad, Cin, _ld(dy))
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            acc = 0
            if d_alias is not None and d_alias.is_contiguous() and d_alias.shape == (N * H * W, Cin):
                dx, acc = d_alias, 1      # accumulate onto the gradient that came in through the alias output (epilogue: TMA reduce-add)
            else:
                dx = torch.empty((N * H * W, Cin), device=dy.device, dtype=torch.float32)
            call('rih_conv2d_dgrad', _p(dy), _p(w), _p(dx), g, acc, _p(_conv_ws(g, 1, dy.device)), s)
            if d_alias is not None and acc == 0:
                dx = dx + d_alias
        elif d_alias is not None:
            dx = d_alias
        if ctx.needs_input_grad[1]:
            g2, _, _ = _geom(N, H, W, Cin, Cout, R, S, stride, pad, _ld(x), _ld(dy))
            tgt = _gt(w)
            if tgt is not None:
                wsb = _conv_ws(g2, 2, dy.device)
                side = _wgrad_fork(dy, x, wsb)
                call('rih_conv2d_wgrad', _p(dy), _p(x), _p(tgt), g2, 1, _p(wsb), side or s)
            else:
                dw = torch.empty_like(w)
                call('rih_conv2d_wgrad', _p(dy), _p(x), _p(dw), g2, 0, _p(_conv_ws(g2, 2, dy.device)), s)
        if has_b and ctx.needs_input_grad[2]:
            tgt = _gt(ctx.bias_ref)
            if tgt is not None:
                call('rih_colsum', _p(dy), _ld(dy), dy.shape[0], Cout, _p(tgt), 1, s)
            else:
                db = torch.empty((Cout,), device=dy.device, dtype=torch.float32)
                call('rih_colsum', _p(dy), _ld(dy), dy.shape[0], Cout, _p(db), 0, s)
        return dx, dw, db, None, None, None, None, None, None, None, None, None


def conv2d(x, w, b, N, H, W, stride=1, pad=0, relu=False, relu_masked_by_consumer=False, stats=None, alias_input=False):
    """stats: optional float64 [2*Cout] buffer that receives the output's per-channel sum / sum of squares (fused BN statistics).
    alias_input: also return x as a second output; route every OTHER use of x through it and their gradients are accumulated by this
    convolution's dgrad kernel (no separate add pass over the activation gradient)."""
    return Conv2dFn.apply(x, w, b, N, H, W, stride, pad, relu, relu_masked_by_consumer, stats, alias_input)


# ----------------------------------------------------------------------------- eval-mode BatchNorm folded into the convolution

class BnFold:
    """Per-channel (scale, shift) vectors of every eval-mode BatchNorm2d under `root`, recomputed by ONE kernel launch per forward pass from
    the live parameters / running statistics (`refresh`), so CUDA-graph replays and interleaved training always see current values.
    `bn._rih_fold = (scale, shift)` are views into the flat buffers; conv2d_bn_eval consumes them.  Inference only (no autograd)."""

    def __init__(self, root):
        self.bns = [m for m in root.modules() if isinstance(m, torch.nn.BatchNorm2d)]
        self.device = None
        self._key = None

    def _build(self):
        dev = self.bns[0].weight.device
        sizes = [m.num_features for m in self.bns]
        offs = [0]
        for c in sizes:
            offs.append(offs[-1] + c)
        total = offs[-1]
        for m in self.bns:
            for t in (m.weight, m.bias, m.running_mean, m.running_var):
                if t is None or not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
                    raise RuntimeError('renderih_b200: BatchNorm folding needs affine fp32 CUDA BatchNorm2d modules with running statistics')
        self.table = torch.tensor([[t.data_ptr() for t in (m.weight, m.bias, m.running_mean, m.running_var)] for m in self.bns],
                                  dtype=torch.int64).to(dev)
        self.chan_bn = torch.repeat_interleave(torch.arange(len(sizes), dtype=torch.int32), torch.tensor(sizes)).to(dev)
        self.bn_off = torch.tensor(offs[:-1], dtype=torch.int32).to(dev)
        self.eps = torch.tensor([m.eps for m in self.bns], dtype=torch.float32).to(dev)
        self.scale = torch.empty(total, device=dev)
        self.shift = torch.empty(total, device=dev)
        self.total = total
        for m, o, c in zip(self.bns, offs, sizes):
            m._rih_fold = (self.scale[o:o + c], self.shift[o:o + c])
        self.device = dev

    def refresh(self):
        if not self.bns:
            return
        key = tuple(t.data_ptr() for m in self.bns for t in (m.weight, m.bias, m.running_mean, m.running_var))
        if key != self._key:           # first use, or a parameter / buffer was re-allocated (.to(), load with assign=True ...)
            if torch.cuda.is_current_stream_capturing():
                if self._key is None:
                    raise RuntimeError('renderih_b200: run one eval-mode forward before capturing it into a CUDA graph (BatchNorm fold table)')
                raise RuntimeError('renderih_b200: BatchNorm storage moved since the fold table was built; cannot rebuild it during capture')
            self._build()
            self._key = key
        call('rih_bn_fold', self.table.data_ptr(), self.chan_bn.data_ptr(), self.bn_off.data_ptr(), _p(self.eps), _p(self.scale), _p(self.shift),
             self.total, _stream())


def bn_fold_refresh(root):
    """Recompute the folded BatchNorm vectors of `root` (cached BnFold) when the folded inference path applies; returns True when it does."""
    if torch.is_grad_enabled():
        return False
    f = root.__dict__.get('_rih_bn_fold')
    if f is None:
        f = BnFold(root)
        root.__dict__['_rih_bn_fold'] = f
    f.refresh()
    return True


def conv2d_bn_eval(x, w, N, H, W, stride, pad, fold, order=0, relu=True, res=None):
    """Convolution + eval-mode BatchNorm (+ residual)(+ ReLU) in one kernel (rih_conv2d_bn_eval_fwd); fold = (scale, shift) from BnFold.
    order 0: Conv -> BN -> (+res) -> ReLU (torchvision blocks); order 1: Conv -> ReLU -> BN (models/encoder.py:52-54).  No autograd."""
    if torch.is_grad_enabled() and (x.requires_grad or w.requires_grad):
        raise RuntimeError('renderih_b200: conv2d_bn_eval is an inference kernel (call it under torch.no_grad())')
    x = _rows(x); _w_phys(_check(w, 'weight'))
    Cout, Cin, R, S = w.shape
    assert x.shape == (N * H * W, Cin), (x.shape, N, H, W, Cin)
    g, Ho, Wo = _geom(N, H, W, Cin, Cout, R, S, stride, pad, _ld(x), Cout)
    scale, shift = fold
    assert scale.numel() == Cout and shift.numel() == Cout
    if res is not None:
        res = _rows(res)
        assert res.shape == (N * Ho * Wo, Cout), (res.shape, N, Ho, Wo, Cout)
    y = torch.empty((N * Ho * Wo, Cout), device=x.device, dtype=torch.float32)
    call('rih_conv2d_bn_eval_fwd', _p(x), _p(w), _p(y), g, _p(scale), _p(shift), int(order), int(relu), _p(res), _ld(res) if res is not None else 0,
         _p(_conv_ws(g, 0, x.device)), _stream())
    return y


class PatchifyFn(Function):
    """Non-overlapping p x p patches as rows: [N*H*W, C] -> [N*(H/p)*(W/p), p*p*C]  (kernel == stride convolutions of
    img_feat_to_grid, models/model_attn/img_attn.py:46-48,60, become one dense GEMM)."""

    @staticmethod
    def forward(ctx, x, N, H, W, p):
        x = _rows(x)
        C = x.shape[1]
        P = torch.empty((N * (H // p) * (W // p), p * p * C), device=x.device, dtype=torch.float32)
        call('rih_patchify', _p(x), _ld(x), _p(P), N, H, W, C, p, 0, _stream())
        ctx.dims = (N, H, W, C, p)
        return P

    @staticmethod
    def backward(ctx, dP):
        N, H, W, C, p = ctx.dims
        dP = dP.contiguous()
        dx = torch.empty((N * H * W, C), device=dP.device, dtype=torch.float32)
        call('rih_patchify', _p(dx), C, _p(dP), N, H, W, C, p, 1, _stream())
        return dx, None, None, None, None


def patchify(x, N, H, W, p):
    return PatchifyFn.apply(x, N, H, W, p)


class Im2colFn(Function):
    """Explicit im2col of a few-channel input (the RGB stem): [N*H*W, C] -> [N*Ho*Wo, Kpad]; no gradient w.r.t. the image."""

    @staticmethod
    def forward(ctx, x, N, H, W, R, S, stride, pad, Kpad):
        x = _rows(x)
        C = x.shape[1]
        Ho, Wo = (H + 2 * pad - R) // stride + 1, (W + 2 * pad - S) // stride + 1
        A = torch.empty((N * Ho * Wo, Kpad), device=x.device, dtype=torch.float32)
        call('rih_im2col', _p(x), _ld(x), _p(A), N, H, W, C, R, S, stride, pad, Kpad, _stream())
        return A

    @staticmethod
    def backward(ctx, dA):
        raise RuntimeError('renderih_b200: im2col has no input gradient (use it only on inputs that do not require grad)')


def im2col(x, N, H, W, R, S, stride, pad, Kpad):
    assert not x.requires_grad
    return Im2colFn.apply(x, N, H, W, R, S, stride, pad, Kpad)


class StemConvFn(Function):
    """torchvision resnet.conv1 (7x7 / stride 2 / pad 3, 3 -> 64; models/encoder.py:108) as a wgmma implicit GEMM over the zero-bordered NHWC4
    image (csrc/gemm_tc.cuh StemFwdProducer): no im2col buffer (the old path wrote and re-read 671 MB at batch 64).  w224 = the filter
    repacked [64][7][8][4].  The image receives no gradient."""

    @staticmethod
    def forward(ctx, xp, w224, N, H, W, stats):
        y = torch.empty((N * (H // 2) * (W // 2), 64), device=xp.device, dtype=torch.float32)
        call('rih_stem_conv_fwd', _p(xp), _p(w224), _p(y), N, H, W, _p(stats), _stream())
        ctx.save_for_backward(xp)
        ctx.dims = (N, H, W)
        return y

    @staticmethod
    def backward(ctx, dy):
        (xp,) = ctx.saved_tensors
        N, H, W = ctx.dims
        dy = _rows(dy.contiguous() if dy.stride(-1) != 1 else dy)
        dw = torch.empty((64, 224), device=dy.device, dtype=torch.float32)
        call('rih_stem_conv_wgrad', _p(dy), _ld(dy), _p(xp), _p(dw), N, H, W, 0, _stream())
        return None, dw, None, None, None, None


def stem_supported(H, W):
    """The implicit-GEMM stem needs a tensor-core convolution mode and 256 x 256 images (one output row = one 128-pixel tile)."""
    return MODE['conv'] != 'simt' and H == W == 256


def stem_conv(img, weight, stats=None, fold=None):
    """img: [N,3,H,W] (no gradient), weight: conv1.weight [64,3,7,7] channels_last.  -> NHWC rows [N*(H/2)*(W/2), 64]."""
    img = _check(img).contiguous()
    N, C, H, W = img.shape
    assert C == 3 and tuple(weight.shape) == (64, 3, 7, 7) and not img.requires_grad
    xp = torch.empty((N, H + 6, W + 8, 4), device=img.device, dtype=torch.float32)
    call('rih_nchw_to_nhwc4_pad', _p(img), _p(xp), N, H, W, _stream())
    # [64,3,7,7] (memory [64][7][7][3]) -> [64][7][8][4]: one zero column (the 8th pixel of every 128-byte row) and one zero channel
    w224 = torch.nn.functional.pad(weight.permute(0, 2, 3, 1), (0, 1, 0, 1)).reshape(64, 224)
    if fold is not None:         # inference: eval-mode bn1 + ReLU in the epilogue
        if torch.is_grad_enabled() and weight.requires_grad:
            raise RuntimeError('renderih_b200: the folded stem is an inference kernel (call it under torch.no_grad())')
        y = torch.empty((N * (H // 2) * (W // 2), 64), device=img.device, dtype=torch.float32)
        call('rih_stem_conv_bn_eval_fwd', _p(xp), _p(w224), _p(y), N, H, W, _p(fold[0]), _p(fold[1]), 1, _stream())
        return y
    return StemConvFn.apply(xp, w224, N, H, W, stats)


class BatchNormFn(Function):
    """BatchNorm2d over NHWC rows (+residual)(+relu); training uses per-rank batch statistics (no SyncBN, SURVEY 2.1)."""

    @staticmethod
    def forward(ctx, x, gamma, beta, rmean, rvar, res, training, momentum, eps, relu, mask_input, stats, tracked):
        x = _rows(x)
        M, C = x.shape
        dev = x.device
        mean = torch.empty((C,), device=dev); rstd = torch.empty((C,), device=dev)
        s = _stream()
        if training and stats is None:        # column sums not produced by the convolution's epilogue: one reduction pass
            stats = torch.empty((2 * C,), device=dev, dtype=torch.float64)
            call('rih_bn_colstats', _p(x), _ld(x), M, C, _p(stats), s)
        y = torch.empty((M, C), device=dev, dtype=torch.float32)
        if res is not None:
            res = _rows(res)
        # ONE launch: mean / rstd from the column sums (or the running statistics in eval mode), running-stat + num_batches_tracked
        # update, normalise (+res)(+relu)
        # the ReLU mask of a residual block cannot be recomputed from x alone: the forward kernel records it as one byte per channel quad
        # (1/16 of the output's bytes), which the two backward passes read instead of the output; otherwise it is recomputed from x.
        # Every gradient of a residual block passes that gate (dres, dgamma and dbeta too), so it is recorded whenever a backward may run.
        mask = torch.empty((M, C // 4), device=dev, dtype=torch.uint8) if (relu and res is not None and any(ctx.needs_input_grad)) else None
        call('rih_bn_forward', _p(x), _ld(x), _p(stats) if training else None, M, C, float(eps), float(momentum), _p(gamma), _p(beta),
             _p(res), _ld(res) if res is not None else 0, _p(y), C, int(relu), _p(mask), _p(mean), _p(rstd), _p(rmean), _p(rvar),
             _p(tracked) if training else None, s)
        ctx.save_for_backward(x, gamma, mean, rstd, mask)
        ctx.meta = (training, relu, mask_input, res is not None)
        ctx.beta_ref = beta
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gamma, mean, rstd, mask = ctx.saved_tensors
        y = None
        training, relu, mask_input, has_res = ctx.meta
        dy = _rows(dy.contiguous() if dy.stride(-1) != 1 else dy)
        M, C = x.shape
        dev = dy.device
        dx = torch.empty((M, C), device=dev)
        dres = torch.empty((M, C), device=dev) if (has_res and ctx.needs_input_grad[5]) else None
        tg, tb = _gt(gamma), _gt(ctx.beta_ref)
        direct = tg is not None and tb is not None
        dgamma = tg if direct else torch.empty((C,), device=dev)
        dbeta = tb if direct else torch.empty((C,), device=dev)
        ws = torch.empty((2 * C,), device=dev, dtype=torch.float64)
        call('rih_bn_bwd', _p(dy), _ld(dy), _p(y), C, _p(mask), _p(x), _ld(x), _p(mean), _p(rstd), _p(gamma), _p(ctx.beta_ref),
             _p(dx), C, _p(dres), C, 0, _p(dgamma), _p(dbeta), int(direct), M, C, int(relu), int(training), int(mask_input),
             _p(ws), _stream())
        if direct:
            dgamma = dbeta = None
        return dx, dgamma, dbeta, None, None, dres, None, None, None, None, None, None, None


def batchnorm(x, gamma, beta, rmean, rvar, res=None, training=True, momentum=0.1, eps=1e-5, relu=False, mask_input=False, stats=None,
              tracked=None):
    """tracked: the module's `num_batches_tracked` buffer (int64, on the device): incremented by the kernel in training mode, like
    torch.nn.BatchNorm2d does, so saved checkpoints carry the same buffer values as the reference's."""
    if tracked is not None and not (tracked.is_cuda and tracked.dtype == torch.int64):
        raise RuntimeError('renderih_b200: num_batches_tracked must be an int64 CUDA tensor')
    return BatchNormFn.apply(x, gamma, beta, rmean, rvar, res, training, momentum, eps, relu, mask_input, stats, tracked)


class MaxPoolFn(Function):
    """3x3 / stride 2 / pad 1 max-pool of the torchvision stem (NHWC)."""

    @staticmethod
    def forward(ctx, x, N, H, W):
        x = _check(x).contiguous()
        C = x.shape[1]
        Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        y = torch.empty((N * Ho * Wo, C), device=x.device)
        idx = torch.empty((N * Ho * Wo, C), device=x.device, dtype=torch.uint8)
        call('rih_maxpool3x3s2_fwd', _p(x), _p(y), idx.data_ptr(), N, H, W, C, _stream())
        ctx.save_for_backward(idx)
        ctx.dims = (N, H, W, C)
        return y

    @staticmethod
    def backward(ctx, dy):
        (idx,) = ctx.saved_tensors
        N, H, W, C = ctx.dims
        dy = dy.contiguous()
        dx = torch.empty((N * H * W, C), device=dy.device)
        call('rih_maxpool3x3s2_bwd', _p(dy), idx.data_ptr(), _p(dx), N, H, W, C, _stream())
        return dx, None, None, None


def maxpool3x3s2(x, N, H, W):
    return MaxPoolFn.apply(x, N, H, W)


class Bilinear2xFn(Function):
    """nn.Upsample(scale_factor=2, mode='bilinear', align_corners=True) -- models/encoder.py:51"""

    @staticmethod
    def forward(ctx, x, N, H, W):
        x = _rows(x)
        C = x.shape[1]
        y = torch.empty((N * 4 * H * W, C), device=x.device)
        call('rih_bilinear2x_fwd', _p(x), _ld(x), _p(y), C, N, H, W, C, _stream())
        ctx.dims = (N, H, W, C)
        return y

    @staticmethod
    def backward(ctx, dy):
        N, H, W, C = ctx.dims
        dy = _rows(dy.contiguous() if dy.stride(-1) != 1 else dy)
        dx = torch.zeros((N * H * W, C), device=dy.device)
        call('rih_bilinear2x_bwd', _p(dy), _ld(dy), _p(dx), C, N, H, W, C, _stream())
        return dx, None, None, None


def bilinear2x(x, N, H, W):
    return Bilinear2xFn.apply(x, N, H, W)


class HrConcatFn(Function):
    """cat([y0, up(y1), up(y2), up(y3)], channels) with bilinear align_corners=True up-sampling to y0's size --
    HRnet_encoder.forward, models/encoder.py:226-231.  Each branch is interpolated straight into its channel slice."""

    @staticmethod
    def forward(ctx, N, H0, *xs):
        xs = [_rows(x) for x in xs]
        widths = [x.shape[1] for x in xs]
        Ct = sum(widths)
        y = torch.empty((N * H0 * H0, Ct), device=xs[0].device)
        s = _stream()
        off = 0
        hs = []
        for i, x in enumerate(xs):
            Hi = int(round((x.shape[0] // N) ** 0.5))
            assert Hi * Hi * N == x.shape[0] and H0 % Hi == 0
            hs.append(Hi)
            dst = y.data_ptr() + 4 * off
            if Hi == H0:
                call('rih_copy2d', _p(x), _ld(x), dst, Ct, x.shape[0], x.shape[1], 0, s)
            else:
                call('rih_bilinear_up_fwd', _p(x), _ld(x), dst, Ct, N, Hi, Hi, x.shape[1], H0 // Hi, s)
            off += x.shape[1]
        ctx.meta = (N, H0, widths, hs)
        return y

    @staticmethod
    def backward(ctx, dy):
        N, H0, widths, hs = ctx.meta
        dy = _rows(dy.contiguous() if dy.stride(-1) != 1 else dy)
        s = _stream()
        outs = []
        off = 0
        for i, (w, Hi) in enumerate(zip(widths, hs)):
            if not ctx.needs_input_grad[2 + i]:
                outs.append(None)
            elif Hi == H0:
                outs.append(dy[:, off:off + w])
            else:
                dx = torch.empty((N * Hi * Hi, w), device=dy.device)
                call('rih_bilinear_up_bwd', dy.data_ptr() + 4 * off, _ld(dy), _p(dx), w, N, Hi, Hi, w, H0 // Hi, s)
                outs.append(dx)
            off += w
        return (None, None) + tuple(outs)


def hr_concat(xs, N, H0):
    return HrConcatFn.apply(N, H0, *xs)


class FuseSumFn(Function):
    """y = act(t0 + up(t1) + ...), nearest x f_j up-sampling of coarser terms folded into the read --
    HighResolutionModule.forward fuse sums (models/model_zoo/hrnet.py:222-230) and the `+` of hrnet_mid's head (encoder.py:339-341)."""

    @staticmethod
    def forward(ctx, N, H, relu, factors, *ts):
        ts = [_rows(t) for t in ts]
        C = ts[0].shape[1]
        y = torch.empty((N * H * H, C), device=ts[0].device)
        n = len(ts)
        lds = (ctypes.c_int * n)(*[_ld(t) for t in ts])
        fs = (ctypes.c_int * n)(*factors)
        call('rih_fuse_sum', _ptr_array(ts), lds, fs, n, _p(y), C, N, H, H, C, int(relu), _stream())
        ctx.save_for_backward(y if relu else None)
        ctx.meta = (N, H, C, relu, tuple(factors))
        return y

    @staticmethod
    def backward(ctx, dy):
        (y,) = ctx.saved_tensors
        N, H, C, relu, factors = ctx.meta
        dy = _rows(dy.contiguous() if dy.stride(-1) != 1 else dy)
        s = _stream()
        g = None
        outs = []
        for j, f in enumerate(factors):
            if not ctx.needs_input_grad[4 + j]:
                outs.append(None)
            elif f == 1:
                if g is None:
                    if relu:
                        g = torch.empty((N * H * H, C), device=dy.device)
                        call('rih_relu_bwd', _p(dy), _ld(dy), _p(y), C, _p(g), C, N * H * H, C, s)
                    else:
                        g = dy
                outs.append(g)
            else:
                Hc = H // f
                dx = torch.empty((N * Hc * Hc, C), device=dy.device)
                call('rih_pool_sum', _p(dy), _ld(dy), _p(y) if relu else None, C, _p(dx), C, N, Hc, Hc, C, f, s)
                outs.append(dx)
        return (None, None, None, None) + tuple(outs)


def fuse_sum(terms, factors, N, H, relu=True):
    return FuseSumFn.apply(N, H, relu, tuple(int(f) for f in factors), *terms)


class GapFn(Function):
    """AdaptiveAvgPool2d(1)+Flatten -- models/encoder.py:153-156,166"""

    @staticmethod
    def forward(ctx, x, N, HW):
        x = _rows(x)
        C = x.shape[1]
        y = torch.empty((N, C), device=x.device)
        call('rih_gap_fwd', _p(x), _ld(x), _p(y), N, HW, C, _stream())
        ctx.dims = (N, HW, C)
        return y

    @staticmethod
    def backward(ctx, dy):
        N, HW, C = ctx.dims
        dy = dy.contiguous()
        dx = torch.empty((N * HW, C), device=dy.device)
        call('rih_gap_bwd', _p(dy), _p(dx), C, N, HW, C, 0, _stream())
        return dx, None, None


def global_avgpool(x, N, HW):
    return GapFn.apply(x, N, HW)


class ConcatFn(Function):
    """channel concat of NHWC row tensors -- torch.cat(dim=1) in resnet_mid.forward, models/encoder.py:169-171"""

    @staticmethod
    def forward(ctx, *xs):
        M = xs[0].shape[0]
        widths = [x.shape[1] for x in xs]
        C = sum(widths)
        y = torch.empty((M, C), device=xs[0].device)
        off = 0
        s = _stream()
        for x in xs:
            x = _rows(x)
            call('rih_copy2d', _p(x), _ld(x), y.data_ptr() + 4 * off, C, M, x.shape[1], 0, s)
            off += x.shape[1]
        ctx.widths = widths
        return y

    @staticmethod
    def backward(ctx, dy):
        outs = []
        off = 0
        for w in ctx.widths:
            outs.append(dy[:, off:off + w])
            off += w
        return tuple(outs)


def concat_channels(xs):
    return ConcatFn.apply(*xs)


class ConcatRowsFn(Function):
    """per-batch token concat: y[b] = cat(x1[b] (V1 rows), x2[b] (V2 rows)) -- img_attn.py:86"""

    @staticmethod
    def forward(ctx, x1, x2, B, V1, V2):
        x1, x2 = _rows(x1), _rows(x2)
        F = x1.shape[1]
        y = torch.empty((B * (V1 + V2), F), device=x1.device)
        s = _stream()
        # view y as [B, (V1+V2)*F] and copy the [B, V1*F] / [B, V2*F] blocks (sources must be contiguous)
        x1c, x2c = x1.contiguous(), x2.contiguous()
        call('rih_copy2d', _p(x1c), V1 * F, _p(y), (V1 + V2) * F, B, V1 * F, 0, s)
        call('rih_copy2d', _p(x2c), V2 * F, y.data_ptr() + 4 * V1 * F, (V1 + V2) * F, B, V2 * F, 0, s)
        ctx.dims = (B, V1, V2, F)
        return y

    @staticmethod
    def backward(ctx, dy):
        B, V1, V2, F = ctx.dims
        d3 = dy.contiguous().view(B, V1 + V2, F)
        d1 = torch.empty((B * V1, F), device=dy.device)
        d2 = torch.empty((B * V2, F), device=dy.device)
        s = _stream()
        call('rih_copy2d', _p(d3), (V1 + V2) * F, _p(d1), V1 * F, B, V1 * F, 0, s)
        call('rih_copy2d', d3.data_ptr() + 4 * V1 * F, (V1 + V2) * F, _p(d2), V2 * F, B, V2 * F, 0, s)
        return d1, d2, None, None, None


def concat_rows(x1, x2, B, V1, V2):
    return ConcatRowsFn.apply(x1, x2, B, V1, V2)


class NchwToNhwcFn(Function):
    @staticmethod
    def forward(ctx, x):
        x = _check(x).contiguous()
        N, C, H, W = x.shape
        y = torch.empty((N * H * W, C), device=x.device)
        call('rih_nchw_to_nhwc', _p(x), _p(y), N, C, H * W, C, C, _stream())
        ctx.dims = (N, C, H, W)
        return y

    @staticmethod
    def backward(ctx, dy):
        N, C, H, W = ctx.dims
        dy = _rows(dy.contiguous() if dy.stride(-1) != 1 else dy)
        dx = torch.empty((N, C, H, W), device=dy.device)
        call('rih_nhwc_to_nchw', _p(dy), _p(dx), N, C, H * W, _ld(dy), 0, _stream())
        return dx


def nchw_to_nhwc(x):
    return NchwToNhwcFn.apply(x)


class NhwcToNchwFn(Function):
    @staticmethod
    def forward(ctx, x, N, H, W, c_off, C):
        x = _rows(x)
        y = torch.empty((N, C, H, W), device=x.device)
        call('rih_nhwc_to_nchw', _p(x), _p(y), N, C, H * W, _ld(x), c_off, _stream())
        ctx.dims = (N, H, W, c_off, C, x.shape[1])
        return y

    @staticmethod
    def backward(ctx, dy):
        N, H, W, c_off, C, Ctot = ctx.dims
        dy = dy.contiguous()
        dx = torch.zeros((N * H * W, Ctot), device=dy.device)
        call('rih_nchw_to_nhwc', _p(dy), dx.data_ptr() + 4 * c_off, N, C, H * W, C, Ctot, _stream())
        return dx, None, None, None, None, None


def nhwc_to_nchw(x, N, H, W, c_off=0, C=None):
    return NhwcToNchwFn.apply(x, N, H, W, c_off, x.shape[1] if C is None else C)
