"""The fused tensor-core attention core (rih_attn_tc_fwd / rih_attn_tc_bwd: attn_fused_fwd_kernel, attn_fused_bwd_dq_kernel,
attn_fused_bwd_dkdv_kernel) on what the decoder-shaped tests do not reach: head dims that are not powers of two or up to 128, query / key
counts that are not multiples of the 64-row blocks, three heads, strided q / k / v slices, the exact dropout mask, determinism and the
memory the core needs.  Tolerances as tests/test_ops_gpu.py::test_attention_tensor_core: 3xTF32 5e-5 and TF32 5e-3 relative to each
tensor's max, here against fp64."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = 'cuda'
TOL = {'tf32x3': 5e-5, 'tf32': 5e-3}


@pytest.fixture(scope='module')
def ops():
    from renderih_b200 import ops as o
    yield o
    o.set_gemm_mode('simt', 'simt')


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-20))


def randn(*shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).to(DEV)


def ref_attention(q, k, v, B, H, Sq, Sk, d):
    qh, kh, vh = (t.double().reshape(B, -1, H, d).transpose(1, 2) for t in (q, k, v))
    o = torch.matmul(torch.softmax(torch.matmul(qh, kh.transpose(-1, -2)) / d ** 0.5, -1), vh)
    return o.transpose(1, 2).reshape(B * Sq, H * d)


def run_tc(ops, mode, q, k, v, B, H, Sq, Sk, do, p_drop=0.0, wrt=None):
    ops.set_gemm_mode('simt', mode)
    try:
        o = ops.attention(q, k, v, B, H, Sq, Sk, p_drop=p_drop, impl='tc')
        g = torch.autograd.grad(o, wrt or [q, k, v], do)
    finally:
        ops.set_gemm_mode('simt', 'simt')
    return o, g


SHAPES = [(2, 2, 33, 40, 4), (2, 2, 70, 50, 12), (2, 3, 65, 129, 32), (1, 2, 65, 129, 128), (1, 1, 40, 512, 128), (3, 1, 129, 65, 20)]


@pytest.mark.parametrize('mode', ['tf32x3', 'tf32'])
@pytest.mark.parametrize('B,H,Sq,Sk,d', SHAPES)
def test_fused_attention_matches_fp64(ops, mode, B, H, Sq, Sk, d):
    s = B + H + Sq + Sk + d
    q, k, v = (randn(B * S, H * d, seed=s + i).requires_grad_(True) for i, S in enumerate((Sq, Sk, Sk)))
    do = randn(B * Sq, H * d, seed=s + 3)
    o, grads = run_tc(ops, mode, q, k, v, B, H, Sq, Sk, do)
    qd, kd, vd = (t.detach().double().requires_grad_(True) for t in (q, k, v))
    ref = ref_attention(qd, kd, vd, B, H, Sq, Sk, d)
    refg = torch.autograd.grad(ref, [qd, kd, vd], do.double())
    assert rel(o, ref) < TOL[mode], ('o', rel(o, ref))
    for n, a, r in zip('qkv', grads, refg):
        assert rel(a, r) < TOL[mode], ('d' + n, rel(a, r))


@pytest.mark.parametrize('mode', ['tf32x3', 'tf32'])
def test_fused_attention_strided_slices(ops, mode):
    """q / k / v as column slices of one [rows, 3 HD] buffer (row stride 3 HD), as the fused projection node passes them."""
    B, H, S, d = 3, 4, 97, 16
    qkv = randn(B * S, 3 * H * d, seed=5).requires_grad_(True)
    do = randn(B * S, H * d, seed=6)
    q, k, v = qkv[:, :H * d], qkv[:, H * d:2 * H * d], qkv[:, 2 * H * d:]
    o, (g,) = run_tc(ops, mode, q, k, v, B, H, S, S, do, wrt=[qkv])
    qd = qkv.detach().double().requires_grad_(True)
    ref = ref_attention(qd[:, :H * d], qd[:, H * d:2 * H * d], qd[:, 2 * H * d:], B, H, S, S, d)
    (rg,) = torch.autograd.grad(ref, [qd], do.double())
    assert rel(o, ref) < TOL[mode] and rel(g, rg) < TOL[mode], (rel(o, ref), rel(g, rg))


def test_fused_attention_rejects_wide_heads(ops):
    B, H, S, d = 1, 1, 8, 132
    q = randn(B * S, H * d, seed=1)
    ops.set_gemm_mode('simt', 'tf32x3')
    try:
        with pytest.raises(RuntimeError, match='head dim 132 unsupported'):
            ops.attention(q, q, q, B, H, S, S, impl='tc')
    finally:
        ops.set_gemm_mode('simt', 'simt')


def hash_u32(seed, idx):
    """common.cuh hash_u32 over uint64 indices (numpy, wrapping uint32 arithmetic)."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    key = np.uint32((seed & 0xFFFFFFFF) ^ (((seed >> 32) * 0x9E3779B1) & 0xFFFFFFFF))
    idx = idx.astype(np.uint64)
    with np.errstate(over='ignore'):
        x = ((idx & np.uint64(0xFFFFFFFF)).astype(np.uint32) ^ key) + (idx >> np.uint64(32)).astype(np.uint32) * np.uint32(0x85EBCA6B)
        x ^= x >> np.uint32(16); x *= np.uint32(0x85EBCA6B)
        x ^= x >> np.uint32(13); x *= np.uint32(0xC2B2AE35)
        x ^= x >> np.uint32(16)
    return x


@pytest.mark.parametrize('mode', ['tf32x3', 'tf32'])
def test_fused_attention_dropout_mask(ops, mode):
    """Sk = d = 16 and V = I in every head, so O is the dropped-out probability matrix P~; it must equal the fp64 softmax times the mask
    recomputed on the host from hash_u32(seed + site * 0xD1B54A32D192ED03, ((b H + h) Sq + i) Sk + j) times 1 / (1 - p)."""
    from renderih_b200._lib import call
    B, H, Sq, Sk, d, p, site, seed = 3, 2, 70, 16, 16, 0.3, 5, 0x123456789ABCDEF
    q, k = randn(B * Sq, H * d, seed=1), randn(B * Sk, H * d, seed=2)
    v = torch.eye(Sk, device=DEV).repeat(B, H)
    o = torch.empty(B * Sq, H * d, device=DEV)
    stats = torch.empty(B * H * Sq, 2, device=DEV)
    seed_t = torch.tensor([seed], dtype=torch.int64, device=DEV)
    call('rih_attn_tc_fwd', q.data_ptr(), H * d, k.data_ptr(), H * d, v.data_ptr(), H * d, o.data_ptr(), H * d, stats.data_ptr(), None, 0,
         B, H, Sq, Sk, d, 1.0 / d ** 0.5, p, seed_t.data_ptr(), site, {'tf32x3': 3, 'tf32': 1}[mode], ops._stream())
    torch.cuda.synchronize()
    qh, kh = (t.double().reshape(B, -1, H, d).transpose(1, 2) for t in (q, k))
    P = torch.softmax(torch.matmul(qh, kh.transpose(-1, -2)) / d ** 0.5, -1).cpu().numpy()         # [B, H, Sq, Sk]
    idx = np.arange(B * H * Sq * Sk, dtype=np.uint64).reshape(B, H, Sq, Sk)
    s_eff = (seed + site * 0xD1B54A32D192ED03) & 0xFFFFFFFFFFFFFFFF
    thresh = np.uint32(min(float(np.float32(p)) * 4294967296.0, 4294967295.0))
    keep = hash_u32(s_eff, idx) >= thresh
    inv_keep = float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))
    want = P * keep * inv_keep
    got = o.reshape(B, Sq, H, d).transpose(1, 2).double().cpu().numpy()
    assert 0.2 < 1 - keep.mean() < 0.4
    assert np.array_equal(got == 0, ~keep), 'dropped positions differ from the host mask'
    err = np.abs(got - want).max() / np.abs(want).max()
    assert err < TOL[mode], err


def test_fused_attention_deterministic(ops):
    B, H, Sq, Sk, d = 4, 4, 252, 316, 16
    q, k, v = (randn(B * S, H * d, seed=i).requires_grad_(True) for i, S in enumerate((Sq, Sk, Sk)))
    do = randn(B * Sq, H * d, seed=9)
    outs = []
    for _ in range(2):
        ops.seed_state.manual_seed(77, q.device)
        ops.seed_state.begin_forward()
        o, g = run_tc(ops, 'tf32x3', q, k, v, B, H, Sq, Sk, do, p_drop=0.1)
        outs.append([o] + list(g))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_fused_attention_memory(ops):
    """Forward + backward at the decoder's largest level need less extra memory than one score matrix [B H, Sq, Sk] of fp32."""
    B, H, Sq, Sk, d = 64, 4, 252, 316, 16
    q, k, v = (randn(B * S, H * d, seed=i).requires_grad_(True) for i, S in enumerate((Sq, Sk, Sk)))
    do = randn(B * Sq, H * d, seed=9)
    run_tc(ops, 'tf32x3', q, k, v, B, H, Sq, Sk, do)            # warm-up: module loads, cached allocations
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    o, g = run_tc(ops, 'tf32x3', q, k, v, B, H, Sq, Sk, do)
    torch.cuda.synchronize()
    outputs = sum(t.numel() * 4 for t in [o] + list(g))
    extra = torch.cuda.max_memory_allocated() - base - outputs
    assert extra < B * H * Sq * Sk * 4, (extra, B * H * Sq * Sk * 4)
