"""The CUDA quaternion hand model (renderih_b200/manopth.py, csrc/manopth.cu) against the unmodified reference's outputs and gradients
(tests/golden/manopth_synth.pt) and against autograd through the float64 restatement (oracle/manopth_ref.py).

Tolerances are those of the fused MANO layer's tests: 2e-6 absolute on outputs, 2e-5 of each gradient's max magnitude (fp32 reductions
over 2334 terms)."""
import os

import numpy as np
import pytest
import torch
from scipy.spatial import ConvexHull

from oracle import make_golden_manopth as golden
from oracle import manopth_ref as M
from renderih_b200 import assets as A
from renderih_b200.manopth import ManoLayer


pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'manopth_synth.pt')
QUAT = dict(use_pca=False, root_rot_mode='quat', joint_rot_mode='quat')
OUT_TOL, GRAD_TOL = 2e-6, 2e-5


def _rel(a, r):
    return float((a.detach().double().cpu() - r.double().cpu()).abs().max() / r.double().abs().max())


def _layer(side='right', center_idx=None, transf=True, **kw):
    return ManoLayer(mano_root=A.synthetic_mano(0, side), side=side, center_idx=center_idx, return_transf=transf, **QUAT, **kw).cuda()


def _inputs(B, seed, unit=False):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, 16, 4, generator=g) * 0.35
    q[..., 0] += 1.0
    if not unit:
        q = q * (0.6 + 0.8 * torch.rand(B, 16, 1, generator=g))
    return q.reshape(B, 64), torch.randn(B, 10, generator=g), torch.randn(B, 3, generator=g) * 0.1


def _run(layer, q, betas, trans, weights=None, **kw):
    """CUDA forward + backward of <verts, wv> + <joints, wj> + <transf, wt> -> outputs, gradients (None where no input)."""
    q = q.cuda().clone().requires_grad_(True)
    betas = None if betas is None else betas.cuda().clone().requires_grad_(True)
    trans = None if trans is None else trans.cuda().clone().requires_grad_(True)
    out = layer(q, betas, trans, **kw)
    if weights is not None:
        sum(((o * w.cuda()).sum() for o, w in zip(out, weights) if w is not None)).backward()
    return out, tuple(None if t is None else t.grad for t in (q, betas, trans))


def test_matches_reference_golden():
    g = golden.load(GOLD)
    inp = g['inputs']
    for case in g['cases']:
        c = case['cfg']
        layer = _layer(c['side'], c['center_idx'], return_full_pose=True)
        betas = inp['betas'] if c['betas'] == 'rows' else None
        trans = {'none': None, 'zeros': torch.zeros(5, 3), 'nonzero': inp['trans']}[c['trans']]
        palm = torch.tensor([float(c['root_palm'])], device='cuda')
        share = torch.tensor([float(c['share_betas'])], device='cuda')
        out, grads = _run(layer, inp['quat'], betas, trans, (inp['wv'], inp['wj'], inp['wt'], None), root_palm=palm, share_betas=share)
        v, j, tf, full = out
        assert full.shape == (5, 64) and full.requires_grad
        assert torch.equal(tf[:, :, 3].cpu(), torch.tensor([0.0, 0, 0, 1]).expand(5, 16, 4))
        errs = [float((o.detach().cpu() - case[k]).abs().max()) for o, k in ((v[:, g['vert_idx']], 'verts'), (j, 'joints'), (tf[:, :, :3], 'transf'))]
        gerrs = {k: _rel(t, case[k]) for k, t in zip(('d_quat', 'd_betas', 'd_trans'), grads) if case[k] is not None}
        print(c, ['%.1e' % e for e in errs], {k: '%.1e' % e for k, e in gerrs.items()})
        assert max(errs) < OUT_TOL, (c, errs)
        assert all((case[k] is None) == (t is None) for k, t in zip(('d_quat', 'd_betas', 'd_trans'), grads)), c
        assert all(e < GRAD_TOL for e in gerrs.values()), (c, gerrs)


@pytest.mark.parametrize('B', [1, 64, 257, 4096])
def test_batch_sizes_against_oracle(B):
    q, betas, trans = _inputs(B, B)
    side = 'left' if B % 2 else 'right'
    center = 9 if B < 4096 else 0
    g = torch.Generator().manual_seed(B + 1)
    w = (torch.randn(B, 778, 3, generator=g), torch.randn(B, 21, 3, generator=g), torch.randn(B, 16, 4, 4, generator=g))
    for tr in (None, trans):
        (v, j, tf), grads = _run(_layer(side, center), q, betas, tr, w)
        inp = {'quat': q, 'betas': betas, 'trans': trans, 'wv': w[0], 'wj': w[1], 'wt': w[2]}
        ref = M.weighted_case(inp, {'side': side, 'betas': 'rows', 'trans': 'none' if tr is None else 'nonzero', 'center_idx': center,
                                'root_palm': False, 'share_betas': False})
        for o, r in zip((v, j, tf), ref[:3]):
            assert float((o.detach().cpu().double() - r.detach()).abs().max()) < OUT_TOL, (B, tr is None)
        for got, r in zip(grads, ref[3:]):
            assert (got is None) == (r is None)
            if r is not None:
                assert _rel(got, r) < GRAD_TOL, (B, tr is None)


def test_empty_batch():
    layer = _layer('left', 0)
    q = torch.zeros(0, 64, device='cuda', requires_grad=True)
    betas = torch.zeros(0, 10, device='cuda', requires_grad=True)
    v, j, tf = layer(q, betas, torch.zeros(0, 3, device='cuda'))
    assert v.shape == (0, 778, 3) and j.shape == (0, 21, 3) and tf.shape == (0, 16, 4, 4)
    (v.sum() + j.sum() + tf.sum()).backward()
    assert q.grad.shape == (0, 64) and betas.grad.shape == (0, 10)


def test_optional_outputs_and_gradients():
    """transf not requested (NULL output), each upstream gradient alone (the others NULL), inputs without gradient (NULL d_*)."""
    B = 6
    q, betas, trans = _inputs(B, 11)
    g = torch.Generator().manual_seed(12)
    w = (torch.randn(B, 778, 3, generator=g), torch.randn(B, 21, 3, generator=g), torch.randn(B, 16, 4, 4, generator=g))
    full = M.weighted_case({'quat': q, 'betas': betas, 'trans': trans, 'wv': w[0], 'wj': w[1], 'wt': w[2]},
                       {'side': 'right', 'betas': 'rows', 'trans': 'nonzero', 'center_idx': 9, 'root_palm': True, 'share_betas': False})
    v, j = _layer('right', 9, transf=False)(q.cuda(), betas.cuda(), trans.cuda(), root_palm=True)
    assert float((v.cpu().double() - full[0].detach()).abs().max()) < OUT_TOL
    assert float((j.cpu().double() - full[1].detach()).abs().max()) < OUT_TOL
    layer = _layer('right', 9)
    zero = [torch.zeros_like(x) for x in w]
    for k in range(3):
        wk = [w[i] if i == k else zero[i] for i in range(3)]
        ref = M.weighted_case({'quat': q, 'betas': betas, 'trans': trans, 'wv': wk[0], 'wj': wk[1], 'wt': wk[2]},
                          {'side': 'right', 'betas': 'rows', 'trans': 'nonzero', 'center_idx': 9, 'root_palm': True, 'share_betas': False})
        _, grads = _run(layer, q, betas, trans, [w[i] if i == k else None for i in range(3)], root_palm=True)
        for got, r in zip(grads, ref[3:]):
            assert _rel(got, r) < GRAD_TOL, k
    # only betas need a gradient: d_quat and d_trans are not computed
    b = betas.cuda().requires_grad_(True)
    v, j, tf = layer(q.cuda(), b, trans.cuda())
    (v * w[0].cuda()).sum().backward()
    ref = M.weighted_case({'quat': q, 'betas': betas, 'trans': trans, 'wv': w[0], 'wj': zero[1], 'wt': zero[2]},
                      {'side': 'right', 'betas': 'rows', 'trans': 'nonzero', 'center_idx': 9, 'root_palm': False, 'share_betas': False})
    assert _rel(b.grad, ref[4]) < GRAD_TOL
    # [B,16,4] input and a [1,3] translation broadcast over the batch
    q3 = q.reshape(B, 16, 4).cuda().requires_grad_(True)
    t1 = trans[:1].cuda().requires_grad_(True)
    v, j, tf = layer(q3, betas.cuda(), t1)
    (tf * w[2].cuda()).sum().backward()
    ref = M.weighted_case({'quat': q, 'betas': betas, 'trans': trans[:1].expand(B, 3), 'wv': zero[0], 'wj': zero[1], 'wt': w[2]},
                      {'side': 'right', 'betas': 'rows', 'trans': 'nonzero', 'center_idx': 9, 'root_palm': False, 'share_betas': False})
    assert q3.grad.shape == (B, 16, 4) and _rel(q3.grad.reshape(B, 64), ref[3]) < GRAD_TOL
    assert t1.grad.shape == (1, 3) and _rel(t1.grad, ref[5].sum(0, keepdim=True)) < GRAD_TOL


def test_bitwise_deterministic():
    q, betas, trans = _inputs(300, 5)
    g = torch.Generator().manual_seed(6)
    w = (torch.randn(300, 778, 3, generator=g), torch.randn(300, 21, 3, generator=g), torch.randn(300, 16, 4, 4, generator=g))
    layer = _layer('left', 0)
    runs = [_run(layer, q, betas, trans, w, share_betas=True) for _ in range(3)]
    for out, grads in runs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(out, runs[0][0]))
        assert all(torch.equal(a, b) for a, b in zip(grads, runs[0][1]))


def test_cuda_graph_replay_follows_the_translation_flag():
    """The centring decision is re-evaluated on the device at every replay: a captured graph gives the centred result while the
    static trans tensor is zero and the translated one once it is not."""
    B = 8
    q, betas, trans = _inputs(B, 21)
    layer = _layer('right', 9)
    sq = q.cuda().requires_grad_(True)
    sb, st = betas.cuda(), torch.zeros(B, 3, device='cuda')
    gw = torch.randn(B, 778, 3, device='cuda')
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):                      # warm-up: tables built, kernels loaded
            v, j, tf = layer(sq, sb, st)
            (gq,) = torch.autograd.grad((v * gw).sum() + j.sum() + tf.sum(), sq)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        v, j, tf = layer(sq, sb, st)
        (gq,) = torch.autograd.grad((v * gw).sum() + j.sum() + tf.sum(), sq)
    for tr in (torch.zeros(B, 3), trans, torch.zeros(B, 3), trans * 2):
        st.copy_(tr.cuda())
        graph.replay()
        torch.cuda.synchronize()
        ev, ej, etf = layer(sq, sb, tr.cuda())
        (eg,) = torch.autograd.grad((ev * gw).sum() + ej.sum() + etf.sum(), sq)
        assert torch.equal(v, ev) and torch.equal(j, ej) and torch.equal(tf, etf) and torch.equal(gq, eg)
        centred = float(j[:, 9].abs().max()) == 0.0
        assert centred == (float(tr.abs().max()) == 0.0)


def test_rejected_inputs():
    layer = _layer('right', 0)
    q = torch.randn(3, 64, device='cuda')
    with pytest.raises(RuntimeError, match='CUDA'):
        layer(q.cpu())
    with pytest.raises(RuntimeError, match='CUDA'):
        layer(q, torch.randn(3, 10))
    with pytest.raises(TypeError, match='float32'):
        layer(q.double())
    with pytest.raises(TypeError, match='float32'):
        layer(q, torch.randn(3, 10, device='cuda', dtype=torch.float64))
    for bad in (torch.randn(3, 63, device='cuda'), torch.randn(3, 16, 3, device='cuda'), torch.randn(64, device='cuda')):
        with pytest.raises(ValueError):
            layer(bad)
    with pytest.raises(ValueError):
        layer(q, torch.randn(2, 10, device='cuda'))
    with pytest.raises(ValueError):
        layer(q, None, torch.randn(2, 3, device='cuda'))
    with pytest.raises(IndexError):
        _layer('right', 21)(q)


def test_two_hands_into_newloss_gradient():
    """The optimiser's composition: both hands' vertices into the anti-penetration loss (renderih_b200.sdf.NewLoss).  The loss and its
    vertex gradient are checked against the SDF oracle, and the quaternion gradient against the float64 restatement's vector-Jacobian
    product with that vertex gradient."""
    from oracle import sdf_ref
    from renderih_b200.sdf import NewLoss
    rng = np.random.default_rng(0)
    pts = rng.normal(size=(778, 3))
    pts *= np.array([1.0, 0.6, 0.35]) / np.linalg.norm(pts, axis=1, keepdims=True)
    faces = ConvexHull(pts).simplices
    parts = [np.arange(k, 778, 16) for k in range(16)] + [np.arange(0, 778, 5)]
    B = 2
    qr, br, _ = _inputs(B, 31, unit=True)
    ql, bl, _ = _inputs(B, 32, unit=True)
    shift = {'right': torch.tensor([0.01, 0.0, 0.0]), 'left': torch.tensor([-0.01, 0.0, 0.0])}
    hands, leaves = {}, {}
    for side, q, b in (('right', qr, br), ('left', ql, bl)):
        leaves[side] = q.cuda().requires_grad_(True)
        v, _, _ = _layer(side, 0)(leaves[side], b.cuda(), shift[side].expand(B, 3).cuda())
        v.retain_grad()
        hands[side] = v
    loss = NewLoss(faces=faces, part_vert=parts)(torch.stack([hands['right'], hands['left']], 1))
    loss.sum().backward()
    mult = sdf_ref.part_counts(parts, 778)
    for b in range(B):
        ref = sdf_ref.newloss(torch.stack([hands['right'][b], hands['left'][b]]).detach().cpu().numpy(), faces, mult, rel=1e-6)
        ok = ~ref['ambiguous']
        dv = torch.stack([hands['right'].grad[b], hands['left'].grad[b]]).cpu().numpy()
        el = abs(float(loss[b]) - ref['loss']) / ref['loss']
        eg = float(np.abs(dv - ref['dLdv'])[ok].max() / np.abs(ref['dLdv']).max())
        print('NewLoss[%d] rel err %.1e, vertex gradient %.1e (%d ambiguous vertices)' % (b, el, eg, (~ok).sum()))
        assert ref['loss'] > 0 and ok.mean() > 0.95 and el < 1e-4 and eg < 1e-3, (el, eg)
    for side, q, b in (('right', qr, br), ('left', ql, bl)):
        qd = q.double().requires_grad_(True)
        v, _, _ = M.forward(M.tables(A.synthetic_mano(0, side), side), side, qd, b.double(), shift[side].double().expand(B, 3), 0)
        (gq,) = torch.autograd.grad(v, qd, hands[side].grad.double().cpu())
        err = _rel(leaves[side].grad, gq)
        print('NewLoss d(quat)[%s] rel err %.1e' % (side, err))
        assert float(gq.abs().max()) > 0 and err < GRAD_TOL, (side, err)
