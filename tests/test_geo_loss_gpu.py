"""The CUDA prior and contact terms (renderih_b200/geo_loss.py, csrc/geo_loss.cu) against the unmodified reference's terms and gradients
(tests/golden/geo_loss_synth.pt) and against autograd through the float64 restatement (oracle/geo_loss_ref.py).

Tolerances: 2e-5 relative on the terms, 1e-4 of each gradient's max magnitude (fp32 atan2 / normalisation chains and sums over
B x 4.6k edges)."""
import os

import numpy as np
import pytest
import torch

from oracle import geo_loss_ref as R
from oracle import make_golden_geo_loss as golden
from renderih_b200 import assets as A
from renderih_b200.geo_loss import AnchorLayer, HandPriorLoss
from renderih_b200.manopth import ManoLayer

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'geo_loss_synth.pt')
QUAT = dict(use_pca=False, root_rot_mode='quat', joint_rot_mode='quat', center_idx=0, return_transf=True, return_full_pose=True)
TERM_TOL, GRAD_TOL = 2e-5, 1e-4
KEYS = ('quat_r', 'quat_l', 'verts_r', 'verts_l')
GRADS = ('d_quat_r', 'd_quat_l', 'd_verts_r', 'd_verts_l')


def _rel(a, r):
    return float((a.detach().double().cpu() - r.double().cpu()).abs().max() / r.double().abs().max())


@pytest.fixture(scope='module')
def gold():
    return golden.load(GOLD)


@pytest.fixture(scope='module')
def layers():
    return {side: ManoLayer(mano_root=A.synthetic_mano(0, side), side=side, **QUAT).cuda() for side in ('right', 'left')}


@pytest.fixture(scope='module')
def prior(gold, layers):
    return HandPriorLoss(layers['right'], layers['left'], face_vert_idx=gold['anchor_fvi'].numpy(), anchor_weight=gold['anchor_w'].numpy())


@pytest.fixture(scope='module')
def tab(gold):
    return R.tables(A.synthetic_mano(0, 'right'), A.synthetic_mano(0, 'left'), gold['anchor_fvi'].numpy(), gold['anchor_w'].double().numpy())


def _run(prior, inp, weights=R.WEIGHTS):
    leaves = [inp[k].cuda().float().clone().requires_grad_(True) for k in KEYS]
    prior.set_contacts(inp['anchor_id'], inp['elastic'].float(), inp['mask'])
    terms = prior(*leaves)
    sum(w * t for w, t in zip(weights, terms)).backward()
    return torch.stack([t.detach() for t in terms]), [l.grad for l in leaves]


def _inputs(B, seed, D=4):
    g = torch.Generator().manual_seed(seed)
    out = {}
    for side in ('right', 'left'):
        q = torch.randn(B, 16, 4, generator=g) * 0.45
        q[..., 0] += 1.0
        out['quat_' + side[0]] = q * (0.6 + 0.8 * torch.rand(B, 16, 1, generator=g))
        vt = torch.from_numpy(np.asarray(A.synthetic_mano(0, side)['v_template']))
        out['verts_' + side[0]] = vt[None] + 0.003 * torch.randn(B, 778, 3, generator=g) + 0.01 * torch.randn(B, 1, 3, generator=g)
    out['anchor_id'] = torch.randint(0, 108, (B, 108, D), generator=g)
    out['elastic'] = torch.rand(B, 108, D, generator=g)
    out['mask'] = (torch.rand(B, 108, D, generator=g) < 0.3).long()
    return out


def _check(got, ref, flags=None, what=''):
    terms, grads = got
    rt, rg, rflags = ref
    ok = ~rflags if flags is None else flags
    for i in range(4):
        r = float(rt[i])
        assert abs(float(terms[i]) - r) <= TERM_TOL * max(abs(r), 1e-12), (what, i, float(terms[i]), r)
    for k, g, r in zip(GRADS, grads, rg):
        if k.startswith('d_quat'):
            err = float((g.cpu().double() - r)[ok].abs().max() / r.abs().max()) if ok.any() else 0.0
        else:
            err = _rel(g, r)
        assert err < GRAD_TOL, (what, k, err)


def test_matches_reference_golden(gold, prior):
    for case in gold['cases']:
        terms, grads = _run(prior, case['inputs'])
        rt = case['terms'].double()
        errs = [abs(float(terms[i]) - float(rt[i])) / max(abs(float(rt[i])), 1e-30) for i in range(4)]
        gerrs = [_rel(g, case[k]) for k, g in zip(GRADS, grads)]
        print(case['name'], ['%.1e' % e for e in errs], ['%.1e' % e for e in gerrs])
        assert max(errs) < TERM_TOL and max(gerrs) < GRAD_TOL, (case['name'], errs, gerrs)
    assert float(_run(prior, gold['cases'][1]['inputs'])[0][2]) == 0.0


def test_rest_lengths_and_converter(prior, tab, gold):
    for i, side in enumerate(('right', 'left')):
        assert _rel(prior.static_edge_len[i], tab['rest'][side]) < 1e-5
        for a, g in zip(prior.converter[side], gold['converter'][side]):
            np.testing.assert_allclose(a, g.numpy(), atol=2e-6)


@pytest.mark.parametrize('B', [1, 64, 257, 4096])
def test_batch_sizes_against_oracle(B, prior, tab):
    inp = _inputs(B, B)
    got = _run(prior, inp)
    ref = R.weighted_case(tab, inp)
    print(B, 'flagged samples', int(ref[2].sum()))
    _check(got, ref, what=B)


def test_anchor_layer_forward_backward(gold):
    layer = AnchorLayer(face_vert_idx=gold['anchor_fvi'].numpy(), anchor_weight=gold['anchor_w'].numpy()).cuda()
    inp = _inputs(33, 5)
    v = inp['verts_r'].cuda().float().requires_grad_(True)
    a = layer(v)
    w = torch.randn(33, 108, 3, generator=torch.Generator().manual_seed(1))
    (a * w.cuda()).sum().backward()
    vd = inp['verts_r'].double().requires_grad_(True)
    ra = R.anchors(vd, gold['anchor_fvi'].long(), gold['anchor_w'].double())
    (ra * w.double()).sum().backward()
    assert a.shape == (33, 108, 3)
    assert float((a.detach().cpu().double() - ra.detach()).abs().max()) < 2e-7
    assert _rel(v.grad, vd.grad) < 1e-6


def test_empty_mask_gives_zero_contact_and_gradient(prior, tab):
    inp = _inputs(16, 7)
    inp['mask'] = torch.zeros_like(inp['mask'])
    terms, grads = _run(prior, inp, weights=(0.0, 0.0, 1.0, 0.0))
    assert float(terms[2]) == 0.0 and terms[2].dim() == 0
    assert all(float(g.abs().max()) == 0.0 for g in grads)


def test_bitwise_deterministic(prior):
    inp = _inputs(300, 9)
    runs = [_run(prior, inp) for _ in range(3)]
    for terms, grads in runs[1:]:
        assert torch.equal(terms, runs[0][0]) and all(torch.equal(a, b) for a, b in zip(grads, runs[0][1]))


def test_no_host_synchronisation(prior):
    inp = _inputs(32, 10)
    leaves = [inp[k].cuda().float().requires_grad_(True) for k in KEYS]
    prior.set_contacts(inp['anchor_id'].cuda(), inp['elastic'].cuda(), inp['mask'].cuda())
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        terms = prior(*leaves)
        sum(terms).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert all(l.grad is not None for l in leaves)


def test_cuda_graph_replay_follows_set_contacts(prior, tab):
    """A graph captured over forward + backward replays with the contacts set last, the mask flipping between empty and non-empty."""
    B = 8
    inp = _inputs(B, 11)
    leaves = [inp[k].cuda().float().requires_grad_(True) for k in KEYS]
    prior.set_contacts(inp['anchor_id'], inp['elastic'], inp['mask'])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            terms = prior(*leaves)
            grads = torch.autograd.grad(sum(w * t for w, t in zip(R.WEIGHTS, terms)), leaves)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        terms = torch.stack(prior(*leaves))
        grads = torch.autograd.grad(sum(w * t for w, t in zip(R.WEIGHTS, terms)), leaves)
    g2 = torch.Generator().manual_seed(12)
    for empty in (True, False, True, False):
        ids = torch.randint(0, 108, (B, 108, 4), generator=g2)
        mask = torch.zeros(B, 108, 4, dtype=torch.long) if empty else (torch.rand(B, 108, 4, generator=g2) < 0.5).long()
        el = torch.rand(B, 108, 4, generator=g2)
        prior.set_contacts(ids, el, mask)
        graph.replay()
        torch.cuda.synchronize()
        et = torch.stack(prior(*leaves))
        eg = torch.autograd.grad(sum(w * t for w, t in zip(R.WEIGHTS, et)), leaves)
        assert torch.equal(terms, et) and all(torch.equal(a, b) for a, b in zip(grads, eg))
        assert (float(terms[2].detach()) == 0.0) == empty


def test_full_iteration_in_one_cuda_graph(prior, layers):
    """One optimiser iteration: both manopth hands, the translation adds, HandPriorLoss, NewLoss and the backward, captured in a single
    CUDA graph and replayed, equal to eager."""
    from scipy.spatial import ConvexHull
    from renderih_b200.sdf import NewLoss
    rng = np.random.default_rng(0)
    pts = rng.normal(size=(778, 3))
    pts *= np.array([1.0, 0.6, 0.35]) / np.linalg.norm(pts, axis=1, keepdims=True)
    newloss = NewLoss(faces=ConvexHull(pts).simplices, part_vert=[np.arange(k, 778, 16) for k in range(16)])
    B = 16
    inp = _inputs(B, 13)
    g = torch.Generator().manual_seed(14)
    q = {s: inp['quat_' + s[0]].cuda().requires_grad_(True) for s in ('right', 'left')}
    shape = torch.randn(B, 20, generator=g).cuda().requires_grad_(True)
    tsl = {s: (torch.randn(B, 3, generator=g) * 0.01).cuda().requires_grad_(True) for s in ('right', 'left')}
    prior.set_contacts(inp['anchor_id'], inp['elastic'], inp['mask'])
    leaves = [q['right'], q['left'], shape, tsl['right'], tsl['left']]

    def iteration():
        vr = layers['right'](q['right'], shape[:, :10])[0] + tsl['right'].unsqueeze(1)
        vl = layers['left'](q['left'], shape[:, 10:])[0] + tsl['left'].unsqueeze(1)
        qn, edge, contact, ergo = prior(q['right'], q['left'], vr, vl)
        pen = newloss(torch.cat((vr.unsqueeze(1), vl.unsqueeze(1)), 1)).mean()
        loss = qn + edge + 10.0 * contact + 0.02 * 0.5 * pen + ergo
        return [loss.detach()] + list(torch.autograd.grad(loss, leaves))

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            iteration()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = iteration()
    for step in range(3):
        with torch.no_grad():
            for t in leaves:
                t.add_(0.001 * (step + 1))
        graph.replay()
        torch.cuda.synchronize()
        ref = iteration()
        assert all(torch.equal(a, b) for a, b in zip(out, ref)), step
    assert float(out[0]) > 0


def test_rejected_inputs(prior, gold):
    inp = _inputs(3, 15)
    good = [inp[k].cuda().float() for k in KEYS]
    prior.set_contacts(inp['anchor_id'], inp['elastic'], inp['mask'])
    with pytest.raises(RuntimeError, match='CUDA'):
        prior(good[0].cpu(), *good[1:])
    with pytest.raises(TypeError, match='float32'):
        prior(good[0], good[1], good[2].double(), good[3])
    for bad in ((good[0][:, :15], good[1], good[2], good[3]), (good[0], good[1], good[2][:, :777], good[3]),
                (good[0][:2], good[1][:2], good[2][:2], good[3][:2])):
        with pytest.raises(ValueError):
            prior(*bad)
    terms = prior(good[0].reshape(3, 64), *good[1:])        # [B,64] quaternions are accepted
    assert all(t.dim() == 0 for t in terms)
    fresh = HandPriorLoss(ManoLayer(mano_root=A.synthetic_mano(0, 'right'), side='right', **QUAT).cuda(),
                          ManoLayer(mano_root=A.synthetic_mano(0, 'left'), side='left', **QUAT).cuda(),
                          face_vert_idx=gold['anchor_fvi'].numpy(), anchor_weight=gold['anchor_w'].numpy())
    with pytest.raises(RuntimeError, match='set_contacts'):
        fresh(*good)
    with pytest.raises(ValueError):
        prior.set_contacts(inp['anchor_id'] + 108, inp['elastic'], inp['mask'])
    with pytest.raises(RuntimeError, match='CUDA'):
        prior.anchor_layer(good[2].cpu())
