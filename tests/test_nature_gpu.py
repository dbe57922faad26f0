"""The CUDA nature loss (renderih_b200/nature.py, csrc/nature.cu) against the unmodified reference's probabilities, masks, loss and
gradients (tests/golden/nature_synth.pt) and against the float64 restatement (oracle/nature_ref.py), excluding the rows it flags.

Tolerances: 2e-5 relative on the loss, 1e-4 of each gradient's largest magnitude (fp32 sums of 512 terms through six layers and the
atan2 / asin derivatives)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import make_golden_nature as golden
from oracle import nature_ref as R
from renderih_b200.nature import NatureLoss, Pos2dDiscriminator

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'nature_synth.pt')
LOSS_TOL, GRAD_TOL = 2e-5, 1e-4


def _disc(sd):
    d = Pos2dDiscriminator(num_joints=15, hid_dim=512, dropout=0.05).cuda().eval()
    d.load_state_dict(sd, strict=True)
    return d


def _run(disc, right16, left16):
    """The optimiser's call on [B,16,4] leaves -> (loss, d_right16, d_left16)."""
    leaves = [t.cuda().float().clone().requires_grad_(True) for t in (right16, left16)]
    loss = NatureLoss(disc)(leaves[0][:, 1:], leaves[1][:, 1:])
    loss.backward()
    return loss.detach(), leaves[0].grad, leaves[1].grad


def _case(B, seed, scale=40.0):
    """A mixed-mask case: the weights of make_golden_nature's 'median' rule for these poses."""
    w = golden.weights(('case', B, seed, 1000 + seed, scale, 'median'))
    return R.init_state_dict(*w), golden.poses(B, seed)


def _rel_rows(g, r, ok):
    """max |g - r| over the rows ok [B] of a [B,16,4] gradient, over r's largest magnitude."""
    scale = float(r.abs().max())
    if not ok.any():
        return 0.0
    return float((g.detach().double().cpu() - r.double())[ok].abs().max()) / max(scale, 1e-30)


def test_matches_reference_golden():
    gold = golden.load(GOLD)
    for case in gold['cases']:
        disc = _disc(case['state_dict'])
        loss, dr, dl = _run(disc, case['right'], case['left'])
        with torch.no_grad():
            probs = torch.stack([disc(case['right'][:, 1:].cuda()), disc(case['left'][:, 1:].cuda())]).cpu()
        ref = float(case['loss'])
        el = abs(float(loss) - ref) / max(abs(ref), 1e-30)
        eg = [float((g.cpu() - r).abs().max()) / max(float(r.abs().max()), 1e-30) for g, r in ((dr, case['d_right']), (dl, case['d_left']))]
        ep = float((probs - case['probs']).abs().max())
        print('%-10s loss %.6g rel err %.1e, probs max err %.1e, gradient rel err %s' % (case['name'], float(loss), el, ep, ['%.1e' % e for e in eg]))
        assert loss.dim() == 0
        assert torch.equal(probs[..., 1] < 1.5 * probs[..., 0], case['mask']), case['name']
        assert ep < 5e-6, (case["name"], ep)
        if ref == 0.0:
            assert float(loss) == 0.0
        else:
            assert el < LOSS_TOL, (case['name'], el)
        for g, r in ((dr, case['d_right']), (dl, case['d_left'])):
            if float(r.abs().max()) < 1e-20:           # both-empty and saturated cases: float32 rounds the gradient to (almost) 0
                assert float(g.abs().max()) < 1e-20, case['name']
            else:
                assert _rel_rows(g, r, torch.ones(g.shape[0], dtype=torch.bool)) < GRAD_TOL, case['name']
            assert float(g[:, 0].abs().max()) == 0.0


@pytest.mark.parametrize('B', [1, 64, 257, 4096])
def test_batch_sizes_against_oracle(B):
    sd, (right, left) = _case(B, B)
    loss, dr, dl = _run(_disc(sd), right, left)
    rl, rdr, rdl, info = R.weighted_case(sd, right, left)
    flags = R.row_flags(info)
    print(B, 'masked', info['mask'].sum(1).tolist(), 'flagged rows', int(flags.sum()))
    assert not info['flags']['tie'].any()           # a flipped mask row would change every gradient through n
    assert abs(float(loss) - float(rl)) <= LOSS_TOL * abs(float(rl))
    for h, (g, r) in enumerate(((dr, rdr), (dl, rdl))):
        assert _rel_rows(g, r, ~flags[h]) < GRAD_TOL, (B, h)


def test_classifier_forward_and_input_gradient():
    sd, (right, _) = _case(48, 3, scale=1.0)
    disc = _disc(sd)
    x16 = right.cuda().requires_grad_(True)
    w = torch.randn(48, 2, generator=torch.Generator().manual_seed(0))
    p = disc(x16[:, 1:])                                          # the strided [B,15,4] view
    (p * w.cuda()).sum().backward()
    p60 = disc(x16.detach()[:, 1:].reshape(48, 60))               # [B,60]
    xo = right.double()[:, 1:].clone().requires_grad_(True)
    po, _ = R.discriminator(sd, xo)
    (po * w.double()).sum().backward()
    assert p.shape == (48, 2) and torch.equal(p.detach(), p60)
    assert float((p.detach().cpu().double() - po.detach()).abs().max()) < 2e-6
    assert _rel_rows(x16.grad[:, 1:], xo.grad, torch.ones(48, dtype=torch.bool)) < GRAD_TOL
    assert float(x16.grad[:, 0].abs().max()) == 0.0
    with torch.no_grad():
        assert torch.equal(disc(x16[:, 1:]), p.detach())


def test_empty_masks_give_zero_loss_and_gradient():
    sd, (right, left) = _case(16, 21, scale=1.0)
    sd['layer_pred.bias'] = torch.tensor([0.0, 50.0])             # p1 -> 1: neither hand is masked
    loss, dr, dl = _run(_disc(sd), right, left)
    assert loss.dim() == 0 and float(loss) == 0.0
    assert float(dr.abs().max()) == 0.0 and float(dl.abs().max()) == 0.0


def test_bitwise_deterministic():
    sd, (right, left) = _case(300, 9)
    disc = _disc(sd)
    runs = [_run(disc, right, left) for _ in range(3)]
    for r in runs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(r, runs[0]))


def test_no_host_synchronisation():
    sd, (right, left) = _case(32, 10)
    disc = _disc(sd)
    nature = NatureLoss(disc)
    leaves = [t.cuda().requires_grad_(True) for t in (right, left)]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        loss = nature(leaves[0][:, 1:], leaves[1][:, 1:])
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert all(l.grad is not None for l in leaves)


def test_cuda_graph_replay_while_masks_flip():
    """A graph captured over forward + backward replays correctly while layer_pred's bias moves each hand's mask between empty and
    non-empty."""
    sd, (right, left) = _case(24, 31)
    disc = _disc(sd)
    nature = NatureLoss(disc)
    leaves = [t.cuda().requires_grad_(True) for t in (right, left)]

    def step():
        loss = nature(leaves[0][:, 1:], leaves[1][:, 1:])
        return [loss.detach()] + list(torch.autograd.grad(loss, leaves))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    base = disc.layer_pred.bias.detach().clone()
    seen = set()
    for shift in (0.0, -60.0, 0.0, 60.0, 0.0):         # -60: p1 -> 1 (both empty), +60: every row masked
        with torch.no_grad():
            disc.layer_pred.bias.copy_(base + torch.tensor([shift, 0.0], device='cuda'))
        graph.replay()
        torch.cuda.synchronize()
        ref = step()
        assert all(torch.equal(a, b) for a, b in zip(out, ref)), shift
        seen.add(float(out[0]) == 0.0)
    assert seen == {True, False}


def test_rejected_inputs():
    sd, (right, left) = _case(3, 41, scale=1.0)
    disc = _disc(sd)
    nature = NatureLoss(disc)
    r, l = right[:, 1:].cuda(), left[:, 1:].cuda()
    with pytest.raises(RuntimeError, match='CUDA'):
        nature(r.cpu(), l)
    with pytest.raises(TypeError, match='float32'):
        nature(r, l.double())
    with pytest.raises(TypeError, match='float32'):
        disc(r.half())
    for bad in ((r[:, :14], l), (r, l[:2]), (r.reshape(3, 6, 10), l), (r[:0], l[:0])):
        with pytest.raises(ValueError):
            nature(*bad)
    with pytest.raises(ValueError):
        disc(r.reshape(3, 60)[:, :59])
    assert nature(r.reshape(3, 60), l).dim() == 0                  # [B,60] is accepted
    assert disc(r[:0]).shape == (0, 2)
    with pytest.raises(NotImplementedError):
        Pos2dDiscriminator(num_joints=16)


def test_full_iteration_in_one_cuda_graph():
    """One optimiser iteration with the reference's complete total: both manopth hands, the translation adds, HandPriorLoss, NewLoss,
    F.normalize and NatureLoss (weights 1, 1, 10, 1, 0.01, 1; geo_optimizer_both_batch.py:805-825), forward and backward captured in a
    single CUDA graph and replayed, equal to eager bitwise."""
    from scipy.spatial import ConvexHull
    from oracle import make_golden_geo_loss
    from renderih_b200 import assets as A
    from renderih_b200.geo_loss import HandPriorLoss
    from renderih_b200.manopth import ManoLayer
    from renderih_b200.sdf import NewLoss
    quat = dict(use_pca=False, root_rot_mode='quat', joint_rot_mode='quat', center_idx=0, return_transf=True, return_full_pose=True)
    layers = {s: ManoLayer(mano_root=A.synthetic_mano(0, s), side=s, **quat).cuda() for s in ('right', 'left')}
    geo = torch.load(os.path.join(os.path.dirname(GOLD), 'geo_loss_synth.pt'), weights_only=False)
    prior = HandPriorLoss(layers['right'], layers['left'], face_vert_idx=geo['anchor_fvi'].numpy(), anchor_weight=geo['anchor_w'].numpy())
    rng = np.random.default_rng(0)
    pts = rng.normal(size=(778, 3))
    pts *= np.array([1.0, 0.6, 0.35]) / np.linalg.norm(pts, axis=1, keepdims=True)
    newloss = NewLoss(faces=ConvexHull(pts).simplices, part_vert=[np.arange(k, 778, 16) for k in range(16)])
    B = 16
    sd, _ = _case(B, 51)
    nature = NatureLoss(_disc(sd))
    g = torch.Generator().manual_seed(14)
    q = {s: (torch.randn(B, 16, 4, generator=g) * 0.45 + torch.tensor([1.0, 0, 0, 0])).cuda().requires_grad_(True) for s in ('right', 'left')}
    shape = torch.randn(B, 20, generator=g).cuda().requires_grad_(True)
    tsl = {s: (torch.randn(B, 3, generator=g) * 0.01).cuda().requires_grad_(True) for s in ('right', 'left')}
    prior.set_contacts(torch.randint(0, 108, (B, 108, 4), generator=g), torch.rand(B, 108, 4, generator=g),
                       (torch.rand(B, 108, 4, generator=g) < 0.3).long())
    leaves = [q['right'], q['left'], shape, tsl['right'], tsl['left']]
    assert make_golden_geo_loss.WEIGHTS == (1.0, 1.0, 10.0, 1.0)

    def iteration():
        vr = layers['right'](q['right'], shape[:, :10])[0] + tsl['right'].unsqueeze(1)
        vl = layers['left'](q['left'], shape[:, 10:])[0] + tsl['left'].unsqueeze(1)
        qn, edge, contact, ergo = prior(q['right'], q['left'], vr, vl)
        pen = newloss(torch.cat((vr.unsqueeze(1), vl.unsqueeze(1)), 1)).mean()
        nat = nature(F.normalize(q['right'], dim=-1)[:, 1:], F.normalize(q['left'], dim=-1)[:, 1:])
        loss = qn + edge + 10.0 * contact + ergo + 0.01 * pen + nat
        return [loss.detach(), nat.detach()] + list(torch.autograd.grad(loss, leaves))

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
    assert float(out[1]) > 0 and float(out[0]) > float(out[1])
