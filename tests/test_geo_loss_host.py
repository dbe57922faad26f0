"""The float64 restatement of the pose optimiser's prior and contact terms (oracle/geo_loss_ref.py) against the unmodified reference's
terms and gradients (tests/golden/geo_loss_synth.pt), closed forms, the host-side tables of renderih_b200.geo_loss (edge list, converter
matrices, CSRs) and its validation that needs no GPU."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import geo_loss_ref as R
from oracle import make_golden_geo_loss as golden
from oracle import manopth_ref as M
from renderih_b200 import assets as A
from renderih_b200 import geo_loss as GL

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'geo_loss_synth.pt')
GRADS = ('d_quat_r', 'd_quat_l', 'd_verts_r', 'd_verts_l')


def _rel(a, r):
    return float((a.detach().double() - r.double()).abs().max() / r.double().abs().max())


@pytest.fixture(scope='module')
def gold():
    return golden.load(GOLD)


@pytest.fixture(scope='module')
def tab(gold):
    return R.tables(A.synthetic_mano(0, 'right'), A.synthetic_mano(0, 'left'), gold['anchor_fvi'].numpy(), gold['anchor_w'].double().numpy())


def test_oracle_matches_reference_golden(gold, tab):
    assert [c['name'] for c in gold['cases']] == ['contact', 'empty_mask']
    for case in gold['cases']:
        t, grads, flags = R.weighted_case(tab, case['inputs'])
        assert not flags.any(), case['name']
        np.testing.assert_allclose(t.numpy(), case['terms'].double().numpy(), rtol=1e-6, atol=0)
        for k, g in zip(GRADS, grads):
            assert _rel(g, case[k]) < 1e-5, (case['name'], k)
    assert float(gold['cases'][1]['terms'][2]) == 0.0 and float(gold['cases'][0]['terms'][2]) > 0


def test_golden_covers_the_limits(gold, tab):
    """Bend and splank angles on both sides of several limits, a thumb-base twist above 0.5, negative bend angles zeroed before step 4."""
    inp = gold['cases'][0]['inputs']
    below = above = 0
    for side, q in (('right', inp['quat_r']), ('left', inp['quat_l'])):
        Mj = R.local_frames(q.double(), side, tab['conv'][side])
        bend = torch.atan2(Mj[..., 1, 0], Mj[..., 0, 0]) * 180 / math.pi
        lo, hi = torch.tensor([b[0] for b in R.BEND]), torch.tensor([b[1] for b in R.BEND])
        below, above = below + int((bend < lo).sum()), above + int((bend > hi).sum())
        assert int(((bend >= lo) & (bend <= hi)).sum()) > 20
        assert bool((bend[:, 7] < 0).any() or (bend[:, 10] < 0).any()) or side == 'right'
    assert below >= 3 and above >= 3, (below, above)
    twist = (lambda Mj: (Mj[:, 12, 2, 1] - Mj[:, 12, 1, 2]) / 2)(R.local_frames(inp['quat_r'].double(), 'right', tab['conv']['right']))
    assert float(twist.max()) > 0.5


def test_edge_list_and_converter_matrices(gold):
    mr = A.synthetic_mano(0, 'right')
    assert np.array_equal(GL.edge_index(mr['f']), gold['edges'].numpy())
    assert np.array_equal(R.edges(mr['f']), gold['edges'].numpy())
    for side in ('right', 'left'):
        _, joints, transf = R.rest(A.synthetic_mano(0, side), side)
        ours = GL.converter_matrices(side, joints, transf)
        ora = R.converter(side, joints, transf)
        for a, o, g in zip(ours, ora, gold['converter'][side]):
            assert a.dtype == np.float32
            np.testing.assert_allclose(a, g.numpy(), atol=2e-6)
            np.testing.assert_allclose(o, g.double().numpy(), atol=2e-6)


def _identity_inputs(B, tab):
    q = torch.zeros(B, 16, 4, dtype=torch.float64)
    q[..., 0] = 1
    v = {side: R.rest(A.synthetic_mano(0, side), side)[0].expand(B, 778, 3) for side in ('right', 'left')}
    return q, v


def test_closed_forms(tab):
    B = 3
    q, v = _identity_inputs(B, tab)
    ids = torch.zeros(B, 108, 2, dtype=torch.long)
    t, _ = R.terms(tab, q, q, v['right'], v['left'], ids, torch.zeros(B, 108, 2), torch.zeros(B, 108, 2, dtype=torch.long))
    assert float(t[0]) == 0.0                              # unit quaternions
    assert float(t[1]) < 1e-30                             # rest vertices
    assert abs(float(t[3])) < 1e-24                        # identity pose: every local frame is I
    assert float(t[2]) == 0.0                              # empty mask
    # quat-norm of q = 2 (1, 0, 0, 0): ((4 - 1)^2) averaged over the 16 joints, summed over both hands; the pose does not change
    t2, _ = R.terms(tab, 2 * q, q, v['right'], v['left'], ids, torch.zeros(B, 108, 2), torch.zeros(B, 108, 2, dtype=torch.long))
    assert float(t2[0]) == 9.0 and abs(float(t2[3])) < 1e-24


def test_contact_hand_computed():
    """Two anchors, D = 2: sum e |A_main[id] - A_sub|^2 over every entry, over the mask count (e counts even where the mask is 0)."""
    fvi = np.array([[0, 1, 2], [3, 4, 5]])
    aw = np.array([[0.0, 0.0], [1.0, 0.0]])             # anchor 0 = vertex 0, anchor 1 = vertex 4
    vr = torch.zeros(1, 778, 3, dtype=torch.float64)
    vl = torch.zeros(1, 778, 3, dtype=torch.float64)
    vr[0, 0] = torch.tensor([1.0, 0, 0])
    vr[0, 4] = torch.tensor([0.0, 2, 0])
    vl[0, 0] = torch.tensor([0.0, 0, 3])                 # sub anchor 0
    vl[0, 4] = torch.tensor([1.0, 0, 0])                 # sub anchor 1
    a_main, a_sub = R.anchors(vr, torch.from_numpy(fvi), torch.from_numpy(aw)), R.anchors(vl, torch.from_numpy(fvi), torch.from_numpy(aw))
    ids = torch.tensor([[[1, 0], [0, 0]]])
    el = torch.tensor([[[0.5, 2.0], [1.0, 0.25]]])
    mask = torch.tensor([[[1, 0], [1, 0]]])
    picked = a_main[0, ids[0]]
    num = float((el[0].double() * ((a_sub[0][:, None] - picked) ** 2).sum(-1)).sum())
    # |(0,2,0) - (0,0,3)|^2 = 13, |(1,0,0) - (0,0,3)|^2 = 10, |(1,0,0) - (1,0,0)|^2 = 0
    assert num == 0.5 * 13 + 2.0 * 10 + 1.0 * 0 + 0.25 * 0
    tab = {'edges': torch.tensor([[0, 1]]), 'fvi': torch.from_numpy(fvi), 'aw': torch.from_numpy(aw),
           'rest': {'right': torch.zeros(1, dtype=torch.float64), 'left': torch.zeros(1, dtype=torch.float64)},
           'conv': {s: (torch.eye(3, dtype=torch.float64).repeat(16, 1, 1),) * 2 for s in ('right', 'left')}}
    q = torch.zeros(1, 16, 4, dtype=torch.float64)
    q[..., 0] = 1
    t, _ = R.terms(tab, q, q, vr, vl, ids, el, mask)
    assert float(t[2]) == num / 2


def test_anchor_tables_and_csr(gold):
    layer = GL.AnchorLayer(face_vert_idx=gold['anchor_fvi'].numpy(), anchor_weight=gold['anchor_w'].numpy())
    assert layer.face_vert_idx.shape == (1, 108, 3) and layer.face_vert_idx.dtype == torch.int64
    assert layer.anchor_weight.shape == (1, 108, 2) and layer.anchor_weight.dtype == torch.float32
    ptr, ent, coef = layer._ptr.long().numpy(), layer._ent.long().numpy(), layer._coef.double().numpy()
    assert ptr[0] == 0 and ptr[-1] == 3 * 108 and np.all(np.diff(ptr) >= 0)
    # the CSR is the transpose of the dense anchor matrix W [A,778]: anchors = W @ verts
    W = np.zeros((108, 778))
    for v in range(778):
        for p in range(ptr[v], ptr[v + 1]):
            W[ent[p], v] += coef[p]
    v = np.random.default_rng(0).normal(size=(778, 3))
    ref = R.anchors(torch.from_numpy(v)[None], gold['anchor_fvi'].long(), gold['anchor_w'].double())[0].numpy()
    np.testing.assert_allclose(W @ v, ref, atol=1e-6)


def test_anchor_layer_default_tables_from_asset_root():
    root = os.path.join(A.default_asset_root(), GL.ANCHOR_DIR)
    if not os.path.exists(os.path.join(root, 'face_vertex_idx.txt')):
        pytest.skip('reference anchor tables not under the asset root')
    layer = GL.AnchorLayer()
    assert layer.face_vert_idx.shape == (1, 108, 3)


def test_validation_without_gpu(gold):
    fvi, aw = gold['anchor_fvi'].numpy(), gold['anchor_w'].numpy()
    with pytest.raises(ValueError):
        GL.AnchorLayer(face_vert_idx=fvi[:, :2], anchor_weight=aw)
    with pytest.raises(ValueError):
        GL.AnchorLayer(face_vert_idx=fvi, anchor_weight=aw[:5])
    with pytest.raises(ValueError):
        GL.AnchorLayer(face_vert_idx=fvi + 778, anchor_weight=aw)
    with pytest.raises(RuntimeError, match='CUDA'):
        GL.AnchorLayer(face_vert_idx=fvi, anchor_weight=aw)(torch.zeros(2, 778, 3))
    with pytest.raises(TypeError):
        GL.HandPriorLoss(object(), object(), face_vert_idx=fvi, anchor_weight=aw)
    from renderih_b200.manopth import ManoLayer
    quat = dict(use_pca=False, root_rot_mode='quat', joint_rot_mode='quat')
    right = ManoLayer(mano_root=A.synthetic_mano(0, 'right'), side='right', **quat)
    left = ManoLayer(mano_root=A.synthetic_mano(0, 'left'), side='left', **quat)
    with pytest.raises(ValueError, match='left-hand'):
        GL.HandPriorLoss(left, left, face_vert_idx=fvi, anchor_weight=aw)
    with pytest.raises(RuntimeError, match='CUDA'):
        GL.HandPriorLoss(right, left, face_vert_idx=fvi, anchor_weight=aw)
    ids = torch.randint(0, 108, (2, 108, 3), generator=torch.Generator().manual_seed(0))
    ids[0, 0, 0], ids[0, 0, 1] = 0, 107
    el, mk = torch.rand(2, 108, 3), torch.ones(2, 108, 3, dtype=torch.long)
    out = GL.check_contacts(ids, el, mk, 108)
    assert [t.dtype for t in out] == [torch.int32, torch.float32, torch.int32]
    assert torch.equal(out[0].long(), ids) and torch.equal(out[2].long(), mk)
    assert GL.check_contacts(ids, el, mk.bool(), 108)[2].dtype == torch.int32
    for bad, exc in (((ids.float(), el, mk), TypeError), ((ids, el.double(), mk), TypeError), ((ids, el, mk.float()), TypeError),
                     ((ids[:, :100], el[:, :100], mk[:, :100]), ValueError), ((ids, el[:1], mk), ValueError), ((ids, el, mk[..., :2]), ValueError),
                     ((ids + 1, el, mk), ValueError), ((ids - 1, el, mk), ValueError), ((ids[0], el[0], mk[0]), ValueError)):
        with pytest.raises(exc):
            GL.check_contacts(*bad, 108)
