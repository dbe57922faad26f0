"""The mocap driver's host parts against the unmodified reference driver (tests/golden/mocap_synth.pt, oracle/make_golden_mocap.py): the
numpy restatement of search_anchors / update_scene (oracle/mocap_ref.py), the euler <-> MANO quaternion conversions and the attempt table.

The golden vertices came from the reference's CPU ManoLayer; here they come from the float64 statement oracle/manopth_ref.py, so they
differ at rounding level.  The golden generator kept only seeds whose distances and dot products lie at least its recorded margins
(1e-6 m, 2e-6) from every decision, so ids, masks and contacts must agree exactly.  Candidates beyond the unmasked ones tie at 1000.0, where
np.argsort picks an arbitrary order: those ids are not compared."""
import numpy as np
import pytest
import torch

from oracle import manopth_ref, mocap_ref
from renderih_b200 import assets as A
from renderih_b200 import mocap_optimize as MO

GOLD = 'tests/golden/mocap_synth.pt'


@pytest.fixture(scope='module')
def gold():
    import os
    return torch.load(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), GOLD), weights_only=False)


def _verts(side, pose, shape):
    tab = manopth_ref.tables(A.synthetic_mano(0, side), side)
    v = manopth_ref.forward(tab, side, torch.from_numpy(pose).double()[None], torch.from_numpy(shape).double()[None], center_idx=0)[0]
    return v[0].float().numpy()


def test_oracle_matches_reference_search(gold):
    fvi, aw, cls = (t.numpy() for t in gold['anchor_tables'])
    n_tie = 0
    for r in gold['scene']:
        vm = _verts('right', r['hand_pose'], r['hand_shape'][:10])
        vs = _verts('left', r['obj_pose'], r['hand_shape'][10:])
        prev = None if r['prev'] is None else r['prev'].astype(np.int64)
        ma, mn = mocap_ref.frame_geometry(vm, r['hand_tsl'], fvi, aw)
        sa, sn = mocap_ref.frame_geometry(vs, r['obj_tsl'], fvi, aw)
        vc, ids, el, pad, _, _ = mocap_ref.search_anchors(ma, sa, mn, -sn, cls, prev)
        assert np.array_equal(vc, r['vertex_contact'].astype(np.int64))
        assert np.array_equal(pad, r['anchor_padding_mask'].astype(np.int64))
        assert np.abs(el - r['anchor_elasti']).max() <= 1e-6
        ref_ids = r['anchor_id'].astype(np.int64)
        if prev is None:
            n_cand = np.minimum((mocap_ref.dots(-sn, mn) <= mocap_ref.AGAINST).sum(1), 4)
            keep = np.arange(4)[None, :] < n_cand[:, None]
            n_tie += int((~keep).sum())
            assert np.array_equal(ids[keep], ref_ids[keep])
        else:
            assert np.array_equal(ids, ref_ids)
    assert n_tie > 0            # the golden case has sub anchors with fewer than 4 unmasked candidates


def test_golden_covers_contact_and_no_contact(gold):
    fresh = [bool(r['vertex_contact'].any()) for r in gold['scene'] if r['prev'] is None]
    assert any(fresh) and not all(fresh)


def test_conversions_match_hand_pose_converter(gold):
    raw = gold['raw']
    for side in ('right', 'left'):
        m0, u1 = gold['converter'][side]
        q = MO.euler_to_mano_quat(raw[side]['rot'][::gold['optimize_interval']], side, m0, u1)
        assert q.dtype == np.float32
        np.testing.assert_array_max_ulp(q, gold['quat'][side], maxulp=1)
        key = 'hand_pose' if side == 'right' else 'obj_pose'
        final = torch.cat([c['kwargs'][key] for c in gold['calls'][-3:]]).numpy()     # the last attempt's inputs, returned unchanged
        before = final.copy()
        e = MO.mano_quat_to_euler(final, side, m0, u1)
        assert np.array_equal(final, before)
        np.testing.assert_allclose(e, gold['saved'][side]['rot'], rtol=0, atol=1e-9)


def test_attempt_table_matches_reference_sequence(gold):
    n = gold['n_frames'] // gold['optimize_interval'] if gold['n_frames'] % gold['optimize_interval'] == 0 else None
    bs = gold['batch_size']
    sizes = [min(bs, n - s) for s in range(0, n, bs)]
    table = MO.attempt_table(0.0, gold['lambda_contact_loss'])
    want = [(rep, con, it, b) for rep, con, it, _ in table for b in sizes]
    got = [(c['coef_val']['lambda_repulsion_loss'], c['coef_val']['lambda_contact_loss'], c['n_iter'], c['batch_size']) for c in gold['calls']]
    assert got == want
    assert sizes[-1] < bs                                    # the last batch is partial
    assert [k for k, (_, _, _, rec) in enumerate(MO.attempt_table(1.0, 1.0)) if rec] == [0, 3]


def test_update_scene_rejects_cpu_tensors():
    scene = object.__new__(MO.Scene)
    scene.device = torch.device('cuda', 0)
    scene.n_anchors = 108
    t = torch.zeros(2, 16, 4)
    with pytest.raises(RuntimeError):
        MO.Scene.update_scene(scene, t, t, torch.zeros(2, 3), torch.zeros(2, 3), torch.zeros(2, 20))
