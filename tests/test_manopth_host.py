"""The float64 restatement of the pose optimiser's quaternion hand model (oracle/manopth_ref.py) against the unmodified reference's outputs
and gradients (tests/golden/manopth_synth.pt), closed forms of its quaternion conversion, and the host-side behaviour of
renderih_b200.manopth.ManoLayer (argument validation, MANO loading, no CPU path).  No GPU needed."""
import math
import os
import pickle

import numpy as np
import pytest
import torch

from oracle import make_golden_manopth as golden
from oracle import manopth_ref as M
from renderih_b200 import assets as A
from renderih_b200.manopth import ManoLayer

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'manopth_synth.pt')
QUAT = dict(use_pca=False, root_rot_mode='quat', joint_rot_mode='quat')


def _rel(a, r):
    return float((a.detach().double() - r.double()).abs().max() / r.double().abs().max())


def test_oracle_matches_reference_golden():
    g = golden.load(GOLD)
    assert len(g['cases']) == 24
    for case in g['cases']:
        v, j, tf, dq, db, dt = M.weighted_case(g['inputs'], case['cfg'])
        assert torch.equal(tf[:, :, 3].detach(), torch.tensor([0.0, 0, 0, 1], dtype=torch.float64).expand(5, 16, 4))
        for out, ref in ((v[:, g['vert_idx']], case['verts']), (j, case['joints']), (tf[:, :, :3], case['transf'])):
            assert float((out.detach() - ref.double()).abs().max()) < 1e-6, case['cfg']
        assert _rel(dq, case['d_quat']) < 1e-5, case['cfg']
        for got, ref in ((db, case['d_betas']), (dt, case['d_trans'])):
            assert (got is None) == (ref is None), case['cfg']
            if ref is not None:
                assert _rel(got, ref) < 1e-5, case['cfg']


def test_golden_covers_the_centring_rule():
    g = golden.load(GOLD)
    by = {(c['cfg']['side'], c['cfg']['center_idx'], c['cfg']['trans']): c for c in g['cases'] if c['cfg']['betas'] == 'rows'
          and not c['cfg']['root_palm'] and not c['cfg']['share_betas']}
    for side in ('right', 'left'):
        for centre in (0, 9):
            for tr in ('none', 'zeros'):       # centred: the centre joint sits at the origin
                assert float(by[(side, centre, tr)]['joints'][:, centre].abs().max()) == 0.0
        nz = by[(side, 0, 'nonzero')]
        free = by[(side, None, 'none')]
        assert torch.allclose(nz['joints'], free['joints'] + g['inputs']['trans'][:, None], atol=1e-6)   # trans added, nothing subtracted
        assert float(by[(side, 0, 'zeros')]['d_trans'].abs().max()) > 0      # zero trans still reaches transf


def _axis_angle_R(axis, theta):
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + math.sin(theta) * K + (1 - math.cos(theta)) * K @ K


@pytest.mark.parametrize('scale', [1.0, 0.3, 2.5])
def test_quaternion_conversion_closed_forms(scale):
    rng = np.random.default_rng(7)
    for _ in range(20):
        axis, theta = rng.normal(size=3), rng.uniform(-math.pi, math.pi)
        u = axis / np.linalg.norm(axis)
        q = scale * np.concatenate([[math.cos(theta / 2)], math.sin(theta / 2) * u])
        R = M.quat_to_rotmat(torch.from_numpy(q)).numpy()
        np.testing.assert_allclose(R, _axis_angle_R(axis, theta), atol=1e-12)     # |q| != 1 still gives the rotation of q / |q|
    s = scale
    np.testing.assert_allclose(M.quat_to_rotmat(torch.tensor([s, 0.0, 0, 0], dtype=torch.float64)).numpy(), np.eye(3), atol=1e-15)
    np.testing.assert_allclose(M.quat_to_rotmat(torch.tensor([0.0, s, 0, 0], dtype=torch.float64)).numpy(), np.diag([1.0, -1, -1]), atol=1e-15)
    np.testing.assert_allclose(M.quat_to_rotmat(torch.tensor([s, s, 0, 0], dtype=torch.float64)).numpy(),
                               [[1, 0, 0], [0, 0, -1], [0, 1, 0]], atol=1e-15)           # 90 degrees about x


def test_left_hand_quaternion_sign():
    """Left hands use (w, x, -y, -z): the mirror of the right-hand rotation through the x = 0 plane."""
    q = torch.tensor([[0.9, 0.2, -0.4, 0.3]], dtype=torch.float64)
    R = M.quat_to_rotmat(q)[0]
    Rl = M.quat_to_rotmat(q * torch.tensor([1.0, 1, -1, -1], dtype=torch.float64))[0]
    S = torch.diag(torch.tensor([-1.0, 1, 1], dtype=torch.float64))
    assert torch.allclose(Rl, S @ R @ S, atol=1e-14)


@pytest.mark.parametrize('kw, exc', [
    (dict(root_rot_mode='euler'), KeyError),
    (dict(use_pca=True, joint_rot_mode='quat', root_rot_mode='quat'), TypeError),
    (dict(use_pca=False, joint_rot_mode='axisang', root_rot_mode='quat'), KeyError),
    (dict(use_pca=False, joint_rot_mode='quat', root_rot_mode='rotmat'), KeyError),
    (dict(use_pca=False, joint_rot_mode='euler', root_rot_mode='axisang'), KeyError),
    (dict(), NotImplementedError),                                        # the reference's defaults: PCA + axis-angle
    (dict(use_pca=False), NotImplementedError),
    (dict(use_pca=False, joint_rot_mode='rotmat', root_rot_mode='rotmat'), NotImplementedError),
])
def test_constructor_validation(kw, exc):
    with pytest.raises(exc) as e:
        ManoLayer(mano_root=A.synthetic_mano(0, 'right'), **kw)
    if exc is NotImplementedError:
        assert 'joint_rot_mode=%s' % kw.get('joint_rot_mode', 'axisang') in str(e.value)


def test_loads_mano_root_directory_without_chumpy(tmp_path):
    for side in ('left', 'right'):
        with open(tmp_path / ('MANO_%s.pkl' % side.upper()), 'wb') as f:
            pickle.dump(A.synthetic_mano(0, side), f)
    for side in ('left', 'right'):
        m = A.synthetic_mano(0, side)
        layer = ManoLayer(mano_root=str(tmp_path), side=side, center_idx=0, **QUAT)
        sd = torch.from_numpy(m['shapedirs'])
        if side == 'left':
            sd[:, 0, :] *= -1
        assert torch.equal(layer.th_shapedirs, sd)
        assert torch.equal(layer.th_J_regressor, torch.from_numpy(m['J_regressor'].toarray()))
        assert layer.th_v_template.shape == (1, 778, 3) and layer.th_betas.shape == (1, 10) and float(layer.th_betas.abs().max()) == 0
        assert layer.th_faces.dtype == torch.int64 and layer.th_faces.shape == (1538, 3)
        assert layer.kintree_parents[1:] == [0, 1, 2, 0, 4, 5, 0, 7, 8, 0, 10, 11, 0, 13, 14]
        assert layer.side == side
    names = {n for n, _ in layer.named_buffers()}
    assert {'th_betas', 'th_shapedirs', 'th_posedirs', 'th_v_template', 'th_J_regressor', 'th_weights', 'th_faces'} <= names


def test_cpu_tensors_are_rejected():
    layer = ManoLayer(mano_root=A.synthetic_mano(0, 'right'), **QUAT)
    with pytest.raises(RuntimeError, match='CUDA'):
        layer(torch.randn(2, 64))
