"""The float64 restatement of the pose optimiser's nature loss (oracle/nature_ref.py) against the unmodified reference's probabilities,
masks, loss and gradients (tests/golden/nature_synth.pt), closed forms of the Euler features, torch's cross-entropy and softmax
backward, the discriminator's state_dict keys and the validation of renderih_b200.nature that needs no GPU."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import make_golden_nature as golden
from oracle import nature_ref as R
from renderih_b200 import nature as N

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'nature_synth.pt')


@pytest.fixture(scope='module')
def gold():
    return golden.load(GOLD)


def test_oracle_matches_reference_golden(gold):
    assert [c['name'] for c in gold['cases']] == ['mixed', 'one_empty', 'both_empty', 'saturated', 'batch_1']
    for case in gold['cases']:
        loss, dr, dl, info = R.weighted_case(case['state_dict'], case['right'], case['left'])
        assert not R.row_flags(info).any(), case['name']
        assert torch.equal(info['mask'], case['mask']), case['name']
        np.testing.assert_allclose(info['probs'].numpy(), case['probs'].double().numpy(), rtol=0, atol=1e-6)
        ref = float(case['loss'])
        assert abs(float(loss) - ref) <= 1e-5 * max(abs(ref), 1e-30), (case['name'], float(loss), ref)
        for g, r in ((dr, case['d_right']), (dl, case['d_left'])):
            scale = float(r.abs().max())
            err = float((g - r.double()).abs().max())
            assert err <= 1e-4 * scale or (scale < 1e-20 and err < 1e-20), (case['name'], err, scale)
            assert float(g[:, 0].abs().max()) == 0.0            # the root rows are not read


def test_golden_covers_the_cases(gold):
    cases = {c['name']: c for c in gold['cases']}
    n = {k: c['mask'].sum(1).tolist() for k, c in cases.items()}
    assert all(0 < k < 32 for k in n['mixed'])
    assert sorted(k == 0 for k in n['one_empty']) == [False, True]
    assert n['both_empty'] == [0, 0] and float(cases['both_empty']['loss']) == 0.0
    p = cases['saturated']['probs'][cases['saturated']['mask']]
    assert bool((p[:, 0] == 1).any()) and bool((p[:, 1] == 0).any())      # the -100 clamps and the 1e-12 floor
    assert float(cases['saturated']['loss']) > 150
    assert cases['batch_1']['batch'] == 1


def _quat_axis(axis, a):
    q = torch.zeros(4, dtype=torch.float64)
    q[0] = math.cos(a / 2)
    q[1 + axis] = math.sin(a / 2)
    return q


def _qmul(p, q):
    w1, x1, y1, z1 = p
    w2, x2, y2, z2 = q
    return torch.stack([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                        w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2])


def test_euler_features_of_known_rotations():
    """R = Rx(a) Ry(b) Rz(c) (euler_angles_to_matrix(.., 'XYZ')) -> features (a, b, c), for any scale of the quaternion."""
    rng = np.random.default_rng(0)
    angles = np.stack([rng.uniform(-3.0, 3.0, 15), rng.uniform(-1.5, 1.5, 15), rng.uniform(-3.0, 3.0, 15)], 1)
    q = torch.stack([_qmul(_qmul(_quat_axis(0, a), _quat_axis(1, b)), _quat_axis(2, c)) for a, b, c in angles])
    for scale in (1.0, 0.3, 2.5):
        f, r02 = R.features((scale * q)[None])
        np.testing.assert_allclose(f[0].reshape(15, 3).numpy(), angles, atol=1e-12)
        np.testing.assert_allclose(r02[0].numpy(), np.sin(angles[:, 1]), atol=1e-12)


def test_bce_and_softmax_backward_match_torch():
    """torch's binary_cross_entropy and softmax on CPU against the oracle's statement, saturated rows included."""
    p0 = torch.tensor([0.3, 0.6, 0.99, 1.0, 1.0, 1 - 1e-7, 0.5], dtype=torch.float32)
    p1 = torch.tensor([0.7, 0.4, 0.01, 0.0, 1e-13, 1e-7, 0.5], dtype=torch.float32)
    p = torch.stack([p0, p1], 1)
    y = torch.cat([torch.zeros(7, 1), torch.ones(7, 1)], 1)
    pt = p.clone().requires_grad_(True)
    lt = torch.nn.functional.binary_cross_entropy(pt, y)
    lt.backward()
    po = p.double().requires_grad_(True)
    lo = R.bce(po, y.double())
    lo.backward()
    assert abs(float(lt) - float(lo)) <= 1e-6 * float(lo)
    np.testing.assert_allclose(pt.grad.double().numpy(), po.grad.numpy(), rtol=1e-6)
    assert float(lo) > 3 * 100 / p.numel()                  # three elements hit the -100 clamps
    # softmax backward p * (g - sum g p), the formula rih_nature_disc_bwd applies
    z = torch.tensor([[0.3, -1.2], [40.0, 0.0], [2.0, 2.0]], dtype=torch.float64, requires_grad=True)
    g = torch.tensor([[1.0, -2.0], [1e12, -1e12], [0.5, 0.25]], dtype=torch.float64)
    s = torch.softmax(z, 1)
    s.backward(g)
    sd = s.detach()
    np.testing.assert_allclose(z.grad.numpy(), (sd * (g - (g * sd).sum(1, keepdim=True))).numpy(), rtol=1e-12, atol=1e-12)


def test_state_dict_keys_and_shapes(gold):
    disc = N.Pos2dDiscriminator(num_joints=15, hid_dim=512, dropout=0.05)
    sd = disc.state_dict()
    assert list(sd.keys()) == gold['keys'] == R.state_dict_keys()
    for name, shape in R.SHAPES.items():
        assert tuple(sd[name + '.weight'].shape) == shape and tuple(sd[name + '.bias'].shape) == (shape[0],)
    assert not any(p.requires_grad for p in disc.parameters())
    disc.load_state_dict(gold['cases'][0]['state_dict'], strict=True)
    assert torch.equal(disc.layer_pred.bias, gold['cases'][0]['state_dict']['layer_pred.bias'])


def test_validation_without_gpu():
    with pytest.raises(NotImplementedError):
        N.Pos2dDiscriminator(num_joints=16)
    with pytest.raises(NotImplementedError):
        N.Pos2dDiscriminator(hid_dim=100)
    with pytest.raises(TypeError):
        N.NatureLoss(object())
    disc = N.Pos2dDiscriminator()
    loss = N.NatureLoss(disc)
    x = torch.zeros(2, 15, 4)
    with pytest.raises(RuntimeError, match='CUDA'):
        disc(x)
    with pytest.raises(RuntimeError, match='CUDA'):
        loss(x, x)
    with pytest.raises(TypeError):
        loss(x.numpy(), x)
