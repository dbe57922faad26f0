"""oracle/mano_fit_ref.py against the unmodified reference (tests/golden/mano_fit_synth.pt, made by oracle/make_golden_mano_fit.py) and
the host side of renderih_b200.mano_from_3djoint: the CSV column rule, adaptive_IK to 1e-9 and the learning-rate sequence exactly."""
import os

import numpy as np
import pytest
import torch

from oracle import make_golden_mano_fit as MG
from oracle import mano_fit_ref as M
from renderih_b200 import mano_from_3djoint as MF

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'mano_fit_synth.pt')


@pytest.fixture(scope='module')
def gold():
    return torch.load(GOLD, weights_only=False)


def test_column_rule(gold, tmp_path):
    order = list(range(MG.N_ROWS))
    f = MG.FRAMES[-1]
    order[MG.SCRIPT_ROW], order[f] = order[f], order[MG.SCRIPT_ROW]
    path = str(tmp_path / 'take.csv')
    MG.write_csv(path, gold['take'], order)
    data = MF.read_worldpos_csv(path)
    assert any('End' in k for k in data)                    # the '_End' columns exist and are skipped
    ref = gold['csv_rows'][f]            # parsed by pandas, whose fast float parser may differ from float() in the last bit
    for got in (MF.get_3djoints(data, MG.SCRIPT_ROW), M.get_3djoints(data, MG.SCRIPT_ROW)):
        for a, b in zip(got, ref):
            assert a.shape == (21, 3) and np.allclose(a, b, rtol=0, atol=1e-12)
    left, right = MF.get_3djoints_batch(data, [MG.SCRIPT_ROW, 0])
    assert np.allclose(left[0], ref[0], rtol=0, atol=1e-12) and np.allclose(right[0], ref[1], rtol=0, atol=1e-12)
    assert left.shape == (2, 21, 3)
    assert np.array_equal(left[1], MF.get_3djoints(data, 0)[0])
    for s in ('left', 'right'):
        assert np.array_equal(MF.get_3djoints(data, MG.SCRIPT_ROW)[0 if s == 'left' else 1], gold['frames'][f][s]['joints'])


def test_wrong_joint_count_raises():
    data = {'%s.%s' % (n, a): [0.0] for n in M.LEFT + M.RIGHT for a in 'XYZ'}
    del data['PinkyFinger4_R.X']
    with pytest.raises(ValueError):
        MF.get_3djoints(data, 0)
    data['PinkyFinger4_R.X'] = [0.0]
    data['PinkyFinger4_RX.W'] = [0.0]                      # contains a joint name: a 64th value
    with pytest.raises(ValueError):
        MF.get_3djoints_batch(data, [0])


def test_aik_oracle_matches_reference(gold):
    for name, T, P, R in gold['aik_cases']:
        o = M.adaptive_IK(T, P)
        assert np.array_equal(np.isnan(o), np.isnan(R)), name
        assert np.nanmax(np.abs(o - R)) < 1e-9, name
    names = {c[0] for c in gold['aik_cases']}
    assert {'near_reflection', 'kept_reflection', 'parallel_bone', 'flat_palm', 'flat_palm_1e-9'} <= names
    assert np.isnan(dict((c[0], c[3]) for c in gold['aik_cases'])['parallel_bone']).any()     # the parallel bone's NaN is in the contract
    for f, d in gold['frames'].items():
        for s in ('left', 'right'):
            h = d[s]
            assert np.abs(M.prescale(h['template'], h['joints']) - h['P']).max() < 1e-12
            assert np.abs(M.adaptive_IK(h['template'], h['P']) - h['aik']).max() < 1e-9


def test_lr_sequence_exact(gold):
    for d in gold['frames'].values():
        for s in ('left', 'right'):
            assert d[s]['lrs'] == M.lr_schedule(0.1, 200)
            assert len(d[s]['loss']) == 200
