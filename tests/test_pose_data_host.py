"""Host checks of the pose data pipeline's conversion and augmentation stages: the numpy / scipy oracle against the unmodified reference's
outputs (tests/golden/pose_data_synth.pt, oracle/make_golden_pose_data.py), the numpy draw order, and the drivers' bookkeeping
(splicing, file names, save_id, confidence) with the device classes replaced by oracle-backed CPU stand-ins."""
import os

import numpy as np
import pytest
import torch

from oracle import make_golden_pose_data, manopth_ref, pose_data_ref
from renderih_b200 import assets
from renderih_b200 import pose_data

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = torch.load(os.path.join(ROOT, 'tests', 'golden', 'pose_data_synth.pt'), weights_only=False)
SIDES = ('right', 'left')


@pytest.mark.parametrize('side', SIDES)
def test_oracle_converters_equal_reference(side):
    c = G['converter'][side]
    m0, u1, hm = c['inv_m0'], c['inv_u1'], c['hands_mean']
    assert np.array_equal(pose_data_ref.euler_2_mano_quat(c['euler'], side, m0, u1), c['quat'])
    quat = c['quat'].copy()
    assert np.array_equal(pose_data_ref.mano_quat_2_euler(quat, side, m0, u1), c['quat_euler'])
    assert np.array_equal(quat, c['quat'])                           # the input is not modified
    assert np.array_equal(pose_data_ref.axis_angle_2_mano_quat(c['aa'], side, hm), c['aa_quat'])
    assert np.array_equal(pose_data_ref.axis_angle_2_mano_quat(c['aa'], side, hm, flat_hand=True), c['aa_quat_flat'])
    assert np.array_equal(pose_data_ref.mano_quat_flat_2_normal(c['aa_quat'], side, hm, 'aa'), c['flat_aa'])
    assert np.array_equal(pose_data_ref.mano_quat_flat_2_normal(c['aa_quat'], side, hm), c['flat_quat'])


@pytest.mark.parametrize('key', sorted(G['argue']))
def test_oracle_argue_equals_reference_and_draw_order(key):
    name, side = key
    rec = G['argue'][key]
    np.random.seed(rec['seed'])
    u = pose_data_ref.draw_uniforms(*rec['u'].shape[::2])
    assert np.array_equal(u, rec['u'])
    level = make_golden_pose_data.LEVEL if name == 'PoseArguer' else 1.0
    assert np.array_equal(pose_data_ref.argue_pose(rec['euler'], u, name, level), rec['out'])


def test_draw_tables_match_module():
    for name, cls in (('HandPoseArguer', pose_data.HandPoseArguer), ('PoseArguer', pose_data.PoseArguer)):
        assert np.array_equal(pose_data._ranges(cls.NORMAL_BEND, cls.SPLANK), pose_data_ref.ranges(name))
        assert (cls.MAX_BEND, cls.MAX_SPLANK) == pose_data_ref.ARGUERS[name][2:]
    assert pose_data.BEND_JOINTS == pose_data_ref.BEND_JOINTS and pose_data.SPLANK_JOINTS == pose_data_ref.SPLANK_JOINTS


# ------------------------------------------------------------------------------------------------ drivers with CPU stand-ins
def _np(x):
    return x.numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _like(out, x):
    return torch.from_numpy(np.ascontiguousarray(out)) if isinstance(x, torch.Tensor) else out


class _Converter:
    def __init__(self, shape=None, side='right', root=None, device=None):
        self.side, self.device = side, torch.device('cpu')
        c = G['converter'][side]
        self.m0, self.u1, self.hm = c['inv_m0'], c['inv_u1'], c['hands_mean']
        self.tab = manopth_ref.tables(assets.synthetic_mano(0, side), side)

    def euler_2_mano_quat(self, e):
        return _like(pose_data_ref.euler_2_mano_quat(_np(e), self.side, self.m0, self.u1), e)

    def mano_quat_2_euler(self, q):
        return _like(pose_data_ref.mano_quat_2_euler(_np(q), self.side, self.m0, self.u1), q)

    def axis_angle_2_mano_quat(self, aa, flat_hand=False):
        return pose_data_ref.axis_angle_2_mano_quat(aa, self.side, self.hm, flat_hand)

    def mano_quat_flat_2_normal(self, q, return_type='quat'):
        return _like(pose_data_ref.mano_quat_flat_2_normal(_np(q), self.side, self.hm, return_type), q)

    def _root(self, vec, shape):
        q = torch.from_numpy(np.asarray(vec, dtype=np.float64))
        return manopth_ref.forward(self.tab, self.side, q, torch.from_numpy(np.asarray(shape, dtype=np.float64)))[1][:, 0].numpy()

    def trans_2_loc(self, vec, shape, trans, idx):
        return self._root(vec, shape) + np.asarray(trans)

    def loc_2_trans(self, vec, shape, loc, idx):
        return np.asarray(loc) - self._root(vec, shape)


class _Arguer:
    NAME = None

    def __init__(self, shape=None, side='right', root=None, device=None):
        self.hpc = _Converter(side=side)

    def argue_pose(self, pose, argue_size=10, pose_type='quat', random_level=1.0, generator=None):
        e = _np(pose)
        return _like(pose_data_ref.argue_pose(e, pose_data_ref.draw_uniforms(e.shape[0], argue_size), self.NAME, random_level), pose)


class _HandPoseArguer(_Arguer):
    NAME = 'HandPoseArguer'


class _PoseArguer(_Arguer):
    NAME = 'PoseArguer'


@pytest.fixture
def cpu_classes(monkeypatch):
    monkeypatch.setattr(pose_data, 'HandPoseConverter', _Converter)
    monkeypatch.setattr(pose_data, 'HandPoseArguer', _HandPoseArguer)
    monkeypatch.setattr(pose_data, 'PoseArguer', _PoseArguer)


def check_converted(got, want, loc_tol):
    assert list(got) == list(want) and np.array_equal(got['capture_frame_id'], want['capture_frame_id'])
    for s in SIDES:
        assert list(got[s]) == list(want[s])
        assert np.array_equal(got[s]['rot'], want[s]['rot']) if loc_tol == 0 else np.allclose(got[s]['rot'], want[s]['rot'], rtol=0, atol=1e-9)
        assert np.array_equal(got[s]['shape'], want[s]['shape'])
        assert np.abs(got[s]['loc'] - want[s]['loc']).max() <= loc_tol


def check_argued(paths, want, splice):
    """The splices of argue_data concatenated equal the reference's single file; each has splice rows but the last."""
    assert [os.path.basename(p) for p in paths] == ['template_argued_data%d.npy' % k for k in range(len(paths))]
    subs = [np.load(p, allow_pickle=True).item() for p in paths]
    assert all(len(s['capture_frame_id']) == splice for s in subs[:-1])
    got = {k: (np.concatenate([s[k] for s in subs]) if k == 'capture_frame_id' else
               {leaf: np.concatenate([s[k][leaf] for s in subs]) for leaf in want[k]}) for k in want}
    return got


def check_reconverted(paths, want, trans_tol):
    names = [os.path.basename(p) for p in paths]
    assert sorted(names) == want['names'] and len(set(names)) == len(names)
    for n, d in want['files'].items():
        got = np.load(paths[names.index(n)], allow_pickle=True).item()
        assert list(got) == list(d) and list(got['mano_params']) == list(d['mano_params'])
        for s in SIDES:
            g, w = got['mano_params'][s], d['mano_params'][s]
            assert list(g) == list(w) and g['oripose'].size == 0
            assert np.array_equal(g['shape'], w['shape']) and g['pose'].shape == w['pose'].shape
            assert np.abs(g['pose'] - w['pose']).max() <= trans_tol[0]
            assert np.abs(g['trans'] - w['trans']).max() <= trans_tol[1]


def check_birth(paths, want, rot_tol):
    assert [os.path.basename(p) for p in paths] == ['argued_hand_pose_%d.npy' % k for k in range(len(want))]
    for p, w in zip(paths, want):
        d = np.load(p, allow_pickle=True).item()
        assert list(d) == ['rot', 'confidence'] and isinstance(d['confidence'], list)
        assert d['confidence'] == [float(c) for c in w['confidence']]
        assert d['rot'].shape == w['rot'].shape and np.abs(d['rot'] - w['rot']).max() <= rot_tol


def test_driver_bookkeeping(cpu_classes, tmp_path):
    got = pose_data.convert_annotations([G['annotation']] * 10)
    check_converted(got, G['converted'], 1e-4)
    for splice in (5000, 20):
        out = tmp_path / ('argue%d' % splice)
        out.mkdir()
        np.random.seed(G['template_seed'])
        paths = pose_data.argue_data(G['converted'], argue_size=5, splice_data_length=splice, out_dir=str(out))
        assert len(paths) == (1 if splice == 5000 else 3)
        check_converted(check_argued(paths, G['argued'], splice), G['argued'], 0)
    src = tmp_path / 'template_optimized_data0.npy'
    np.save(src, make_golden_pose_data.optimized_layout(G['argued']))
    paths = pose_data.reconvert_optimized([str(src)], G['annotation'], out_dir=str(tmp_path / 'reconv'))
    check_reconverted(paths, G['reconverted'], (0.0, 1e-6))
    S = make_golden_pose_data
    np.random.seed(G['birth_seed'])
    paths = pose_data.birth_data(G['converted'], argue_size=S.BIRTH_A, end_id=S.BIRTH_FRAMES, splice_data_length=S.BIRTH_SPLICE,
                                 out_dir=str(tmp_path))
    check_birth(paths, G['birth'], 0.0)
