"""GPU checks of the pose data pipeline's conversion and augmentation stages (csrc/pose_data.cu, renderih_b200/pose_data.py) against the
unmodified reference's outputs (tests/golden/pose_data_synth.pt), the host conversions of mocap_optimize and the numpy / scipy oracle.
Tolerances: euler angles 1e-9 degree after wrapping the difference into (-180, 180] (on random poses, widened near the gimbal point
by its conditioning); float32 quaternions 1 ulp (with a 1e-15 floor:
near zero, float64 rounding spans several float32 ulps); axis-angle 1e-12 rad; loc / trans the joint tolerance of
tests/test_manopth_gpu.py.  Where outputs are compared with the reference's, the converters take the reference's converter matrices
(the device rest pose's float32 joints differ from a CPU torch forward's in the last bits)."""
import os

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import make_golden_pose_data, pose_data_ref
from renderih_b200 import assets, mocap_optimize, pose_data
from test_pose_data_host import G, SIDES, check_argued, check_birth, check_converted, check_reconverted

pytestmark = pytest.mark.gpu
EULER_TOL, AA_TOL, JOINT_TOL = 1e-9, 1e-12, 2e-6
MANO = {s: assets.synthetic_mano(0, s) for s in SIDES}


def euler_err(a, b):
    d = (np.asarray(a, np.float64) - np.asarray(b, np.float64) + 180.0) % 360.0 - 180.0
    return float(np.abs(d).max())


def conditioned_euler_err(a, b):
    """euler_err in units of its tolerance: EULER_TOL, plus for the first and third angles 1e-12 degree over |cos| of the second,
    since near the gimbal point those two are ill-conditioned and two float64 computations differ by rounding / |cos|."""
    d = np.abs((np.asarray(a, np.float64) - b + 180.0) % 360.0 - 180.0)
    tol = np.full(d.shape, EULER_TOL)
    tol[..., [0, 2]] += 1e-12 / np.abs(np.cos(np.deg2rad(b[..., 1:2])))
    return float((d / tol).max())


def ulp_err(a, b):
    """float32 arrays -> the largest |a - b| in units of (1 ulp of max(|a|, |b|) + 1e-15)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    unit = np.spacing(np.maximum(np.abs(a), np.abs(b))).astype(np.float64) + 1e-15
    return float((np.abs(a.astype(np.float64) - b) / unit).max())


class _RefConverter(pose_data.HandPoseConverter):
    """HandPoseConverter with the reference's converter matrices, as the golden file records them."""

    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        c = G['converter'][self.side]
        self.invM_U_n_0, self.invU_M_n_1 = c['inv_m0'], c['inv_u1']


@pytest.fixture(scope='module')
def conv():
    return {s: pose_data.HandPoseConverter(side=s, root=MANO[s]) for s in SIDES}


@pytest.mark.parametrize('side', SIDES)
def test_converters_match_reference(conv, side):
    c, h = G['converter'][side], _RefConverter(side=side, root=MANO)
    assert np.abs(conv[side].invM_U_n_0 - c['inv_m0']).max() <= 1e-6 and np.abs(conv[side].invU_M_n_1 - c['inv_u1']).max() <= 1e-6
    q = h.euler_2_mano_quat(c['euler'])
    assert q.dtype == np.float32 and q.shape == c['quat'].shape and ulp_err(q, c['quat']) <= 1
    quat = c['quat'].copy()
    assert euler_err(h.mano_quat_2_euler(quat), c['quat_euler']) <= EULER_TOL
    assert np.array_equal(quat, c['quat'])
    assert ulp_err(h.axis_angle_2_mano_quat(c['aa']), c['aa_quat']) <= 1
    assert ulp_err(h.axis_angle_2_mano_quat(c['aa'], flat_hand=True), c['aa_quat_flat']) <= 1
    aa = h.mano_quat_flat_2_normal(c['aa_quat'], return_type='aa')
    assert aa.dtype == np.float64 and np.abs(aa - c['flat_aa']).max() <= AA_TOL
    assert ulp_err(h.mano_quat_flat_2_normal(c['aa_quat']), c['flat_quat']) <= 1
    # CUDA tensors stay on the device
    qt = h.euler_2_mano_quat(torch.from_numpy(c['euler']).cuda())
    assert qt.is_cuda and ulp_err(qt.cpu().numpy(), c['quat']) <= 1


def _random_euler(rng, B):
    e = rng.uniform(-180, 180, size=(B, 16, 3))
    e[..., 1] = rng.uniform(-90, 90, size=(B, 16))
    # exact +-90 degree second angles are left out: at the root (identity converter) they tie from_matrix's branch values, where the
    # quaternion's sign is decided by rounding; the gimbal branch is forced below on quaternions instead
    e[5::11] = 0.0                          # identity joints: the orthogonal (no projection) path where the converter is identity
    return e


@pytest.mark.parametrize('B', [1, 37, 100000])
@pytest.mark.parametrize('side', SIDES)
def test_converters_match_host_and_oracle(conv, side, B):
    rng = np.random.default_rng(B + (0 if side == 'right' else 1))
    h = conv[side]
    m0, u1, hm = h.invM_U_n_0, h.invU_M_n_1, h.th_hands_mean
    e = _random_euler(rng, B)
    q = h.euler_2_mano_quat(e)
    q_host = mocap_optimize.euler_to_mano_quat(e, side, m0, u1)
    assert ulp_err(q, q_host) <= 1 and ulp_err(q, pose_data_ref.euler_2_mano_quat(e, side, m0, u1)) <= 1
    back = h.mano_quat_2_euler(q_host)
    assert conditioned_euler_err(back, mocap_optimize.mano_quat_to_euler(q_host, side, m0, u1)) <= 1
    _, mats = pose_data_ref.mano_quat_2_euler(q_host, side, m0, u1, stages=True)
    gram = mats @ mats.swapaxes(1, 2)
    assert not np.all(np.isclose(gram, np.eye(3), atol=1e-12)), 'no matrix took the SVD projection'
    # the gimbal branch: a root turned by +-90 degrees about y, as float64 CUDA quaternions (the root's converter matrices are identities)
    qg = np.tile(np.asarray([1.0, 0, 0, 0]), (3, 16, 1))
    qg[:, 0] = [[np.cos(np.pi / 4), 0, np.sin(np.pi / 4), 0], [np.cos(np.pi / 4), 0, -np.sin(np.pi / 4), 0], [0.5, 0.5, 0.5, 0.5]]
    eg = h.mano_quat_2_euler(torch.from_numpy(qg).cuda())
    he = mocap_optimize.mano_quat_to_euler(qg, side, m0, u1)
    assert eg.is_cuda and euler_err(eg.cpu().numpy(), he) <= EULER_TOL
    assert np.all(he[:2, 0, 2] == 0) and np.allclose(np.abs(he[:2, 0, 1]), 90)
    aa = (rng.normal(size=(B, 16, 3)) * 0.8).astype(np.float32)
    aa[::5] *= 1e-4                          # from_rotvec's / as_rotvec's small-angle series
    qa = h.axis_angle_2_mano_quat(aa)
    assert ulp_err(qa, pose_data_ref.axis_angle_2_mano_quat(aa, side, hm)) <= 1
    assert np.abs(h.mano_quat_flat_2_normal(qa, return_type='aa') - pose_data_ref.mano_quat_flat_2_normal(qa, side, hm, 'aa')).max() <= AA_TOL
    assert ulp_err(h.mano_quat_flat_2_normal(qa), pose_data_ref.mano_quat_flat_2_normal(qa, side, hm)) <= 1


@pytest.mark.parametrize('key', sorted(G['argue']))
def test_arguers_match_reference(key):
    name, side = key
    rec = G['argue'][key]
    cls = getattr(pose_data, name)
    kw = {'random_level': make_golden_pose_data.LEVEL} if name == 'PoseArguer' else {}
    a = cls(side=side, root=MANO[side])
    np.random.seed(rec['seed'])
    out = a.argue_pose(rec['euler'], argue_size=rec['u'].shape[2], pose_type='euler', **kw)
    assert out.shape == rec['out'].shape and euler_err(out, rec['out']) <= EULER_TOL
    q = a.hpc.euler_2_mano_quat(rec['euler'])            # pose_type 'quat' goes through mano_quat_2_euler first
    np.random.seed(rec['seed'])
    outq = a.argue_pose(q, argue_size=rec['u'].shape[2], **kw)
    ref = pose_data_ref.argue_pose(pose_data_ref.mano_quat_2_euler(q, side, a.hpc.invM_U_n_0, a.hpc.invU_M_n_1), rec['u'], name,
                                   kw.get('random_level', 1.0))
    assert euler_err(outq, ref) <= 1e-7                    # the quaternion round trip's angles feed the adjustment bounds


@pytest.mark.parametrize('B,A', [(1, 1), (37, 15), (2000, 15)])
def test_argue_large_batch_matches_oracle(B, A):
    rng = np.random.default_rng(B)
    a = pose_data.PoseArguer(side='left', root=MANO['left'])
    e = rng.uniform(-100, 100, size=(B, 16, 3))
    np.random.seed(B)
    u = pose_data_ref.draw_uniforms(B, A)
    np.random.seed(B)
    out = a.argue_pose(e, argue_size=A, pose_type='euler', random_level=0.6)
    assert euler_err(out, pose_data_ref.argue_pose(e, u, 'PoseArguer', 0.6)) <= EULER_TOL


def test_philox_path():
    B, A = 4000, 15
    rng = np.random.default_rng(9)
    a = pose_data.HandPoseArguer(side='right', root=MANO['right'])
    e = torch.from_numpy(rng.uniform(-60, 120, size=(B, 16, 3))).cuda()
    state = np.random.get_state()
    o1, adj = a.argue_pose(e, 15, 'euler', generator=123, return_adjust=True)
    o2 = a.argue_pose(e, 15, 'euler', generator=123)
    o3 = a.argue_pose(e, 15, 'euler', generator=124)
    assert o1.is_cuda and torch.equal(o1, o2) and not torch.equal(o1, o3)
    g = torch.Generator(device='cuda').manual_seed(5)
    g1 = a.argue_pose(e, 15, 'euler', generator=g)
    assert not torch.equal(g1, a.argue_pose(e, 15, 'euler', generator=g))      # the generator's offset advances
    assert all(np.array_equal(x, y) for x, y in zip(np.random.get_state(), state) if not isinstance(x, str))   # numpy untouched
    en, adj = e.cpu().numpy(), adj.cpu().numpy().astype(np.float64)
    rg = pose_data_ref.ranges('HandPoseArguer')
    lo = pose_data_ref.adjustments(en, np.zeros((B, 20, A)), rg, 120, 30)
    hi = pose_data_ref.adjustments(en, np.ones((B, 20, A)), rg, 120, 30)
    assert np.all(adj >= lo) and np.all(adj <= hi)
    u = (adj - lo) / (hi - lo)
    assert u.size >= 10 ** 6 and stats.kstest(u.ravel(), 'uniform').pvalue > 1e-4
    ref = pose_data_ref.argue_pose(en, u, 'HandPoseArguer')
    assert euler_err(o1.cpu().numpy(), ref) <= 1e-7          # u recovered from the adjustments up to float64 rounding


def test_drivers_write_golden_outputs(tmp_path, monkeypatch):
    monkeypatch.setattr(pose_data, 'HandPoseConverter', _RefConverter)
    got = pose_data.convert_annotations([G['annotation']] * 10, root=_mano_dir(tmp_path))
    check_converted(got, G['converted'], 100 * JOINT_TOL)
    np.random.seed(G['template_seed'])
    paths = pose_data.argue_data(G['converted'], argue_size=5, out_dir=str(tmp_path), root=_mano_dir(tmp_path))
    argued = check_argued(paths, G['argued'], 5000)
    assert euler_err(np.concatenate([argued[s]['rot'] for s in SIDES]), np.concatenate([G['argued'][s]['rot'] for s in SIDES])) <= EULER_TOL
    for s in SIDES:
        argued[s]['rot'] = G['argued'][s]['rot']
    check_converted(argued, G['argued'], 0)
    src = tmp_path / 'template_optimized_data0.npy'
    np.save(src, make_golden_pose_data.optimized_layout(G['argued']))
    paths = pose_data.reconvert_optimized([str(src)], G['annotation'], out_dir=str(tmp_path / 'reconv'), root=_mano_dir(tmp_path))
    check_reconverted(paths, G['reconverted'], (AA_TOL, JOINT_TOL))
    S = make_golden_pose_data
    np.random.seed(G['birth_seed'])
    paths = pose_data.birth_data(G['converted'], argue_size=S.BIRTH_A, end_id=S.BIRTH_FRAMES, splice_data_length=S.BIRTH_SPLICE,
                                 out_dir=str(tmp_path), root=_mano_dir(tmp_path))
    check_birth(paths, G['birth'], 1e-9)


def _mano_dir(tmp_path):
    import pickle
    d = tmp_path / 'mano'
    if not d.exists():
        d.mkdir()
        for s in SIDES:
            with open(d / ('MANO_%s.pkl' % s.upper()), 'wb') as f:
                pickle.dump(MANO[s], f)
    return str(d)


def test_rejected_inputs(conv):
    h = conv['right']
    e = np.zeros((2, 16, 3))
    with pytest.raises(RuntimeError):
        h.euler_2_mano_quat(torch.zeros(2, 16, 3, dtype=torch.float64))
    with pytest.raises(TypeError):
        h.euler_2_mano_quat(torch.zeros(2, 16, 3, device='cuda'))
    with pytest.raises(TypeError):
        h.mano_quat_2_euler(torch.zeros(2, 16, 4, dtype=torch.int32, device='cuda'))
    with pytest.raises(ValueError):
        h.euler_2_mano_quat(np.zeros((2, 15, 3)))
    with pytest.raises(ValueError):
        h.axis_angle_2_mano_quat(np.zeros((2, 47)))
    a = pose_data.HandPoseArguer(side='right', root=MANO['right'])
    with pytest.raises(NotImplementedError):
        a.argue_pose(e, 2, 'euler', vis=True)
    with pytest.raises(ValueError):
        a.argue_pose(np.zeros((2, 16, 4)), 2, 'euler')
    with pytest.raises(RuntimeError):
        a.argue_pose(torch.zeros(2, 16, 3, dtype=torch.float64), 2, 'euler')
