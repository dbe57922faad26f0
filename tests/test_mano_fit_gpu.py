"""renderih_b200.mano_from_3djoint on the GPU against the unmodified reference (tests/golden/mano_fit_synth.pt) and against an eager loop
of the same CUDA layer with torch.optim.Adam (oracle/mano_fit_ref.eager_fit).

Tolerances:
* adaptive_IK (float64) to 1e-9 with identical NaN positions, flat palms included; mat2aa's forward to 1e-6; its backward to 1e-5 of
  the largest gradient against float64 autograd of renderih_b200.myhand.rotmat_to_axis_angle and to MAT2AA_BWD_TOL of each matrix's
  largest gradient against the reference's own float32 gradient, and NaN in every entry at the exact identity.
* One iteration against the reference: loss LOSS1_TOL relative, gradients GRAD_TOL of the largest entry.  The difference is fp32: the
  CPU and GPU layers round differently, and so does the template the IK starts from.
* The output meshes of the reference's own final pose_R and beta: cur_frame to MESH_TOL and ori_frame (the quaternion manopth path
  against the reference's axis-angle layer) to MESH_TOL of the mesh's extent.
* The graph replay equals the same kernel sequence launched eagerly, bitwise, and the device learning rates equal the schedule exactly.
* Graph against torch.optim.Adam (same kernels for the layer and mat2aa, same start): the L1 gradient is sign(d) / 63, so where a
  residual d sits at rounding level the two loops step in opposite directions, and Adam normalises that to a full step.  Once the
  fit nears its minimum this happens every iteration; pose_R is a free matrix and 21 joints leave directions of the parameters
  unconstrained, so single frames' trajectories split while their losses stay close, and the parameters cannot be held to a fraction
  of an Adam step (measured: 69-96% of the entries end more than a quarter of the last step apart).  So: the first EARLY iterations'
  losses agree to EAGER_LOSS_TOL relative for all but EAGER_FRAC of the (iteration, frame) pairs; in every one of the 200 iterations
  the median over frames of the relative loss difference is below MEDIAN_TOL (B > 1); the final loss agrees to FINAL_LOSS_TOL for all
  but EAGER_FRAC of the frames and its mean over frames to MEAN_LOSS_TOL.
* The full fit against the reference's CPU run starts from the IK of a template that differs in the last float32 bits, and then the
  same drift applies: of the six fits (three frames, two hands) five followed the reference to within 0.6% of the final loss and one
  ended 10% apart (measured on an H100 80GB HBM3 at 700 W).  Every final loss must agree to FIT_LOSS_TOL relative and all but one to
  FIT_CLOSE; where the final loss agrees to FIT_CLOSE, the cur_frame mesh must agree to FIT_VERT_TOL cm (measured at most 0.97 cm on a
  20 cm hand).  convert()'s .obj files are held to FIT_VERT_TOL cm (the ori_frame mesh is 1000 times smaller, and so is its bound)."""
import os

import numpy as np
import pytest
import torch

from oracle import make_golden_mano_fit as MG
from oracle import mano_fit_ref as M
from renderih_b200 import mano_from_3djoint as MF
from renderih_b200.myhand import rotmat_to_axis_angle

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'mano_fit_synth.pt')
LOSS1_TOL, GRAD_TOL = 1e-4, 1e-3
MAT2AA_BWD_TOL, MESH_TOL = 1e-4, 1e-5
EAGER_LOSS_TOL, EAGER_FRAC, EARLY, MEDIAN_TOL = 1e-3, 0.05, 20, 5e-3
FINAL_LOSS_TOL, MEAN_LOSS_TOL = 0.05, 0.01
FIT_LOSS_TOL, FIT_CLOSE, FIT_VERT_TOL = 0.15, 0.01, 1.5


@pytest.fixture(scope='module')
def gold():
    return torch.load(GOLD, weights_only=False)


@pytest.fixture(scope='module')
def fitter():
    return MF.JointFitter(MG.mano_dicts(), 'cuda')


def _frames(gold):
    return sorted(gold['frames'])


def test_aik_kernel_matches_reference(gold):
    assert {'near_reflection', 'kept_reflection', 'parallel_bone', 'flat_palm', 'flat_palm_1e-9'} <= {c[0] for c in gold['aik_cases']}
    for name, T, P, R in gold['aik_cases']:
        out = MF.adaptive_IK(T, P)
        assert out.shape == (1, 16, 3, 3) and out.dtype == np.float64
        assert np.array_equal(np.isnan(out), np.isnan(R)), name
        err = np.nanmax(np.abs(out - R))
        print('%-16s max err %.2e' % (name, err))
        assert err < 1e-9, name
    # the scaling step on the device: template + CSV joints -> the reference's AIK output
    for f in _frames(gold):
        for s in ('left', 'right'):
            h = gold['frames'][f][s]
            T = torch.from_numpy(h['template'].astype(np.float64)).cuda()
            J = torch.from_numpy(h['P']).cuda()[None]
            assert np.abs(MF.adaptive_IK(T, J)[0].cpu().numpy() - h['aik'][0]).max() < 1e-9
            out = torch.empty(1, 16, 3, 3, dtype=torch.float64, device='cuda')
            MF.call('rih_mfit_aik', T.data_ptr(), 0, float(np.linalg.norm(h['template'][9] - h['template'][0])), 1,
                    torch.from_numpy(h['joints']).cuda().data_ptr(), 1, out.data_ptr(), torch.cuda.current_stream().cuda_stream)
            assert np.abs(out[0].cpu().numpy() - h['aik'][0]).max() < 1e-9


def test_mat2aa_forward_and_backward(gold):
    m = gold['mat2aa']
    R = torch.from_numpy(m['R']).cuda().requires_grad_(True)
    aa = MF.mat2aa(R)
    assert (aa.detach().cpu() - torch.from_numpy(m['aa'])).abs().max() < 1e-6
    (aa * torch.from_numpy(m['g_aa']).cuda()).sum().backward()
    dR = R.grad.cpu()
    eye = 5                                                                 # the identity: NaN in every entry, as in the reference
    assert torch.isnan(dR[eye]).all() and np.isnan(m['dR'][eye]).all()
    keep = [i for i in range(R.shape[0]) if i != eye]
    R64 = torch.from_numpy(m['R'][keep]).double().requires_grad_(True)
    (rotmat_to_axis_angle(R64) * torch.from_numpy(m['g_aa'][keep]).double()).sum().backward()
    for i, k in enumerate(keep):
        ref = R64.grad[i]
        err = float((dR[k].double() - ref).abs().max() / ref.abs().max())
        assert err < 1e-5, (k, err)
    for k in keep:                                                          # the reference's own float32 gradient
        ref = torch.from_numpy(m['dR'][k]).double()
        err = float((dR[k].double() - ref).abs().max() / ref.abs().max())
        assert err < MAT2AA_BWD_TOL, (k, err)
    branches = set()
    for r in m['R']:
        t = r.T
        branches.add((0 if t[0, 0] > t[1, 1] else 1) if t[2, 2] < 1e-6 else (2 if t[0, 0] < -t[1, 1] else 3))
    assert branches == {0, 1, 2, 3}


def test_one_iteration_matches_reference(gold, fitter):
    for f in _frames(gold):
        for s in ('left', 'right'):
            h = gold['frames'][f][s]
            J = torch.from_numpy(h['joints']).cuda()[None]
            out = fitter.fit(*((J, None) if s == 'left' else (None, J)), iterations=1, return_history=True)[s]
            sd = fitter._sides[(s, 1, 1, 0.1)]
            loss = float(out['loss'][0, 0])
            assert abs(loss - h['loss'][0]) / h['loss'][0] < LOSS1_TOL, (f, s, loss, h['loss'][0])
            g = sd.grad.cpu()
            gp = torch.cat([g[:9].view(1, 9), g[9:144].view(15, 9)]).reshape(-1)
            for got, ref in ((gp, h['grad0']['pose_R'].reshape(-1)), (g[144:], h['grad0']['beta'].reshape(-1))):
                ref = torch.from_numpy(ref)
                assert float((got - ref).abs().max()) <= GRAD_TOL * float(ref.abs().max()), (f, s)
            # the first Adam step moves every entry by lr = 0.1 against the sign of its gradient
            step = out['pose_R'].cpu().reshape(-1) - torch.from_numpy(h['aik']).float().reshape(-1)
            ref_step = torch.from_numpy(h['after0']['pose_R']).reshape(-1) - torch.from_numpy(h['aik']).float().reshape(-1)
            big = torch.from_numpy(h['grad0']['pose_R']).reshape(-1).abs() > 1e-4
            assert float((step - ref_step)[big].abs().max()) < 1e-4


def _batch(gold, B, seed):
    """B frames: the golden frames' joints with 0.5 cm of noise, both hands."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for s in ('left', 'right'):
        base = torch.from_numpy(np.stack([gold['frames'][f][s]['joints'] for f in _frames(gold)]))
        J = base[torch.arange(B) % base.shape[0]] + torch.randn(B, 21, 3, generator=g, dtype=torch.float64) * 0.5
        out.append(J.cuda())
    return out


@pytest.mark.parametrize('B', [1, 64, 4096])
def test_graph_matches_eager(gold, fitter, B):
    JL, JR = _batch(gold, B, 11 + B)
    out = fitter.fit(JL, JR, return_history=True)
    for s, J in (('left', JL), ('right', JR)):
        sd = fitter._sides[(s, B, 200, 0.1)]
        start = sd.pose64.float()
        pose, beta, hist = M.eager_fit(fitter.mano_layer[s], start, J, MF.mat2aa)
        rel = (out[s]['loss'] - hist).abs() / hist.abs().clamp_min(1e-12)
        early = float((rel[:EARLY] > EAGER_LOSS_TOL).float().mean())
        med = rel.median(dim=1).values
        fin = rel[-1]
        mean_fin = abs(float(out[s]['loss'][-1].mean() - hist[-1].mean())) / float(hist[-1].mean())
        q = lambda t: ' '.join('%.2e' % float(torch.quantile(t.float().cpu(), x)) for x in (0.5, 0.95, 1.0))
        print('B=%d %s: first %d iterations, loss pairs beyond %.0e: %.4f; per-iteration median rel diff max %.2e; final loss rel diff '
              'q50/q95/max %s (mean over frames %.2e)' % (B, s, EARLY, EAGER_LOSS_TOL, early, float(med.max()), q(fin), mean_fin))
        assert early <= EAGER_FRAC
        assert B == 1 or float(med.max()) < MEDIAN_TOL
        assert float((fin > FINAL_LOSS_TOL).float().mean()) <= EAGER_FRAC and mean_fin < MEAN_LOSS_TOL
        assert bool(out[s]['finite'].all())


def test_full_fit_matches_reference(gold, fitter):
    frames = _frames(gold)
    close = 0
    for s in ('left', 'right'):
        J = torch.from_numpy(np.stack([gold['frames'][f][s]['joints'] for f in frames])).cuda()
        out = fitter.fit(*((J, None) if s == 'left' else (None, J)), return_history=True)[s]
        for i, f in enumerate(frames):
            h = gold['frames'][f][s]
            lt, lr_ = float(out['loss'][-1, i]), float(h['loss'][-1])
            verts = (out['verts'][i] * 100).double().cpu().numpy() + h['joints'][0:1]
            vert_err = np.abs(verts - h['cur_obj']).max()
            print('frame %d %s: final loss %.5f vs %.5f, loss trajectory max rel %.2e, cur_obj max err %.3f cm' % (
                f, s, lt, lr_, float(((out['loss'][:, i].cpu() - torch.from_numpy(h['loss'])).abs() / torch.from_numpy(h['loss'])).max()),
                vert_err))
            assert abs(lt - lr_) / lr_ < FIT_LOSS_TOL
            if abs(lt - lr_) / lr_ < FIT_CLOSE:
                close += 1
                assert vert_err < FIT_VERT_TOL
    assert close >= 2 * len(frames) - 1


def test_convert_writes_reference_objs(gold, fitter, tmp_path):
    f = _frames(gold)[-1]
    order = list(range(MG.N_ROWS))
    order[MG.SCRIPT_ROW], order[f] = order[f], order[MG.SCRIPT_ROW]
    csv = str(tmp_path / 'take.csv')
    MG.write_csv(csv, gold['take'], order)
    res = MF.convert(csv, frames=[MG.SCRIPT_ROW, 0], out_dir=str(tmp_path / 'out'), fitter=fitter)
    assert res['frames'] == [MG.SCRIPT_ROW, 0] and res['left']['ori_pose'].shape == (2, 48)
    for s in ('left', 'right'):
        for kind in ('cur', 'ori'):
            got = MG.read_obj(str(tmp_path / 'out' / ('%s_frame%d_%s.obj' % (kind, MG.SCRIPT_ROW, s))))
            ref = gold['frames'][f][s][kind + '_obj']
            print('%s %s obj max err %.3g' % (s, kind, np.abs(got - ref).max()))
            assert got.shape == ref.shape and np.abs(got - ref).max() < FIT_VERT_TOL / (1 if kind == 'cur' else 1000)
        assert os.path.exists(str(tmp_path / 'out' / ('cur_frame0_%s.obj' % s)))


def test_output_meshes_from_reference_parameters(gold, fitter):
    """The reference's final pose_R and beta through the cur_frame path (ManoLayer of mat2aa) and the ori_frame path (ori_pose as
    quaternions through the manopth layer, the left hand's y / z sign included) give its .obj vertices."""
    for f in _frames(gold):
        for s in ('left', 'right'):
            h = gold['frames'][f][s]
            pose_R = torch.from_numpy(h['pose_R']).cuda()
            beta = torch.from_numpy(h['beta']).cuda()
            j0 = h['joints'][0:1]
            with torch.no_grad():
                v, j = fitter.mano_layer[s](pose_R[:, 0], MF.mat2aa(pose_R[:, 1:].reshape(-1, 3, 3)).reshape(1, 45), beta)
                ov, oj = fitter.ori_mesh(s, {'pose_R': pose_R, 'beta': beta})
            cur = ((v - j[:, 0:1]) * 100)[0].double().cpu().numpy() + j0
            ori = ((ov / 1000 - oj[:, 0:1] / 1000) * 100)[0].double().cpu().numpy() + j0
            for name, got, ref in (('cur', cur, h['cur_obj']), ('ori', ori, h['ori_obj'])):
                ext = float(np.abs(ref - ref.mean(0)).max())
                err = float(np.abs(got - ref).max())
                print('frame %d %s %s mesh: max err %.2e of extent %.2e (%.1e)' % (f, s, name, err, ext, err / ext))
                assert err < MESH_TOL * ext, (f, s, name)


def test_lr_kernel_exact():
    lr = torch.zeros(1, dtype=torch.float64, device='cuda')
    step = torch.zeros(1, dtype=torch.int32, device='cuda')
    got = []
    for i in range(200):
        step.fill_(i + 1)                                                   # rih_ge_adam_step has counted step i
        MF.call('rih_mfit_lr_step', lr.data_ptr(), step.data_ptr(), 0.1, 200, torch.cuda.current_stream().cuda_stream)
        got.append(float(lr))
    assert [0.1] + got[:-1] == M.lr_schedule(0.1, 200)


def test_graph_replay_equals_eager_kernels(gold, fitter):
    """The captured iteration replayed 200 times against the same kernel calls launched one by one: bitwise equal results, the step
    counter at 200 and the learning rate at the schedule's value after the last step."""
    JL, JR = _batch(gold, 64, 3)
    graph = fitter.fit(JL, JR, return_history=True)
    eager = {}
    for s, J in (('left', JL), ('right', JR)):
        sd = fitter._sides[(s, 64, 200, 0.1)]
        assert int(sd.step) == 200 and float(sd.lr) == 0.1 * (200 - 199) / 200
        captured = sd.graph

        class _Eager:
            def replay(self, sd=sd):
                sd.iteration(torch.cuda.current_stream().cuda_stream)
        sd.graph = _Eager()
        try:
            eager[s] = fitter.fit(*((J, None) if s == 'left' else (None, J)), return_history=True)[s]
        finally:
            sd.graph = captured
    for s in ('left', 'right'):
        for key in ('pose_R', 'beta', 'verts', 'loss'):
            assert torch.equal(graph[s][key], eager[s][key]), (s, key)


def test_frame_independent_of_batch(gold, fitter):
    JL, JR = _batch(gold, 4096, 5)
    big = fitter.fit(JL, JR)
    for k in (0, 1234, 4095):
        one = fitter.fit(JL[k:k + 1], JR[k:k + 1])
        for s in ('left', 'right'):
            for key in ('pose_R', 'beta', 'verts'):
                assert torch.equal(one[s][key][0], big[s][key][k]), (k, s, key)


def test_rejects_cpu_and_non_float(fitter):
    J = torch.zeros(2, 21, 3, dtype=torch.float64)
    with pytest.raises(RuntimeError):
        fitter.fit(J, None)
    with pytest.raises(TypeError):
        fitter.fit(J.cuda().long(), None)
    with pytest.raises(ValueError):
        fitter.fit(torch.zeros(2, 20, 3, device='cuda'), None)
    with pytest.raises(RuntimeError):
        MF.mat2aa(torch.eye(3)[None])
    with pytest.raises(TypeError):
        MF.mat2aa(torch.eye(3, device='cuda', dtype=torch.float64)[None])
    with pytest.raises(RuntimeError):
        MF.JointFitter(MG.mano_dicts(), 'cpu')
