"""The mocap driver on the GPU (renderih_b200/mocap_optimize.py, csrc/scene.cu): the kernel against the numpy restatement
oracle/mocap_ref.py on the same device vertices, update_scene and optimize_mocap against the unmodified reference driver
(tests/golden/mocap_synth.pt), optimize_mocap against the eager per-frame driver, and rejected inputs.

On the same vertices the kernel and the oracle perform the same float32 / float64 operations in the same order, so ids, masks, contacts and
optimize_it are exact; elasticities (cos), anchors and normals are held to 1e-6.  Against the golden file the vertices come from a
different hand model implementation (CPU reference against CUDA), see tests/test_mocap_host.py for the margins and the tie rule."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import ge_optimizer_ref as G
from oracle import mocap_ref
from renderih_b200 import assets as A
from renderih_b200 import mocap_optimize as MO

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def gold():
    return torch.load(os.path.join(ROOT, 'tests', 'golden', 'mocap_synth.pt'), weights_only=False)


@pytest.fixture(scope='module')
def scene(gold):
    fvi, aw, cls = (t.numpy() for t in gold['anchor_tables'])
    return MO.Scene(mano_root={s: A.synthetic_mano(0, s) for s in ('right', 'left')}, face_vert_idx=fvi, anchor_weight=aw, class_types=cls)


def _inputs(B, seed):
    g = torch.Generator().manual_seed(seed)
    q = [torch.randn(B, 16, 4, generator=g) * 0.25 + torch.tensor([1.0, 0, 0, 0]) for _ in range(2)]
    t = [torch.tensor([x, 0.0, 0.0]) + 0.02 * torch.randn(B, 3, generator=g) for x in (0.02, -0.02)]
    shape = torch.randn(B, 20, generator=g) * 0.5
    return [x.cuda() for x in (q[0], q[1], t[0], t[1], shape)]


def _oracle(scene, args, prev=None):
    qr, ql, tr, tl, shape = args
    with torch.no_grad():
        vm = scene.main_hand(qr, shape[:, :10])[0].cpu().numpy()
        vs = scene.sub_hand(ql, shape[:, 10:])[0].cpu().numpy()
    fvi, aw, cls = mocap_ref.tables(scene)
    return mocap_ref.scene_frames(vm, vs, tr.cpu().numpy(), tl.cpu().numpy(), fvi, aw, cls, None if prev is None else prev.cpu().numpy())


def _compare(out, ref, what):
    for k in ('anchor_id', 'anchor_padding_mask', 'vertex_contact', 'optimize_it'):
        got = out[k].cpu().numpy()
        assert got.dtype == ref[k].dtype and np.array_equal(got, ref[k]), (what, k)
    for k in ('anchor_elasti', 'obj_anchors', 'obj_normals'):
        err = float(np.abs(out[k].cpu().numpy() - ref[k]).max())
        assert out[k].dtype == torch.float32 and err <= 1e-6, (what, k, err)


@pytest.mark.parametrize('B', [1, 37, 4096])
def test_kernel_against_oracle(scene, B):
    args = _inputs(B, 100 + B)
    out = scene.update_scene(*args)
    ref = _oracle(scene, args)
    _compare(out, ref, 'fresh B=%d' % B)
    print('B=%d: %d frames in contact' % (B, int(out['optimize_it'].sum())))
    prev = out['anchor_id'].flip(-1).contiguous()          # any valid ids
    out2 = scene.update_scene(*args, anchor_id=prev)
    _compare(out2, _oracle(scene, args, prev), 'previous ids B=%d' % B)
    assert torch.equal(out2['anchor_id'], prev)
    assert out2['hand_region'].dtype == torch.int64 and int(out2['hand_region'].abs().sum()) == 0


def _n_cand(scene, args):
    """Per frame and sub anchor: the number of unmasked candidates (capped at 4), from the oracle's normals on these vertices."""
    qr, ql, tr, tl, shape = args
    fvi, aw, _ = mocap_ref.tables(scene)
    with torch.no_grad():
        vm = scene.main_hand(qr, shape[:, :10])[0].cpu().numpy()
        vs = scene.sub_hand(ql, shape[:, 10:])[0].cpu().numpy()
    out = []
    for b in range(len(vm)):
        _, mn = mocap_ref.frame_geometry(vm[b], tr[b].cpu().numpy(), fvi, aw)
        _, sn = mocap_ref.frame_geometry(vs[b], tl[b].cpu().numpy(), fvi, aw)
        out.append(np.minimum((mocap_ref.dots(-sn, mn) <= mocap_ref.AGAINST).sum(1), 4))
    return np.stack(out)


def test_update_scene_against_golden(scene, gold):
    recs = gold['scene']
    for fresh in (True, False):
        sel = [r for r in recs if (r['prev'] is None) == fresh]
        f32 = lambda k: torch.from_numpy(np.stack([np.asarray(r[k], np.float32) for r in sel])).cuda()
        args = [f32('hand_pose'), f32('obj_pose'), f32('hand_tsl'), f32('obj_tsl'), f32('hand_shape')]
        prev = None if fresh else torch.from_numpy(np.stack([r['prev'] for r in sel]).astype(np.int64)).cuda()
        out = scene.update_scene(*args, anchor_id=prev)
        for k in ('vertex_contact', 'anchor_padding_mask'):
            assert np.array_equal(out[k].cpu().numpy(), np.stack([r[k] for r in sel]).astype(np.int64)), (fresh, k)
        err = float(np.abs(out['anchor_elasti'].cpu().numpy() - np.stack([r['anchor_elasti'] for r in sel])).max())
        assert err <= 1e-6, (fresh, err)
        ids, ref = out['anchor_id'].cpu().numpy(), np.stack([r['anchor_id'] for r in sel]).astype(np.int64)
        if fresh:
            keep = np.arange(4)[None, None, :] < _n_cand(scene, args)[..., None]
            assert (~keep).any()
            assert np.array_equal(ids[keep], ref[keep])
        else:
            assert np.array_equal(ids, ref)
        assert np.array_equal(out['optimize_it'].cpu().numpy()[:, 0], np.stack([r['vertex_contact'].any() for r in sel]))


class _Recorder:
    """A stand-in optimiser: records set_opt_val's arguments and returns its inputs unchanged, as the golden generator's does."""

    def __init__(self, lambda_contact_loss, lambda_repulsion_loss):
        self.coef_val = {'lambda_contact_loss': lambda_contact_loss, 'lambda_repulsion_loss': lambda_repulsion_loss}
        self.n_iter = 100
        self.calls = []

    def set_opt_val(self, **kw):
        self.calls.append(dict(kw, coef_val=dict(self.coef_val), n_iter=self.n_iter))

    def optimize(self, progress=False):
        kw = self.calls[-1]
        pose = lambda g, i: torch.cat([kw[g][1], kw[i][1]], 1).cpu()
        return {'optimized_hand_pose': pose('hand_pose_gt', 'hand_pose_init'), 'optimized_hand_tsl': kw['hand_tsl_init'].cpu(),
                'optimized_sub_hand_pose': pose('obj_pose_gt', 'obj_pose_init'), 'optimized_sub_hand_tsl': kw['obj_tsl_init'].cpu()}


def test_driver_against_golden(scene, gold):
    rec = _Recorder(gold['lambda_contact_loss'], 0.0)
    saved = MO.optimize_mocap(gold['raw'], rec, scene, gold['batch_size'], gold['optimize_interval'], 1.0)
    assert len(rec.calls) == len(gold['calls'])
    frames = gold['n_frames']
    for c, g in zip(rec.calls, gold['calls']):
        assert c['batch_size'] == g['batch_size'] and c['n_iter'] == g['n_iter'] and c['coef_val'] == {
            k: g['coef_val'][k] for k in c['coef_val']}
        gk = g['kwargs']
        for k in ('vertex_contact', 'anchor_padding_mask'):
            assert torch.equal(c[k].cpu(), gk[k].long()), k
        assert c['optimize_it'].shape == (c['batch_size'], 1) and torch.equal(c['optimize_it'].cpu(), gk['optimize_it'])
        assert float((c['anchor_elasti'].cpu() - gk['anchor_elasti']).abs().max()) <= 1e-6
        # the converter matrices come from the CUDA hand model here, from the CPU one in the reference: the quaternions differ in the last bits
        assert float((c['hand_pose_gt'][1].cpu() - gk['hand_pose'][:, :1]).abs().max()) <= 1e-6
        assert float((c['obj_pose_init'][1].cpu() - gk['obj_pose'][:, 1:]).abs().max()) <= 1e-6
        assert torch.equal(c['hand_shape_init'].cpu(), gk['hand_shape_init'])
        assert torch.equal(c['consistent_mask'][0].cpu(), torch.zeros(c['batch_size'], 16))
    for side in ('right', 'left'):
        np.testing.assert_allclose(saved[side]['rot'], gold['saved'][side]['rot'], rtol=0, atol=1e-4)
        np.testing.assert_allclose(saved[side]['loc'], gold['saved'][side]['loc'], rtol=0, atol=1e-6)
        assert saved[side]['shape'].dtype == np.float32 and np.array_equal(saved[side]['shape'], gold['saved'][side]['shape'])
        assert saved[side]['rot'].shape == (frames, 16, 3)


def _recording(opt):
    calls = []
    orig = opt.set_opt_val

    def set_opt_val(**kw):
        calls.append({'batch_size': kw['batch_size'], 'coef_val': dict(opt.coef_val), 'n_iter': opt.n_iter,
                      **{k: kw[k].detach().cpu().clone() for k in ('anchor_id', 'anchor_elasti', 'anchor_padding_mask', 'vertex_contact',
                                                                  'optimize_it', 'hand_tsl_init', 'obj_tsl_init')}})
        return orig(**kw)
    opt.set_opt_val = set_opt_val
    return calls


def test_driver_against_eager_driver(scene):
    raw = mocap_ref.synthetic_mocap(11, 7)
    weights = (1007, 1.0, (G.THRESH + 3.0, 0.0))
    opts = [G.build(weights, lambda_repulsion_loss=0.5) for _ in range(2)]
    calls = [_recording(o) for o in opts]
    ours = MO.optimize_mocap(raw, opts[0], scene, 4, 1, 1.0)
    ref = mocap_ref.eager_optimize_mocap(raw, opts[1], scene, 4, 1, 1.0)
    assert len(calls[0]) == len(calls[1]) == 12
    assert any(bool(c['optimize_it'].any()) for c in calls[0])
    for a, b in zip(*calls):
        assert a['batch_size'] == b['batch_size'] and a['coef_val'] == b['coef_val'] and a['n_iter'] == b['n_iter']
        for k in ('anchor_id', 'anchor_padding_mask', 'vertex_contact', 'optimize_it', 'anchor_elasti'):
            assert a[k].dtype == b[k].dtype and torch.equal(a[k], b[k]), k
        for k in ('hand_tsl_init', 'obj_tsl_init'):
            assert float((a[k] - b[k]).abs().max()) <= 1e-6, k
    for side in ('right', 'left'):
        np.testing.assert_allclose(ours[side]['rot'], ref[side]['rot'], rtol=0, atol=1e-3)
        np.testing.assert_allclose(ours[side]['loc'], ref[side]['loc'], rtol=0, atol=1e-4)
        assert np.array_equal(ours[side]['shape'], ref[side]['shape'])


def test_rejected_inputs(scene):
    args = _inputs(3, 5)
    with pytest.raises(RuntimeError):
        scene.update_scene(args[0].cpu(), *args[1:])
    with pytest.raises(TypeError):
        scene.update_scene(args[0].double(), *args[1:])
    with pytest.raises(TypeError):
        scene.update_scene(*args[:4], args[4].half())
    with pytest.raises(ValueError):
        scene.update_scene(args[0][:, :15], *args[1:])
    with pytest.raises(ValueError):
        scene.update_scene(*args[:2], args[2][:2], *args[3:])
    ids = torch.zeros(3, 108, 4, dtype=torch.int64, device='cuda')
    with pytest.raises(ValueError):
        scene.update_scene(*args, anchor_id=ids[:, :, :3])
    for bad in (-1, 108):
        wrong = ids.clone()
        wrong[1, 5, 2] = bad
        with pytest.raises(ValueError):
            scene.update_scene(*args, anchor_id=wrong)
    with pytest.raises(RuntimeError):
        scene.update_scene(*args, anchor_id=ids.cpu())
    with pytest.raises(NotImplementedError):
        MO.run_sample('cuda', None, {'batch_size': 1}, vis=True)
    with pytest.raises(NotImplementedError):
        MO.main(types.SimpleNamespace(vis=True))
