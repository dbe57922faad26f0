"""Generate tests/golden/geo_loss_synth.pt by running the UNMODIFIED reference functions of the pose optimiser's prior and contact terms
(hocontact/postprocess/geo_loss.py HandLoss / FieldLoss, manopth/anchorutils.py recover_anchor_batch, manopth/quatutils.py,
scripts/HandPoseConverter.py; imported in place from /root/reference/pose_data_optimize) on the synthetic MANO tensors, in the order
GeOptimizer.loss_fn calls them (geo_optimizer_both_batch.py:567-612, 705-757).

Run in the authoring container only:   python -m oracle.make_golden_geo_loss
loss_fn itself cannot run: GeOptimizer.__init__ loads Ver2Code/Discriminator/discrim.pth and NewLoss code_sdf/right.npy, neither of which
is in the reference tree.  What is substituted to import the functions:
  * empty stand-ins for open3d, trimesh and termcolor (imported at module level, unused by these functions);
  * the numpy aliases np.int / np.long that numpy 2 removed (anchorutils.py:24,30, HandPoseConverter.py:47);
  * the chumpy-free MANO loader of make_golden_manopth for `ready_arguments` in manopth.manolayer and scripts.HandPoseConverter;
  * the two anchor tables read directly with np.loadtxt (anchor_load also opens anchor_mapping_path.pkl, absent from the tree).
The file stores the anchor tables (data of the reference tree), the edge list, the converter matrices, the four terms and the gradients
of the weighted total; the inputs are rebuilt from the seed by load().  Nothing derived from the licence-restricted MANO files is written.
"""
import os
import pickle
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import make_golden_manopth  # noqa: E402
from renderih_b200 import assets as rih_assets  # noqa: E402  (asset *generator* only: no kernels involved)

GOLD = os.path.join(ROOT, 'tests', 'golden')
REF_POSE = os.path.join(os.environ.get('RIH_REFERENCE_ROOT', '/root/reference'), 'pose_data_optimize')
B, D = 5, 4
SEED = 2718
WEIGHTS = (1.0, 1.0, 10.0, 1.0)     # quat-norm, edge, contact (lambda_contact_loss), ergonomics: the optimiser's total (:805-825)
N_DESIGNED = 3                      # samples whose joints are placed at chosen local bend / splank / twist angles


def _rot(axis, deg):
    c, s = np.cos(np.radians(deg)), np.sin(np.radians(deg))
    i, j = [(1, 2), (2, 0), (0, 1)][axis]
    R = np.eye(3)
    R[i, i], R[i, j], R[j, i], R[j, j] = c, -s, s, c
    return R


def _quat_of(R):
    """rotation matrix -> unit quaternion (w, x, y, z) with w >= 0 (Shepperd's method)."""
    t = np.trace(R)
    if t > 0:
        s = np.sqrt(t + 1.0) * 2
        q = [0.25 * s, (R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s]
    else:
        i = int(np.argmax(np.diag(R)))
        j, k = (i + 1) % 3, (i + 2) % 3
        s = np.sqrt(1.0 + R[i, i] - R[j, j] - R[k, k]) * 2
        q = np.zeros(4)
        q[0] = (R[k, j] - R[j, k]) / s
        q[1 + i], q[1 + j], q[1 + k] = 0.25 * s, (R[j, i] + R[i, j]) / s, (R[k, i] + R[i, k]) / s
    q = np.asarray(q)
    return q if q[0] >= 0 else -q


def inputs(converter):
    """Inputs of the golden cases from the seed and the stored converter matrices ({side: (invM_U_n_0, invU_M_n_1)} float32)."""
    g = torch.Generator().manual_seed(SEED)
    rng = np.random.default_rng(SEED)
    out = {}
    for side in ('right', 'left'):
        q = torch.randn(B, 16, 4, generator=g, dtype=torch.float64) * 0.35
        q[..., 0] += 1.0
        q = q.numpy()
        m0, u1 = (np.asarray(a, np.float64) for a in converter[side])
        for b in range(N_DESIGNED):
            for t in range(15):
                bend, splank, twist = rng.uniform(-45, 125), rng.uniform(-45, 45), rng.uniform(-45, 60)
                if b == 0 and t == 12:
                    bend, splank, twist = 10.0, 5.0, 50.0          # thumb twist above 0.5
                Mt = _rot(2, bend) @ _rot(1, -splank) @ _rot(0, twist)
                A, C = m0[t + 1].T, u1[t + 1].T
                P = (A @ C).T @ A
                R = np.linalg.solve(P, Mt) @ np.linalg.inv(C)
                qq = _quat_of(R)
                if side == 'left':
                    qq = qq * np.array([1.0, 1.0, -1.0, -1.0])
                q[b, t + 1] = qq
        scale = 0.6 + 0.8 * torch.rand(B, 16, 1, generator=g, dtype=torch.float64).numpy()
        out['quat_' + side[0]] = torch.from_numpy(q * scale).float()
        vt = torch.from_numpy(np.asarray(rih_assets.synthetic_mano(0, side)['v_template'])).float()
        shift = torch.tensor([0.02 if side == 'right' else -0.02, 0.0, 0.0]) + 0.01 * torch.randn(B, 1, 3, generator=g)
        out['verts_' + side[0]] = (vt[None] + 0.002 * torch.randn(B, 778, 3, generator=g) + shift).contiguous()
    out['anchor_id'] = torch.randint(0, 108, (B, 108, D), generator=g)
    out['elastic'] = torch.rand(B, 108, D, generator=g)
    out['mask'] = (torch.rand(B, 108, D, generator=g) < 0.4).long()
    return out


def load(path):
    """The golden file with each case's inputs rebuilt (the empty-mask case shares the first case's quaternion gradients)."""
    gold = torch.load(path, weights_only=False)
    base = inputs(gold['converter'])
    for case in gold['cases']:
        case['inputs'] = dict(base)
        if case['name'] == 'empty_mask':
            case['inputs']['mask'] = torch.zeros_like(base['mask'])
            case['d_quat_r'], case['d_quat_l'] = gold['cases'][0]['d_quat_r'], gold['cases'][0]['d_quat_l']
    return gold


def import_reference():
    for name in ('open3d', 'trimesh', 'termcolor'):
        sys.modules.setdefault(name, types.ModuleType(name))
    np.int, np.long = int, int
    for p in (REF_POSE, os.path.join(REF_POSE, 'manopth')):
        if p not in sys.path:
            sys.path.insert(0, p)
    import manopth.manolayer as ml
    ml.ready_arguments = make_golden_manopth.plain_ready_arguments
    import scripts.HandPoseConverter as hpc
    hpc.ready_arguments = make_golden_manopth.plain_ready_arguments
    from hocontact.postprocess.geo_loss import FieldLoss, HandLoss
    from manopth.anchorutils import recover_anchor_batch
    from manopth.quatutils import normalize_quaternion
    return ml.ManoLayer, hpc.HandPoseConverter, FieldLoss, HandLoss, recover_anchor_batch, normalize_quaternion


def main():
    ManoLayer, HandPoseConverter, FieldLoss, HandLoss, recover_anchor_batch, normalize_quaternion = import_reference()
    anchor_dir = os.path.join(REF_POSE, 'assets', 'anchor')
    fvi = np.loadtxt(os.path.join(anchor_dir, 'face_vertex_idx.txt'), dtype=np.int64)
    aw = torch.from_numpy(np.loadtxt(os.path.join(anchor_dir, 'anchor_weight.txt'))).float()       # AnchorLayer's float buffer
    ident = torch.from_numpy(np.asarray([[1.0, 0.0, 0.0, 0.0]] * 16, dtype=np.float32)).unsqueeze(0)
    with tempfile.TemporaryDirectory() as tmp:
        for side in ('left', 'right'):
            with open(os.path.join(tmp, 'MANO_%s.pkl' % side.upper()), 'wb') as f:
                pickle.dump(rih_assets.synthetic_mano(0, side), f)
        layers = {side: ManoLayer(joint_rot_mode='quat', root_rot_mode='quat', use_pca=False, mano_root=tmp, center_idx=0, flat_hand_mean=True,
                                  return_transf=True, return_full_pose=True, side=side) for side in ('right', 'left')}
        conv = {side: HandPoseConverter(side=side, root=tmp, data_type='tensor', device='cpu') for side in ('right', 'left')}
    zero = {side: conv[side].mano_quat_2_mat_tensor(ident).repeat(B, 1, 1, 1) for side in conv}        # :98-104, 167-169
    edges = HandLoss.get_edge_idx(layers['right'].th_faces)                                               # :222, and :229 for the left
    static = {}
    for side in ('right', 'left'):
        with torch.no_grad():
            v = layers[side](ident.reshape(1, -1), torch.zeros(1, 10))[0].squeeze(0)                    # :457-470
        static[side] = HandLoss.get_edge_len(v, edges)
    converter = {side: (conv[side].invM_U_n_0.clone(), conv[side].invU_M_n_1.clone()) for side in conv}
    gold = {'meta': {'source': 'hocontact/postprocess/geo_loss.py, manopth/anchorutils.py, manopth/quatutils.py, scripts/HandPoseConverter.py '
                               'executed in place in GeOptimizer.loss_fn order, on the synthetic MANO tensors',
                     'torch': torch.__version__, 'batch': B, 'seed': SEED, 'weights': WEIGHTS,
                     'stored': 'terms [quat_norm, edge, contact, ergonomics]; gradients of the weighted total; inputs rebuilt by load()'},
            'anchor_fvi': torch.from_numpy(fvi).short(), 'anchor_w': aw, 'edges': edges.short(), 'converter': converter, 'cases': []}
    base = inputs(converter)
    fvi_t = torch.from_numpy(fvi).long().unsqueeze(0)
    for name in ('contact', 'empty_mask'):
        inp = dict(base)
        if name == 'empty_mask':
            inp['mask'] = torch.zeros_like(base['mask'])
        q_r, q_l, v_r, v_l = (inp[k].clone().requires_grad_(True) for k in ('quat_r', 'quat_l', 'verts_r', 'verts_l'))
        # geo_optimizer_both_batch.py:567-612
        anchor = recover_anchor_batch(v_r, fvi_t, aw.unsqueeze(0)).contiguous()
        sub_anchor = recover_anchor_batch(v_l, fvi_t, aw.unsqueeze(0)).contiguous()
        indexed = anchor.unsqueeze(2).repeat(1, 1, D, 1).gather(1, inp['anchor_id'].unsqueeze(-1).repeat(1, 1, 1, 3))
        contact = FieldLoss.batch_contact_loss(indexed, sub_anchor.unsqueeze(2).repeat(1, 1, D, 1), inp['mask'], inp['elastic'])
        # :705-757
        qn = HandLoss.batch_pose_quat_norm_loss(q_r)
        ja = conv['right'].mano_quat_2_mat_tensor(normalize_quaternion(q_r))
        ergo = HandLoss.hand_pose_ergonomics_loss(ja[:, 1:, :, :], zero['right'][:, 1:, :, :], 'r')
        edge = HandLoss.edge_len_loss(v_r, edges, static['right'])
        qn = qn + HandLoss.batch_pose_quat_norm_loss(q_l)
        ja = conv['left'].mano_quat_2_mat_tensor(normalize_quaternion(q_l))
        ergo = ergo + HandLoss.hand_pose_ergonomics_loss(ja[:, 1:, :, :], zero['left'][:, 1:, :, :], 'l')
        edge = edge + HandLoss.edge_len_loss(v_l, edges, static['left'])
        terms = [qn, edge, contact, ergo]
        sum(w * t.reshape(()) for w, t in zip(WEIGHTS, terms)).backward()
        case = {'name': name, 'terms': torch.stack([t.detach().reshape(()) for t in terms]),
                'd_verts_r': v_r.grad.clone(), 'd_verts_l': v_l.grad.clone()}
        if name == 'contact':
            case['d_quat_r'], case['d_quat_l'] = q_r.grad.clone(), q_l.grad.clone()
        else:
            assert float(case['terms'][2]) == 0.0 and tuple(contact.shape) == (1,)
            assert torch.equal(q_r.grad, gold['cases'][0]['d_quat_r']) and torch.equal(q_l.grad, gold['cases'][0]['d_quat_l'])
        gold['cases'].append(case)
        print(name, ['%.6g' % float(t) for t in case['terms']])
    torch.save(gold, os.path.join(GOLD, 'geo_loss_synth.pt'))
    print('geo_loss golden: %d edges, %d cases' % (edges.shape[0], len(gold['cases'])))


if __name__ == '__main__':
    main()
