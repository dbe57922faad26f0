"""Generate tests/golden/manopth_synth.pt by running the UNMODIFIED quaternion hand model of the pose optimiser
(pose_data_optimize/manopth/manopth/manolayer.py, imported in place from /root/reference) on the synthetic MANO tensors.

Run in the authoring container only:   python -m oracle.make_golden_manopth
Only the MANO loader is substituted: the layer's `ready_arguments` (mano/webuser/smpl_handpca_wrapper_HAND_only.py:22-67) needs chumpy.
The stand-in reads the same pickle, fills zero `betas` when they are absent as ready_arguments does (:38-43) and exposes each array
through `.r` like a chumpy array.  Nothing derived from the licence-restricted MANO files is written.
"""
import os
import pickle
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from renderih_b200 import assets as rih_assets  # noqa: E402  (asset *generator* only: no kernels involved)

GOLD = os.path.join(ROOT, 'tests', 'golden')
REF_MANOPTH = os.path.join(os.environ.get('RIH_REFERENCE_ROOT', '/root/reference'), 'pose_data_optimize', 'manopth')
B = 5
SEED = 4321
# Stored vertices: every 32nd, the finger tips of both sides and the palm pair.  The gradients are stored in full; they depend on every
# vertex through the weighted sum, so the file stays small without leaving any vertex unchecked.
VERT_IDX = sorted(set(range(0, 778, 32)) | {745, 317, 444, 445, 556, 673, 95, 22})


class _Arr(object):
    def __init__(self, a):
        self.r = np.asarray(a)


def plain_ready_arguments(fname_or_dict, posekey4vposed='pose'):
    """ready_arguments without chumpy: the loaded dict, zero betas filled in, arrays behind `.r`."""
    if isinstance(fname_or_dict, dict):
        dd = dict(fname_or_dict)
    else:
        with open(fname_or_dict, 'rb') as f:
            dd = pickle.load(f, encoding='latin1')
    if 'shapedirs' in dd and 'betas' not in dd:
        dd['betas'] = np.zeros(np.asarray(dd['shapedirs']).shape[-1])
    for k in ('v_template', 'weights', 'posedirs', 'shapedirs', 'betas'):
        dd[k] = _Arr(dd[k])
    return dd


def import_reference_layer():
    if REF_MANOPTH not in sys.path:
        sys.path.insert(0, REF_MANOPTH)
    import manopth.manolayer as ml
    ml.ready_arguments = plain_ready_arguments
    return ml.ManoLayer


def inputs():
    g = torch.Generator().manual_seed(SEED)
    q = torch.randn(B, 16, 4, generator=g) * 0.35
    q[..., 0] += 1.0
    q = q * (0.6 + 0.8 * torch.rand(B, 16, 1, generator=g))          # |q| != 1
    return {'quat': q.reshape(B, 64).contiguous(), 'betas': torch.randn(B, 10, generator=g), 'trans': torch.randn(B, 3, generator=g) * 0.1}


def loss_weights():
    """Weights wv [B,778,3], wj [B,21,3], wt [B,16,4,4] of the golden's weighted sum: a closed form, so they are not stored."""
    w = lambda shape, a: torch.sin(a * torch.arange(int(np.prod(shape)), dtype=torch.float64) + 0.3).float().reshape(shape)
    return {'wv': w((B, 778, 3), 0.731), 'wj': w((B, 21, 3), 1.37), 'wt': w((B, 16, 4, 4), 2.11)}


def load(path):
    """The golden file with its inputs completed by the loss weights and each case's transf [B,16,3,4] rebuilt: the rotation blocks depend
    only on the quaternions and the side, so they are stored once per side."""
    gold = torch.load(path, weights_only=False)
    gold['inputs'].update(loss_weights())
    for case in gold['cases']:
        case['transf'] = torch.cat([gold['transf_rot'][case['cfg']['side']], case.pop('transf_t')[..., None]], -1)
    return gold


def cases():
    out = []
    for side in ('right', 'left'):
        for center in (0, 9, None):
            for trans in ('none', 'zeros', 'nonzero'):
                out.append({'side': side, 'center_idx': center, 'trans': trans, 'betas': 'rows', 'root_palm': False, 'share_betas': False})
        out.append({'side': side, 'center_idx': 9, 'trans': 'none', 'betas': 'rows', 'root_palm': True, 'share_betas': False})
        out.append({'side': side, 'center_idx': 0, 'trans': 'nonzero', 'betas': 'rows', 'root_palm': False, 'share_betas': True})
        out.append({'side': side, 'center_idx': 0, 'trans': 'zeros', 'betas': 'none', 'root_palm': False, 'share_betas': False})
    return out


def main():
    ManoLayer = import_reference_layer()
    inp = inputs()
    w = loss_weights()
    gold = {'meta': {'source': 'pose_data_optimize/manopth/manopth/manolayer.py executed in place, ready_arguments replaced by a plain loader',
                     'torch': torch.__version__, 'batch': B, 'seed': SEED,
                     'stored': 'verts at vert_idx only; transf without its constant bottom row [0, 0, 0, 1], its rotation blocks once per side; '
                               'the loss weights are the closed form of loss_weights(); read it with load()'},
            'vert_idx': torch.tensor(VERT_IDX), 'inputs': inp, 'transf_rot': {}, 'cases': []}
    with tempfile.TemporaryDirectory() as tmp:
        for side in ('left', 'right'):
            with open(os.path.join(tmp, 'MANO_%s.pkl' % side.upper()), 'wb') as f:
                pickle.dump(rih_assets.synthetic_mano(0, side), f)
        for c in cases():
            layer = ManoLayer(center_idx=c['center_idx'], flat_hand_mean=True, side=c['side'], mano_root=tmp, use_pca=False,
                              root_rot_mode='quat', joint_rot_mode='quat', return_transf=True, return_full_pose=True)
            quat = inp['quat'].clone().requires_grad_(True)
            betas = inp['betas'].clone().requires_grad_(True) if c['betas'] == 'rows' else None
            trans = {'none': None, 'zeros': torch.zeros(B, 3), 'nonzero': inp['trans'].clone()}[c['trans']]
            if trans is not None:
                trans.requires_grad_(True)
            verts, joints, transf, full = layer(quat, betas, trans, root_palm=torch.Tensor([int(c['root_palm'])]),
                                                share_betas=torch.Tensor([int(c['share_betas'])]))
            assert full is quat
            ((verts * w['wv']).sum() + (joints * w['wj']).sum() + (transf * w['wt']).sum()).backward()
            grab = lambda t: None if t is None else t.grad.detach().clone()
            assert torch.equal(transf[:, :, 3], torch.tensor([0.0, 0, 0, 1]).expand(B, 16, 4))
            rot = transf.detach()[:, :, :3, :3].clone()
            assert torch.equal(gold['transf_rot'].setdefault(c['side'], rot), rot)
            gold['cases'].append({'cfg': c, 'verts': verts.detach()[:, VERT_IDX].clone(), 'joints': joints.detach().clone(),
                                  'transf_t': transf.detach()[:, :, :3, 3].clone(),
                                  'd_quat': grab(quat), 'd_betas': grab(betas), 'd_trans': grab(trans)})
    torch.save(gold, os.path.join(GOLD, 'manopth_synth.pt'))
    print('manopth golden: %d cases' % len(gold['cases']))


if __name__ == '__main__':
    main()
