"""Generate tests/golden/ge_optimizer_synth.pt by running the UNMODIFIED two-hand pose optimiser loop: GeOptimizer.set_opt_val and
GeOptimizer.optimize of hocontact/postprocess/geo_optimizer_both_batch.py (:133-447, :861-930, with loss_fn :498-859), unbound, on an
instance built with object.__new__ on the CPU, imported in place from /root/reference/pose_data_optimize.

Run in the authoring container only:   python -m oracle.make_golden_ge_optimizer
What is substituted (GeOptimizer.__init__ is not run):
  * the stand-ins of make_golden_nature (open3d, trimesh, termcolor, sdf, the numpy aliases) and the chumpy-free MANO loader and
    synthetic MANO tensors of make_golden_manopth for both ManoLayers and both HandPoseConverters;
  * the AnchorLayer built from the two anchor tables read directly, as make_golden_geo_loss does (anchor_load also opens
    anchor_mapping_path.pkl, absent from the tree); AxisLayer() is the reference's own;
  * synthetic discriminator weights (oracle/nature_ref.init_state_dict, chosen by oracle/ge_optimizer_ref.nature_weights);
  * torch.optim.lr_scheduler.ReduceLROnPlateau accepts and drops the `verbose=False` argument (:431) that this torch no longer takes;
  * anti_penetration_loss_fun is a differentiable zero: the reference's NewLoss needs its CUDA extension and code_sdf/right.npy, which is
    absent.  The GPU tests run the penetration term's place in the loop against an eager loop of the same CUDA modules instead
    (tests/test_ge_optimizer_gpu.py); against this file they run with lambda_repulsion_loss = 0, which gives the same total.
The instance's NatureLoss is wrapped to record the normalised poses it sees, and the scheduler's step to record the loss and the lrs;
both then call the reference's own.  A case is kept only if no scheduler comparison lies within MARGIN (relative) of its threshold and no
nature row is flagged by oracle/nature_ref at any iteration; otherwise the next seed is tried.  The inputs are rebuilt from the seeds by
ge_optimizer_ref.inputs().  Stored per case: the total at every iteration, every group's lr after every scheduler step, the final out_dict.
"""
import os
import pickle
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ge_optimizer_ref as G  # noqa: E402
from oracle import make_golden_geo_loss, nature_ref  # noqa: E402
from renderih_b200 import assets as rih_assets  # noqa: E402  (asset *generator* only: no kernels involved)

GOLD = os.path.join(G.GOLD_DIR, 'ge_optimizer_synth.pt')
MARGIN = 2e-5
MIN_LR_SHAPE = 200.0
UNSORTED = ([7, 0, 12], [15, 3, 1, 9, 2, 4, 5, 6, 8, 10, 11, 13, 14])
UNSORTED_L = ([3, 9, 0, 14], [1, 2, 4, 15, 5, 6, 7, 8, 10, 11, 12, 13])
# name, B, lr, n_iter, split, nature rule, lambda_contact_loss, pose scale, first seed.  'min_lr': lr = 1e-3 puts the translation
# groups at min_lr, near-identity poses with large betas (MIN_LR_SHAPE) and no contact term.  No synthetic case made the reference's total
# stall for 21 iterations within its length, so the halving itself is checked against torch's scheduler (tests/test_ge_optimizer_*.py).
CASES = (('caller_split', 4, 1e-2, 40, (G.CALLER_SPLIT, G.CALLER_SPLIT), 'median', 10.0, 0.3, 100),
         ('unsorted_split', 3, 1e-2, 30, (UNSORTED, UNSORTED_L), 'median', 10.0, 0.3, 200),
         ('min_lr', 2, 1e-3, 40, (G.CALLER_SPLIT, G.CALLER_SPLIT), 'median', 0.0, 0.01, 300),
         ('one_empty', 3, 1e-2, 30, (G.CALLER_SPLIT, G.CALLER_SPLIT), 'one_empty', 10.0, 0.3, 400),
         ('batch_1', 1, 1e-2, 30, (G.CALLER_SPLIT, G.CALLER_SPLIT), 'median', 10.0, 0.3, 500))


def load(path=GOLD):
    """The golden file with each case's set_opt_val keyword arguments (CPU) and weights rebuilt from the stored seeds."""
    gold = torch.load(path, weights_only=False)
    for case in gold['cases']:
        case['kwargs'] = G.inputs(case['batch'], case['seed'], case['split'], scale=case['pose_scale'], shape_scale=case['shape_scale'])
    return gold


def reference_instance(GeOptimizer, layers, conv, AxisLayer, anchor, disc, lr, n_iter, lambda_contact):
    """What GeOptimizer.__init__ (:23-108) sets, from the substitutes, on the CPU."""
    self = object.__new__(GeOptimizer)
    self.mode, self.device, self.lr, self.n_iter = 'both', 'cpu', lr, n_iter
    self.anti_penetration_loss_fun = lambda verts: (verts * 0.0).sum(dim=(1, 2, 3))
    self.verbose, self.runtime_vis, self.compensate_tsl = False, None, False
    self.mano_layer, self.sub_mano_layer = layers['right'], layers['left']
    self.anchor_layer, self.axis_layer = anchor, AxisLayer()
    self.opt_val, self.const_val, self.ctrl_val = {}, {}, {}
    self.coef_val = {'lambda_contact_loss': lambda_contact, 'lambda_repulsion_loss': 0.5, 'repulsion_query': 0.030, 'repulsion_threshold': 0.080}
    self.optimizer, self.optimizing, self.scheduler = None, True, None
    self.rhpc, self.lhpc = conv['right'], conv['left']
    ident = torch.from_numpy(np.asarray([[1.0, 0.0, 0.0, 0.0]] * 16, dtype=np.float32)).unsqueeze(0)
    self.zero_mat_ = self.rhpc.mano_quat_2_mat_tensor(ident)
    self.sub_zero_mat_ = self.lhpc.mano_quat_2_mat_tensor(ident)
    self.disc = disc
    return self


class _Plateau(torch.optim.lr_scheduler.ReduceLROnPlateau):
    def __init__(self, *args, verbose=False, **kwargs):
        super().__init__(*args, **kwargs)


def main():
    from oracle import make_golden_nature
    torch.optim.lr_scheduler.ReduceLROnPlateau = _Plateau
    Pos2dDiscriminator, _ = make_golden_nature.import_reference()
    from hocontact.postprocess.geo_optimizer_both_batch import GeOptimizer
    import manopth.manolayer as ml
    import scripts.HandPoseConverter as hpc
    from manopth.axislayer import AxisLayer
    from manopth.anchorlayer import AnchorLayer
    anchor_dir = os.path.join(make_golden_geo_loss.REF_POSE, 'assets', 'anchor')
    fvi = np.loadtxt(os.path.join(anchor_dir, 'face_vertex_idx.txt'), dtype=np.int64)
    aw = np.loadtxt(os.path.join(anchor_dir, 'anchor_weight.txt'))
    anchor = object.__new__(AnchorLayer)
    torch.nn.Module.__init__(anchor)
    anchor.register_buffer('face_vert_idx', torch.from_numpy(fvi).long().unsqueeze(0))
    anchor.register_buffer('anchor_weight', torch.from_numpy(aw).float().unsqueeze(0))
    with tempfile.TemporaryDirectory() as tmp:
        for side in ('left', 'right'):
            with open(os.path.join(tmp, 'MANO_%s.pkl' % side.upper()), 'wb') as f:
                pickle.dump(rih_assets.synthetic_mano(0, side), f)
        layers = {s: ml.ManoLayer(joint_rot_mode='quat', root_rot_mode='quat', use_pca=False, mano_root=tmp, center_idx=0, flat_hand_mean=True,
                                  return_transf=True, return_full_pose=True, side=s) for s in ('right', 'left')}
        conv = {s: hpc.HandPoseConverter(side=s, root=tmp, data_type='tensor', device='cpu') for s in ('right', 'left')}
    gold = {'meta': {'source': 'GeOptimizer.set_opt_val / optimize (hocontact/postprocess/geo_optimizer_both_batch.py:133-930) executed '
                               'unbound in place on CPU, penetration term replaced by a differentiable zero',
                     'torch': torch.__version__, 'margin': MARGIN,
                     'stored': 'loss [n_iter], lr [n_iter,4] (after each scheduler step), out_dict; kwargs rebuilt by load()'},
            'cases': []}
    for name, B, lr, n_iter, split, rule, lc, pscale, seed0 in CASES:
        for seed in range(seed0, seed0 + 40):
            weights = G.nature_weights(B, seed, 1000 + seed, 40.0, rule, pscale)
            sd = nature_ref.init_state_dict(*weights)
            disc = Pos2dDiscriminator(num_joints=15, hid_dim=512, dropout=0.05).eval()
            disc.load_state_dict(sd, strict=True)
            opt = reference_instance(GeOptimizer, layers, conv, AxisLayer, anchor, disc, lr, n_iter, lc)
            seen, steps = [], []

            def nature(right, left, _opt=opt):
                seen.append((right.detach().clone(), left.detach().clone()))
                return GeOptimizer.NatureLoss(_opt, right, left)
            opt.NatureLoss = nature
            sscale = MIN_LR_SHAPE if name == 'min_lr' else 0.5
            kw = G.inputs(B, seed, split, scale=pscale, shape_scale=sscale)
            GeOptimizer.set_opt_val(opt, **kw)
            step = opt.scheduler.step

            def recorded(loss, _opt=opt, _step=step):
                best = _opt.scheduler.best
                _step(loss)
                steps.append((float(loss), best, [g['lr'] for g in _opt.optimizer.param_groups]))
            opt.scheduler.step = recorded
            out = GeOptimizer.optimize(opt)
            near = [i for i, (a, best, _) in enumerate(steps) if np.isfinite(best) and abs(a - best * (1 - 1e-4)) <= MARGIN * abs(best)]
            flagged = []
            masks = []
            for i, (r, l) in enumerate(seen):
                pad = lambda q: torch.cat([torch.ones(q.shape[0], 1, 4), q], 1)
                _, _, _, info = nature_ref.weighted_case(sd, pad(r), pad(l))
                masks.append(info['mask'].sum(1).tolist())
                if nature_ref.row_flags(info).any():
                    flagged.append(i)
            lrs = torch.tensor([s[2] for s in steps], dtype=torch.float64)
            ok = not near and not flagged
            if name == 'min_lr':
                ok = ok and bool((lrs[:, :2] == 1e-5).all())
            if name == 'one_empty':
                ok = ok and min(masks[0]) == 0 and max(masks[0]) > 0        # one hand's mask empty, the other's not, at the start
            if name != 'one_empty':
                ok = ok and any(min(m) > 0 for m in masks)
            if ok:
                print()
            print('%-15s seed %d: near %s flagged %s masks %s..%s lr %s' % (name, seed, near[:5], flagged[:5], masks[0], masks[-1],
                                                                          lrs[-1].tolist()))
            if ok:
                break
        else:
            raise RuntimeError('no usable seed for case %s' % name)
        gold['cases'].append({'name': name, 'batch': B, 'seed': seed, 'split': split, 'lr': lr, 'n_iter': n_iter, 'weights': weights,
                              'lambda_contact_loss': lc, 'pose_scale': pscale, 'shape_scale': sscale, 'loss': torch.tensor([s[0] for s in steps], dtype=torch.float32), 'lrs': lrs,
                              'out': {k: v.clone() for k, v in out.items()}})
    torch.save(gold, GOLD)
    print('ge_optimizer golden: %d cases, %d bytes' % (len(gold['cases']), os.path.getsize(GOLD)))


if __name__ == '__main__':
    main()
