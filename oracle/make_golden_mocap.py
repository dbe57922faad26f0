"""Generate tests/golden/mocap_synth.pt by running the UNMODIFIED mocap driver of the pose optimiser: main, update_scene, search_anchors and
run_sample of pose_data_optimize/batch_optimize_mocap_origin.py, imported in place from /root/reference/pose_data_optimize, on the CPU
(run_sample is handed 'cpu' for main's cuda:<gpu>).

Run in the authoring container only:   python -m oracle.make_golden_mocap
What is substituted:
  * the stand-ins of make_golden_ge_optimizer: the chumpy-free synthetic MANO (both ManoLayers main builds and both HandPoseConverters),
    GeOptimizer built with object.__new__ (reference_instance) with lambda_repulsion_loss = 0 and its penetration term a differentiable
    zero, synthetic discriminator weights;
  * hoptim.optimize() returns its inputs unchanged (GeOptimizer.optimize itself is covered by tests/golden/ge_optimizer_synth.pt), so
    every pass of main sees the converted mocap poses;
  * anchor_load_driver returns the three anchor tables read directly (the reference's also opens anchor_mapping_path.pkl, absent from the
    tree);
  * empty modules for open3d, trimesh (load() returns an object with empty faces, which run_sample reads for its viewer only), matplotlib,
    tqdm (tqdm() returns its argument) and chumpy.
The mocap dict is oracle/mocap_ref.synthetic_mocap(N_FRAMES, seed) at BATCH = 4, so the last batch is partial.  A seed is kept only if
every search_anchors call keeps its distances and its 4th / 5th candidates MARGIN_D (metres) and its normal dot products MARGIN_DOT away
from a decision, if some fresh-branch frames are in contact and some are not, and if some sub anchor has fewer than 4 unmasked candidates.
Stored: every update_scene call's inputs and outputs (ids, masks, contacts, elasticities: no vertices, anchors or normals), every
set_opt_val call's coef_val, n_iter and inputs, the quaternions euler_2_mano_quat made, and the saved dict.
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
from oracle import ge_optimizer_ref as G  # noqa: E402
from oracle import make_golden_ge_optimizer as MG  # noqa: E402
from oracle import make_golden_geo_loss, mocap_ref, nature_ref  # noqa: E402
from renderih_b200 import assets as rih_assets  # noqa: E402  (asset *generator* only: no kernels involved)

GOLD = os.path.join(G.GOLD_DIR, 'mocap_synth.pt')
N_FRAMES, BATCH, INTERVAL = 10, 4, 1
MARGIN_D, MARGIN_DOT = 1e-6, 2e-6
LAMBDA_CONTACT = 10.0


def import_reference():
    from oracle import make_golden_nature
    torch.optim.lr_scheduler.ReduceLROnPlateau = MG._Plateau
    make_golden_nature.import_reference()
    tq = types.ModuleType('tqdm')
    tq.tqdm = lambda it, *a, **k: it
    tq.__all__ = ['tqdm']
    ch = types.ModuleType('chumpy')
    ch.optimization_internal = None
    mpl, plt = types.ModuleType('matplotlib'), types.ModuleType('matplotlib.pyplot')
    plt.switch_backend = lambda *a: None
    mpl.pyplot = plt
    for name, mod in (('tqdm', tq), ('chumpy', ch), ('matplotlib', mpl), ('matplotlib.pyplot', plt)):
        sys.modules.setdefault(name, mod)
    sys.modules['trimesh'].load = lambda *a, **k: types.SimpleNamespace(faces=np.zeros((0, 3), np.int64))
    import batch_optimize_mocap_origin as R
    return R


def anchor_tables():
    d = os.path.join(make_golden_geo_loss.REF_POSE, 'assets', 'anchor')
    return (np.loadtxt(os.path.join(d, 'face_vertex_idx.txt'), dtype=np.int64), np.loadtxt(os.path.join(d, 'anchor_weight.txt')),
            np.loadtxt(os.path.join(d, 'merged_vertex_assignment.txt'), dtype=np.int64))


def nature_weights(seed):
    """Discriminator weights (seed, scale 1, bias) that mask every row of the mocap's initial poses by 3 logits."""
    return seed, 1.0, (G.THRESH + 3.0, 0.0)


def run(R, tmp, seed):
    from hocontact.postprocess.geo_optimizer_both_batch import GeOptimizer
    import manopth.manolayer as ml
    import scripts.HandPoseConverter as hpc
    from manopth.axislayer import AxisLayer
    from manopth.anchorlayer import AnchorLayer
    fvi, aw, cls = anchor_tables()
    anchor = object.__new__(AnchorLayer)
    torch.nn.Module.__init__(anchor)
    anchor.register_buffer('face_vert_idx', torch.from_numpy(fvi).long().unsqueeze(0))
    anchor.register_buffer('anchor_weight', torch.from_numpy(aw).float().unsqueeze(0))
    R.anchor_load_driver = lambda path: (fvi, aw, cls, None)
    R.manolayer = types.SimpleNamespace(ManoLayer=lambda **kw: ml.ManoLayer(**dict(kw, mano_root=tmp)))
    loss_layers = {s: ml.ManoLayer(joint_rot_mode='quat', root_rot_mode='quat', use_pca=False, mano_root=tmp, center_idx=0, flat_hand_mean=True,
                                   return_transf=True, return_full_pose=True, side=s) for s in ('right', 'left')}
    conv = {s: hpc.HandPoseConverter(side=s, root=tmp, data_type='tensor', device='cpu') for s in ('right', 'left')}
    Pos2dDiscriminator = sys.modules['Ver2Code.Discriminator.discrim'].Pos2dDiscriminator
    weights = nature_weights(1000 + seed)
    disc = Pos2dDiscriminator(num_joints=15, hid_dim=512, dropout=0.05).eval()
    disc.load_state_dict(nature_ref.init_state_dict(*weights), strict=True)
    rec = {'scene': [], 'calls': []}

    def make_optimizer(device, lr=1e-2, n_iter=100, lambda_contact_loss=10.0, lambda_repulsion_loss=0.5, repulsion_query=0.03,
                       repulsion_threshold=0.08, **kw):
        opt = MG.reference_instance(GeOptimizer, loss_layers, conv, AxisLayer, anchor, disc, lr, n_iter, lambda_contact_loss)
        opt.coef_val.update(lambda_repulsion_loss=lambda_repulsion_loss, repulsion_query=repulsion_query,
                            repulsion_threshold=repulsion_threshold)

        def set_opt_val(**kw):
            keep = {k: kw[k] for k in ('vertex_contact', 'anchor_id', 'anchor_elasti', 'anchor_padding_mask', 'hand_shape_init',
                                       'hand_tsl_init', 'obj_tsl_init', 'optimize_it')}
            keep['hand_pose'] = torch.cat([kw['hand_pose_gt'][1], kw['hand_pose_init'][1]], 1)
            keep['obj_pose'] = torch.cat([kw['obj_pose_gt'][1], kw['obj_pose_init'][1]], 1)
            rec['calls'].append({'batch_size': kw['batch_size'], 'coef_val': dict(opt.coef_val), 'n_iter': opt.n_iter,
                                 'kwargs': {k: v.clone() for k, v in keep.items()}})
            return GeOptimizer.set_opt_val(opt, **kw)

        def optimize(progress=False):          # the inputs unchanged: the optimiser has its own golden file
            kw = rec['calls'][-1]['kwargs']
            return {'optimized_hand_pose': kw['hand_pose'].clone(), 'optimized_hand_tsl': kw['hand_tsl_init'].clone(),
                    'optimized_sub_hand_pose': kw['obj_pose'].clone(), 'optimized_sub_hand_tsl': kw['obj_tsl_init'].clone()}
        opt.set_opt_val, opt.optimize = set_opt_val, optimize
        return opt
    R.GeOptimizer = make_optimizer

    update_scene, search_anchors = R.update_scene, R.search_anchors

    def rec_update(**kw):
        rec['scene'].append({'hand_pose': np.array(kw['optimized_hand_pose']), 'obj_pose': np.array(kw['optimized_sub_hand_pose']),
                             'hand_tsl': np.array(kw['optimized_hand_tsl']), 'obj_tsl': np.array(kw['optimized_sub_hand_tsl']),
                             'hand_shape': kw['hand_shape'][0].numpy().copy(),
                             'prev': None if kw['anchor_id'] is None else np.array(kw['anchor_id'])})
        return update_scene(**kw)

    def rec_search(main_anchors, sub_anchors, main_normals, sub_normals, class_types=None, prev_anchor_id=None, **kw):
        res = search_anchors(main_anchors, sub_anchors, main_normals, sub_normals, class_types, prev_anchor_id, **kw)
        ours = mocap_ref.search_anchors(main_anchors, sub_anchors, main_normals, sub_normals, class_types, prev_anchor_id)
        against = sub_normals.dot(main_normals.transpose()) <= -0.6
        r = rec['scene'][-1]
        r.update(vertex_contact=res[0].copy(), anchor_id=res[1].copy(), anchor_elasti=res[2].copy(), anchor_padding_mask=res[3].copy(),
                 margin=ours[4], margin_dot=ours[5], min_candidates=int(against.sum(1).min()), oracle_ids_equal=bool((ours[1] == res[1]).all()))
        return res
    R.update_scene, R.search_anchors = rec_update, rec_search
    run_sample = R.run_sample
    R.run_sample = lambda device, *a, **k: run_sample('cpu', *a, **k)          # main names cuda:<gpu>; everything runs on the CPU

    raw = mocap_ref.synthetic_mocap(N_FRAMES, seed)
    src = os.path.join(tmp, 'mocap.npy')
    dst = os.path.join(tmp, 'optimized.npy')
    np.save(src, {s: dict(v) for s, v in raw.items()})
    args = types.SimpleNamespace(gpu='0', center_idx=0, mano_root=tmp, anchor_root=tmp, manual_seed=0, hand_closed_path='unused',
                                 lambda_contact_loss=LAMBDA_CONTACT, lambda_repulsion_loss=0.0, repulsion_query=0.009, repulsion_threshold=0.05,
                                 mocap_scale=1.0, mocap_path=src, optimized_mocap_path=dst, fps=30, optimize_interval=INTERVAL, vis=False,
                                 reoptimize_raw='', batch_size=BATCH)
    R.main(args)
    saved = np.load(dst, allow_pickle=True).item()
    quat = {s: conv_np(hpc, tmp, s).euler_2_mano_quat(raw[s]['rot'][::INTERVAL]) for s in ('right', 'left')}
    R.update_scene, R.search_anchors, R.run_sample = update_scene, search_anchors, run_sample
    return raw, rec, saved, quat, weights


def conv_np(hpc, tmp, side):
    return hpc.HandPoseConverter(side=side, root=tmp)


def main():
    R = import_reference()
    import scripts.HandPoseConverter as hpc
    with tempfile.TemporaryDirectory() as tmp:
        for side in ('left', 'right'):
            with open(os.path.join(tmp, 'MANO_%s.pkl' % side.upper()), 'wb') as f:
                pickle.dump(rih_assets.synthetic_mano(0, side), f)
        conv = {s: tuple(np.asarray(getattr(conv_np(hpc, tmp, s), k)) for k in ('invM_U_n_0', 'invU_M_n_1')) for s in ('right', 'left')}
        for seed in range(100, 120):
            raw, rec, saved, quat, weights = run(R, tmp, seed)
            sc = rec['scene']
            fresh = [r for r in sc if r['prev'] is None]
            m_d = min(r['margin'] for r in sc)
            m_dot = min(r['margin_dot'] for r in fresh)
            contact = [bool(r['vertex_contact'].any()) for r in fresh]
            few = min(r['min_candidates'] for r in fresh)
            ok = m_d > MARGIN_D and m_dot > MARGIN_DOT and any(contact) and not all(contact) and few < 4
            ok = ok and all(r['oracle_ids_equal'] for r in sc)
            print('seed %d: margin_d %.2e margin_dot %.2e contact %s min candidates %d oracle ids equal %s -> %s' % (
                seed, m_d, m_dot, contact, few, all(r['oracle_ids_equal'] for r in sc), ok))
            if ok:
                break
        else:
            raise RuntimeError('no usable seed')
    for r in sc:                                    # stored compactly: ids < 256, masks and contacts as bool
        del r['oracle_ids_equal']
        r['anchor_id'] = r['anchor_id'].astype(np.uint8)
        r['prev'] = None if r['prev'] is None else r['prev'].astype(np.uint8)
        r['vertex_contact'], r['anchor_padding_mask'] = r['vertex_contact'] > 0, r['anchor_padding_mask'] > 0
    for c in rec['calls']:
        kw = c['kwargs']
        kw['anchor_id'] = kw['anchor_id'].to(torch.uint8)
        for k in ('vertex_contact', 'anchor_padding_mask'):
            kw[k] = kw[k] > 0
    gold = {'meta': {'source': 'main / update_scene / search_anchors / run_sample of pose_data_optimize/batch_optimize_mocap_origin.py '
                               'executed unmodified in place on CPU with the synthetic MANO tensors',
                     'torch': torch.__version__, 'numpy': np.__version__, 'margin_d': MARGIN_D, 'margin_dot': MARGIN_DOT},
            'seed': seed, 'n_frames': N_FRAMES, 'batch_size': BATCH, 'optimize_interval': INTERVAL, 'lambda_contact_loss': LAMBDA_CONTACT,
            'nature_weights': weights, 'anchor_tables': [torch.from_numpy(t) for t in anchor_tables()], 'converter': conv,
            'raw': raw, 'quat': quat, 'scene': sc, 'calls': rec['calls'], 'saved': saved}
    torch.save(gold, GOLD)
    print('mocap golden: %d update_scene calls, %d set_opt_val calls, %d bytes' % (len(sc), len(rec['calls']), os.path.getsize(GOLD)))


if __name__ == '__main__':
    main()
