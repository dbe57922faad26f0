"""Generate tests/golden/pose_data_synth.pt by running the UNMODIFIED conversion and augmentation stages of the pose data pipeline,
imported in place from /root/reference/pose_data_optimize, on the CPU with synthetic MANO:
  * HandPoseConverter's four conversions for both hands, on random poses;
  * HandPoseArguer and PoseArguer (random_level 0.7) argue_pose on random euler poses, under a fixed np.random.seed;
  * data/template_0_pose_convert.py, template_1_pose_argue.py and template_3_pose_reconvert.py via runpy, in order, in a scratch
    directory holding data/template_renderih_data_sample.pkl (a synthetic RenderIH annotation) and assets/mano; template 3 reads
    template 1's first splice, in the optimiser's output layout, as its optimised data, so its capture ids repeat and its save_id bump is exercised;
  * Ver2Code/NatureJudge/data_birth.py's loop, restated here because the script opens an absolute path on import, with the reference's
    PoseArguer and HandPoseConverter, on the first BIRTH_FRAMES converted frames.

Run in the authoring container only:   python -m oracle.make_golden_pose_data
What is substituted: the stand-ins of make_golden_geo_loss.import_reference (numpy 2's removed np.long, the chumpy-free MANO loader, an
empty open3d), a pycocotools stub for PoseArgue.py's unused COCO import and a sys.modules['HandPoseConverter'] alias for its top-level
import.  A seed is kept when every euler angle any stage computes lies EULER_MARGIN degrees from as_euler's branch points (second angle
+-90, first and third +-180) and every matrix given to from_matrix has its two largest branch values BRANCH_MARGIN apart, so that the
GPU's float64 rounding cannot take another branch.
"""
import copy
import glob
import os
import pickle
import runpy
import sys
import tempfile
import types

import numpy as np
import scipy
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import make_golden_geo_loss, pose_data_ref  # noqa: E402
from renderih_b200 import assets as rih_assets  # noqa: E402  (asset *generator* only: no kernels involved)

REF_POSE = make_golden_geo_loss.REF_POSE
GOLD = os.path.join(ROOT, 'tests', 'golden', 'pose_data_synth.pt')
N_CONV, N_ARGUE, A_ARGUE, LEVEL = 4, 3, 4, 0.7
BIRTH_FRAMES, BIRTH_A, BIRTH_SPLICE = 2, 2, 50
KEEP_FILES = 10            # template 3's files stored whole (all names are stored)
EULER_MARGIN, BRANCH_MARGIN = 1e-4, 1e-6


def import_reference():
    sys.modules.setdefault('pycocotools', types.ModuleType('pycocotools'))
    coco = types.ModuleType('pycocotools.coco')
    coco.COCO = object
    sys.modules['pycocotools.coco'] = coco
    make_golden_geo_loss.import_reference()
    import scripts.HandPoseConverter as hpc
    sys.modules['HandPoseConverter'] = hpc
    import scripts.HandPoseArguer as hpa
    sys.path.insert(0, os.path.join(REF_POSE, 'Ver2Code', 'NatureJudge'))
    import PoseArgue
    return hpc.HandPoseConverter, hpa.HandPoseArguer, PoseArgue.PoseArguer


def annotation(rng):
    """A RenderIH annotation's mano_params: per hand oripose [48] axis-angle, trans [1,3], shape [1,10], float32."""
    mp = {}
    for side in ('right', 'left'):
        mp[side] = {'oripose': (rng.normal(size=48) * 0.4).astype(np.float32), 'trans': (rng.normal(size=(1, 3)) * 0.1).astype(np.float32),
                    'shape': (rng.normal(size=(1, 10)) * 0.5).astype(np.float32)}
    return {'mano_params': mp, 'image_id': 7}


def optimized_layout(argued):
    """Template 1's output as the optimiser writes it back (mocap_optimize: 'shape' [N,10] float32 per hand), template 3's input."""
    d = copy.deepcopy(argued)
    for side in ('right', 'left'):
        d[side]['shape'] = np.asarray(d[side]['shape'], dtype=np.float32).reshape(-1, 10)
    return d


def birth(data, PoseArguer, HandPoseConverter, root):
    """data_birth.py:17-69 with argue_size BIRTH_A, end_id BIRTH_FRAMES and splice_data_length BIRTH_SPLICE -> (rot, confidence) per
    splice, in file order."""
    rhpa, lhpa = PoseArguer(side='right', root=root), PoseArguer(side='left', root=root)
    rhpc = HandPoseConverter(side='right', root=root)
    start_id, end_id = 0, BIRTH_FRAMES
    out_rot_data, real_rates = np.asarray([]), []
    for rr in np.arange(0.0, 1.0, 0.1):
        for side_id in list(data.keys()):
            if side_id in ['left', 'right']:
                rot = data[side_id]['rot'][start_id:end_id]
                hpa = rhpa if side_id == 'right' else lhpa
                argued = hpa.argue_pose(rot, pose_type='euler', vis=False, argue_size=BIRTH_A, random_level=1.0 - rr)
                argued = rhpc.mano_quat_flat_2_normal(rhpc.euler_2_mano_quat(argued), return_type='aa')
                real_rates.extend([rr for i in range(len(argued))])
                out_rot_data = argued if len(out_rot_data) == 0 else np.vstack([out_rot_data, argued])
    for side_id in ['left', 'right']:
        out_rot_data = np.vstack([out_rot_data, data[side_id]['rot'][start_id:end_id]])
        real_rates.extend([1.0 for i in range(end_id - start_id)])
    splices = []
    for left_idx in range(0, len(real_rates), BIRTH_SPLICE):
        right_idx = min(len(real_rates), left_idx + BIRTH_SPLICE)
        splices.append({'rot': out_rot_data[left_idx:right_idx], 'confidence': real_rates[left_idx:right_idx]})
    return splices


def run(seed, HandPoseConverter, HandPoseArguer, PoseArguer, tmp):
    rng = np.random.default_rng(seed)
    mano = os.path.join(tmp, 'assets', 'mano')
    conv = {s: HandPoseConverter(side=s, root=mano) for s in ('right', 'left')}
    g = {'converter': {}, 'euler_margin': [], 'branch_margin': []}
    for s, c in conv.items():
        tab = (np.asarray(c.invM_U_n_0), np.asarray(c.invU_M_n_1), np.asarray(c.th_hands_mean))
        euler = rng.uniform(-150, 150, size=(N_CONV, 16, 3))
        euler[..., 1] = rng.uniform(-80, 80, size=(N_CONV, 16))
        aa = (rng.normal(size=(N_CONV, 48)) * 0.6).astype(np.float32)
        quat = c.euler_2_mano_quat(euler)
        aa_q = c.axis_angle_2_mano_quat(aa, flat_hand=False)
        rec = {'inv_m0': tab[0], 'inv_u1': tab[1], 'hands_mean': tab[2], 'euler': euler, 'aa': aa, 'quat': quat,
               'quat_euler': c.mano_quat_2_euler(quat.copy()), 'aa_quat': aa_q, 'aa_quat_flat': c.axis_angle_2_mano_quat(aa, flat_hand=True),
               'flat_aa': c.mano_quat_flat_2_normal(aa_q.copy(), return_type='aa'), 'flat_quat': c.mano_quat_flat_2_normal(aa_q.copy())}
        g['converter'][s] = rec
        _, m1 = pose_data_ref.euler_2_mano_quat(euler, s, tab[0], tab[1], stages=True)
        e2, m2 = pose_data_ref.mano_quat_2_euler(quat, s, tab[0], tab[1], stages=True)
        g['euler_margin'].append(pose_data_ref.euler_margin(e2))
        g['branch_margin'] += [pose_data_ref.branch_margin(m1), pose_data_ref.branch_margin(m2)]
    g['argue'] = {}
    for name, cls in (('HandPoseArguer', HandPoseArguer), ('PoseArguer', PoseArguer)):
        for s in ('right', 'left'):
            euler = rng.uniform(-60, 60, size=(N_ARGUE, 16, 3))
            np.random.seed(seed * 10 + len(g['argue']))
            st = np.random.get_state()
            kw = {'random_level': LEVEL} if name == 'PoseArguer' else {}
            out = cls(side=s, root=mano).argue_pose(euler, argue_size=A_ARGUE, pose_type='euler', **kw)
            np.random.set_state(st)
            u = pose_data_ref.draw_uniforms(N_ARGUE, A_ARGUE)
            g['argue'][(name, s)] = {'seed': seed * 10 + len(g['argue']), 'euler': euler, 'u': u, 'out': out}
            ref, first, mats = pose_data_ref.argue_pose(euler, u, name, kw.get('random_level', 1.0), stages=True)
            assert np.array_equal(ref, out), name
            g['euler_margin'] += [pose_data_ref.euler_margin(out), pose_data_ref.euler_margin(first)]
            g['branch_margin'].append(pose_data_ref.branch_margin(mats))
    # the template scripts, in order, from the scratch directory
    with open(os.path.join(tmp, 'data', 'template_renderih_data_sample.pkl'), 'wb') as f:
        pickle.dump(annotation(rng), f)
    cwd = os.getcwd()
    os.chdir(tmp)
    try:
        runpy.run_path(os.path.join(REF_POSE, 'data', 'template_0_pose_convert.py'), run_name='__main__')
        np.random.seed(seed)
        runpy.run_path(os.path.join(REF_POSE, 'data', 'template_1_pose_argue.py'), run_name='__main__')
        argued = np.load(os.path.join('data', 'template_argued_data0.npy'), allow_pickle=True).item()
        np.save(os.path.join('data', 'template_optimized_data0.npy'), optimized_layout(argued))
        runpy.run_path(os.path.join(REF_POSE, 'data', 'template_3_pose_reconvert.py'), run_name='__main__')
        converted = np.load(os.path.join('data', 'template_converted_data.npy'), allow_pickle=True).item()
        names = sorted(os.path.basename(p) for p in glob.glob(os.path.join('data', 'optimezed_argued_data', '*.npy')))
        reconverted = {'names': names, 'files': {n: np.load(os.path.join('data', 'optimezed_argued_data', n), allow_pickle=True).item()
                                                 for n in names[:KEEP_FILES]}}
        np.random.seed(seed + 1)
        splices = birth(converted, PoseArguer, HandPoseConverter, 'assets/mano')
    finally:
        os.chdir(cwd)
    with open(os.path.join(tmp, 'data', 'template_renderih_data_sample.pkl'), 'rb') as f:
        g['annotation'] = pickle.load(f)
    g.update({'converted': converted, 'argued': argued, 'reconverted': reconverted, 'birth': splices, 'template_seed': seed,
              'birth_seed': seed + 1})
    for side in ('right', 'left'):
        g['euler_margin'] += [pose_data_ref.euler_margin(converted[side]['rot']), pose_data_ref.euler_margin(argued[side]['rot'])]
    return g


def main():
    HandPoseConverter, HandPoseArguer, PoseArguer = import_reference()
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, 'assets', 'mano'))
        os.makedirs(os.path.join(tmp, 'data'))
        for side in ('left', 'right'):
            with open(os.path.join(tmp, 'assets', 'mano', 'MANO_%s.pkl' % side.upper()), 'wb') as f:
                pickle.dump(rih_assets.synthetic_mano(0, side), f)
        for seed in range(1, 40):
            for p in glob.glob(os.path.join(tmp, 'data', '*')):
                if os.path.isdir(p):
                    for q in glob.glob(os.path.join(p, '*')):
                        os.remove(q)
                elif not p.endswith('.pkl'):
                    os.remove(p)
            g = run(seed, HandPoseConverter, HandPoseArguer, PoseArguer, tmp)
            ok = min(g['euler_margin']) >= EULER_MARGIN and min(g['branch_margin']) >= BRANCH_MARGIN
            print('seed %d: euler margin %.3g deg, branch margin %.3g -> %s' % (seed, min(g['euler_margin']), min(g['branch_margin']), ok))
            if ok:
                break
        else:
            raise RuntimeError('no usable seed')
    g['meta'] = {'source': 'pose_data_optimize/scripts/HandPoseConverter.py, HandPoseArguer.py, Ver2Code/NatureJudge/PoseArgue.py and '
                           'data/template_{0,1,3}_*.py executed unmodified on CPU with the synthetic MANO tensors (assets.synthetic_mano(0)); '
                           "data_birth.py's loop restated",
                 'torch': torch.__version__, 'numpy': np.__version__, 'scipy': scipy.__version__, 'seed': seed,
                 'euler_margin_deg': EULER_MARGIN, 'branch_margin': BRANCH_MARGIN,
                 'sizes': {'KEEP_FILES': KEEP_FILES, 'N_CONV': N_CONV, 'N_ARGUE': N_ARGUE, 'A_ARGUE': A_ARGUE, 'LEVEL': LEVEL, 'BIRTH_FRAMES': BIRTH_FRAMES,
                           'BIRTH_A': BIRTH_A, 'BIRTH_SPLICE': BIRTH_SPLICE}}
    torch.save(g, GOLD, pickle_protocol=4)
    print(GOLD, os.path.getsize(GOLD), 'bytes')


if __name__ == '__main__':
    main()
