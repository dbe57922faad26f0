"""Generate tests/golden/collision_synth.pt and tests/golden/valid_judge_synth.pt by running the UNMODIFIED post-optimisation filters of
the pose data pipeline, imported in place from /root/reference/pose_data_optimize, on the CPU:
  * filter_collision_data of collision/CollisionFilter.py (run from a scratch directory whose ../assets/mano holds the synthetic MANO
    pickles, since the function hard-codes that path);
  * ValidJudger.ComputeValidation of Ver2Code/ValidJudge/ValidJudger.py, per file, combined as GetValidRate.py combines them (that
    script runs on import with hard-coded paths, so its five-line loop is restated here).

Run in the authoring container only:   python -m oracle.make_golden_filters
What is substituted: the stand-ins of make_golden_geo_loss (numpy 2's removed np.long, the chumpy-free MANO loader, an empty open3d);
HandPoseConverter's default device 'cuda:0' becomes 'cpu'; and a trimesh stub whose CollisionManager.in_collision_internal returns
as many contacts as oracle/collision_ref counts intersecting face pairs between the two meshes it holds.  So the files check the
reference's data plumbing end to end (loading, euler -> quaternion, both hand layers, translations, the left faces, the threshold, the
saved dict), while the count itself is the oracle's.
Synthetic MANO (assets.synthetic_mano: random faces over a random vertex cloud) and a synthetic mocap dict whose hands sit at varying
distances.  A seed is kept when the counts fall on both sides of MAX_CONTACTS, every count is at least COUNT_MARGIN from it and more than
its fragile pairs away, some frames are valid and some not, and every validity score is 0 or at least SCORE_MARGIN from the threshold.
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
from oracle import collision_ref, make_golden_geo_loss  # noqa: E402
from renderih_b200 import assets as rih_assets  # noqa: E402  (asset *generator* only: no kernels involved)

REF_POSE = make_golden_geo_loss.REF_POSE
GOLD_DIR = os.path.join(ROOT, 'tests', 'golden')
N_FRAMES, SPLIT, MAX_CONTACTS = 16, 9, 75
COUNT_MARGIN, SCORE_MARGIN = 10, 1e-4
CALLS = []


class _Trimesh:
    def __init__(self, vertices, faces, **kw):
        self.vertices, self.faces = np.asarray(vertices), np.asarray(faces)


class _CollisionManager:
    def __init__(self):
        self.objects = {}

    def add_object(self, name, mesh):
        self.objects[name] = mesh

    def in_collision_internal(self, return_data=False):
        a, b = self.objects['right'], self.objects['left']
        n, frag = collision_ref.frame_count(a.vertices, b.vertices, a.faces)
        CALLS.append((n, frag))
        return n > 0, [None] * n


def import_reference():
    tm = types.ModuleType('trimesh')
    tc = types.ModuleType('trimesh.collision')
    tm.Trimesh, tc.CollisionManager, tm.collision = _Trimesh, _CollisionManager, tc
    sys.modules['trimesh'], sys.modules['trimesh.collision'] = tm, tc
    make_golden_geo_loss.import_reference()
    import scripts.HandPoseConverter as hpc
    d = list(hpc.HandPoseConverter.__init__.__defaults__)
    d[-1] = 'cpu'
    hpc.HandPoseConverter.__init__.__defaults__ = tuple(d)
    sys.modules['HandPoseConverter'] = hpc          # CollisionFilter / ValidJudger import it as a top-level module
    for sub in ('collision', os.path.join('Ver2Code', 'ValidJudge')):
        sys.path.insert(0, os.path.join(REF_POSE, sub))
    import CollisionFilter
    import ValidJudger
    return CollisionFilter, ValidJudger, hpc


def synthetic_mocap(seed, rest):
    """The optimised-mocap layout the filter reads: {'right'/'left': {'rot' [N,16,3] degrees, 'loc' [N,3] cm, 'shape' [N,10]}} plus a
    1-D 'capture_frame_id'.  The hands are 4..60 cm apart; in a third of the frames every finger joint is within 1 degree (standard
    deviation) of rest[side], the euler angles of identity MANO quaternions, so those poses are valid."""
    rng = np.random.default_rng(seed)
    sep = rng.uniform(4.0, 60.0, N_FRAMES)
    d = {}
    for side, x in (('right', 0.5), ('left', -0.5)):
        rot = rng.normal(size=(N_FRAMES, 16, 3)) * 15.0
        rot[::3, 1:] = rest[side][1:] + rng.normal(size=rot[::3, 1:].shape)
        rot[:, 0] = rng.normal(size=(N_FRAMES, 3)) * 40.0
        loc = np.stack([x * sep, rng.normal(size=N_FRAMES), rng.normal(size=N_FRAMES)], 1)
        d[side] = {'rot': rot, 'loc': loc, 'shape': rng.normal(size=(N_FRAMES, 10)) * 0.5}
    d['capture_frame_id'] = np.arange(N_FRAMES, dtype=np.int64) * 7 + 3
    return d


def main():
    CF, VJ, hpc = import_reference()
    with tempfile.TemporaryDirectory() as tmp:
        mano = os.path.join(tmp, 'assets', 'mano')
        os.makedirs(mano)
        os.makedirs(os.path.join(tmp, 'work'))
        for side in ('left', 'right'):
            with open(os.path.join(mano, 'MANO_%s.pkl' % side.upper()), 'wb') as f:
                pickle.dump(rih_assets.synthetic_mano(0, side), f)
        cwd = os.getcwd()
        os.chdir(os.path.join(tmp, 'work'))
        try:
            conv = {s: tuple(np.asarray(getattr(hpc.HandPoseConverter(side=s), k)) for k in ('invM_U_n_0', 'invU_M_n_1'))
                    for s in ('right', 'left')}
            ident = np.tile(np.asarray([1.0, 0, 0, 0], np.float32), (1, 16, 1))
            rest = {s: hpc.HandPoseConverter(side=s).mano_quat_2_euler(ident.copy())[0] for s in ('right', 'left')}
            for seed in range(200, 260):
                raw = synthetic_mocap(seed, rest)
                src, dst = os.path.join(tmp, 'in.npy'), os.path.join(tmp, 'out.npy')
                np.save(src, raw)
                del CALLS[:]
                CF.filter_collision_data(src, dst)
                counts = np.array([c[0] for c in CALLS])
                fragile = np.array([c[1] for c in CALLS])
                judger = VJ.ValidJudger(mano, device='cpu')
                quat = {s: hpc.HandPoseConverter(side=s).euler_2_mano_quat(raw[s]['rot']) for s in ('right', 'left')}
                scores, rates = {}, []
                th = np.float32(0.1 / 180 * np.pi)
                for lo, hi in ((0, SPLIT), (SPLIT, N_FRAMES)):
                    ql, qr = (torch.from_numpy(quat[s][lo:hi]) for s in ('left', 'right'))
                    rates.append(judger.ComputeValidation(ql, qr))
                r_s = judger.ValidationJudge(judger.rhpc.mano_quat_2_mat_tensor(torch.from_numpy(quat['right']))[:, 1:], judger.zero_mat_[:, 1:], 'r')
                l_s = judger.ValidationJudge(judger.lhpc.mano_quat_2_mat_tensor(torch.from_numpy(quat['left']))[:, 1:], judger.sub_zero_mat_[:, 1:], 'l')
                scores = {'right': r_s, 'left': l_s}
                total = rates[0] * SPLIT + rates[1] * (N_FRAMES - SPLIT)
                rate = total / N_FRAMES
                allsc = torch.cat([r_s, l_s]).numpy()
                gap = np.abs(counts - MAX_CONTACTS)
                invalid = ((r_s > th) | (l_s > th)).numpy()
                ok = ((counts <= MAX_CONTACTS).any() and (counts > MAX_CONTACTS).any() and (gap >= COUNT_MARGIN).all() and (gap > fragile).all()
                      and invalid.any() and not invalid.all() and ((allsc == 0) | (np.abs(allsc - th) > SCORE_MARGIN)).all())
                print('seed %d: counts %s fragile %d invalid %d -> %s' % (seed, counts.tolist(), fragile.sum(), invalid.sum(), ok))
                if ok:
                    break
            else:
                raise RuntimeError('no usable seed')
            saved = np.load(dst, allow_pickle=True).item()
            faces = CF.ManoLayer(mano_root='../assets/mano', use_pca=False, flat_hand_mean=True, side='left', root_rot_mode='quat',
                                 joint_rot_mode='quat').th_faces
            # the reference's vertices, recomputed as filter_collision_data computes them (:71-99), so the oracle can be rerun on them
            lay = {s: CF.ManoLayer(mano_root='../assets/mano', use_pca=False, ncomps=6, flat_hand_mean=True, center_idx=0, return_transf=False,
                                   side=s, root_rot_mode='quat', joint_rot_mode='quat') for s in ('right', 'left')}
            verts = {s: lay[s](torch.from_numpy(quat[s]), torch.from_numpy(raw[s]['shape'].astype(np.float32)))[0] for s in ('right', 'left')}
        finally:
            os.chdir(cwd)
    loc = {s: torch.from_numpy(raw[s]['loc'] * 1.0 / 100) for s in ('right', 'left')}
    xr = verts['right'].double().numpy() + loc['right'].numpy()[:, None]
    xl = verts['left'].double().numpy() + loc['left'].numpy()[:, None]
    assert collision_ref.counts(xr, xl, np.asarray(faces))[0].tolist() == counts.tolist()
    meta = {'source': 'pose_data_optimize/collision/CollisionFilter.py filter_collision_data and Ver2Code/ValidJudge/ValidJudger.py executed '
                      'unmodified in place on CPU with the synthetic MANO tensors; the contact count is oracle/collision_ref.py',
            'torch': torch.__version__, 'numpy': np.__version__, 'seed': seed}
    torch.save({'meta': meta, 'raw': raw, 'saved': saved, 'kept_fraction': float((counts <= MAX_CONTACTS).mean()), 'max_contacts': MAX_CONTACTS,
                'counts': torch.from_numpy(counts), 'fragile': torch.from_numpy(fragile), 'kept': (counts <= MAX_CONTACTS).tolist(),
                'rv': verts['right'].contiguous(), 'lv': verts['left'].contiguous(), 'right_loc': loc['right'], 'left_loc': loc['left'],
                'faces': faces.to(torch.int32)}, os.path.join(GOLD_DIR, 'collision_synth.pt'))
    torch.save({'meta': meta, 'raw': raw, 'split': SPLIT, 'quat': {s: torch.from_numpy(quat[s]) for s in quat}, 'converter': conv,
                'scores': scores, 'file_rates': [float(r) for r in rates], 'rate': torch.as_tensor(rate)},
               os.path.join(GOLD_DIR, 'valid_judge_synth.pt'))
    for f in ('collision_synth.pt', 'valid_judge_synth.pt'):
        print(f, os.path.getsize(os.path.join(GOLD_DIR, f)), 'bytes')


if __name__ == '__main__':
    main()
