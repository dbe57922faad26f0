"""Generate tests/golden/mano_fit_synth.pt by running the UNMODIFIED utils/mano_from_3djoint/convert2mano.py (with runpy, in a temporary
directory, on the CPU) once per recorded frame of a synthetic motion-capture take.

Run in the authoring container only:   python -m oracle.make_golden_mano_fit

Set-up: the take (make_take) is a world-position CSV in the reference's column naming ('<Joint>.X/.Y/.Z', plus '_End' columns the
column rule must skip) whose rows are MANO joints of random poses of the synthetic hands, in centimetres, with noise.  The script reads
row frame_idx = 40 of the CSV it opens; for recorded frame f the CSV written for that run holds take row f at row 40.  MANO is
assets.synthetic_mano in mano/MANO_{LEFT,RIGHT}.pkl.  Stand-ins: transforms3d.axangles.axangle2mat (oracle.mano_fit_ref's restatement of
the published formula), matplotlib (no-op figure), and manopth's chumpy loader (make_golden_manopth.plain_ready_arguments).

Recorded per frame and hand: the template and P given to adaptive_IK and its output, every iteration's loss (Tensor.backward wrapped),
the first step's gradients and parameters after it (Adam.step wrapped), the final pose_R / beta, and both .obj files' vertices.  Isolated
cases: adaptive_IK on random pairs, on a near-reflection palm (flipped), on a reflected palm that is kept, on a bone exactly parallel
to its template bone (NaN), and on palms flat exactly and to 1e-9 in planes off the axes; the reference's mat2aa and its gradient on matrices of all four branches, the identity and free matrices.
"""
import os
import pickle
import runpy
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import make_golden_manopth, mano_fit_ref, ref_bridge  # noqa: E402
from renderih_b200 import assets as rih_assets  # noqa: E402  (asset *generator* only: no kernels involved)

GOLD = os.path.join(ROOT, 'tests', 'golden', 'mano_fit_synth.pt')
SCRIPT_DIR = os.path.join(ref_bridge.REF_ROOT, 'utils', 'mano_from_3djoint')
CSV_NAME = 'EP04_HZ800_SC220427_HZ_shot17_242_0427_ani_worldpos.csv'
SEED, N_ROWS = 5, 48
FRAMES = [40, 3, 17]
SCRIPT_ROW = 40


def mano_dicts():
    return {s: rih_assets.synthetic_mano(0, s) for s in ('left', 'right')}


def _rodrigues(a):
    th = np.linalg.norm(a)
    k = a / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def take_joints(seed=SEED, n=N_ROWS):
    """{'left','right'}: [n,21,3] float64 joints in centimetres: the synthetic layer (renderih-independent torch CPU statement of the
    reference ManoLayer, imported from the reference) at random poses, scaled and moved, plus 0.05 cm noise."""
    if ref_bridge.REF_ROOT not in sys.path:
        sys.path.insert(0, ref_bridge.REF_ROOT)
    from models.manolayer import ManoLayer
    rng = np.random.default_rng(seed)
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for s, d in mano_dicts().items():
            p = os.path.join(tmp, s + '.pkl')
            with open(p, 'wb') as f:
                pickle.dump(d, f)
            layer = ManoLayer(p)
            R = torch.from_numpy(np.stack([_rodrigues(rng.normal(size=3)) for _ in range(n)])).float()
            pca = torch.from_numpy(rng.normal(size=(n, 45)) * 0.6).float()
            beta = torch.from_numpy(rng.normal(size=(n, 10))).float()
            with torch.no_grad():
                j = layer(R, pca, beta)[1].double().numpy()
            j = j * (900 + 200 * rng.random((n, 1, 1))) + rng.normal(size=(n, 1, 3)) * 50 + rng.normal(size=j.shape) * 0.05
            out[s] = j
    return out


def write_csv(path, joints, row_order):
    """The take as a world-position CSV: a Frame column, then per joint of both hands '<name>.X/.Y/.Z', and an '_End' joint per finger."""
    names = mano_fit_ref.LEFT + mano_fit_ref.RIGHT
    cols, data = ['Frame'], [np.arange(len(row_order), dtype=np.float64)]
    for side, hand in (('left', mano_fit_ref.LEFT), ('right', mano_fit_ref.RIGHT)):
        for i, n in enumerate(hand):
            for c, ax in enumerate('XYZ'):
                cols.append('%s.%s' % (n, ax))
                data.append(joints[side][row_order, i, c])
            if n.endswith('4_' + n[-1]):
                for c, ax in enumerate('XYZ'):
                    cols.append('%s_End.%s' % (n, ax))
                    data.append(joints[side][row_order, i, c] + 1.0)
    assert len(names) == 42
    with open(path, 'w') as f:
        f.write(','.join(cols) + '\n')
        for r in range(len(row_order)):
            f.write(','.join(repr(float(d[r])) for d in data) + '\n')


class _Any:
    def __getattr__(self, k):
        return lambda *a, **kw: _Any()


def _stubs():
    t3d = types.ModuleType('transforms3d')
    t3d.axangles = types.ModuleType('transforms3d.axangles')
    t3d.axangles.axangle2mat = lambda axis, angle, is_normalized=False: mano_fit_ref.axangle2mat(axis, float(np.asarray(angle).reshape(-1)[0]))
    mpl = types.ModuleType('matplotlib')
    mpl.pyplot = types.ModuleType('matplotlib.pyplot')
    mpl.pyplot.figure = lambda *a, **k: _Any()
    return {'transforms3d': t3d, 'transforms3d.axangles': t3d.axangles, 'matplotlib': mpl, 'matplotlib.pyplot': mpl.pyplot}


def read_obj(path):
    v = [list(map(float, l.split()[1:4])) for l in open(path) if l.startswith('v ')]
    return np.array(v)


def run_frame(tmp, joints, f):
    """Run the script with take row f at row 40 -> per-hand records."""
    order = list(range(N_ROWS))
    order[SCRIPT_ROW], order[f] = order[f], order[SCRIPT_ROW]
    write_csv(os.path.join(tmp, CSV_NAME), joints, order)
    import AIK
    rec = {'aik': [], 'hands': []}
    aik = AIK.adaptive_IK

    def rec_aik(T, P):
        out = aik(T, P)
        rec['aik'].append((np.array(T), np.array(P), out.copy()))
        return out
    AIK.adaptive_IK = rec_aik
    adam_init, adam_step, backward = torch.optim.Adam.__init__, torch.optim.Adam.step, torch.Tensor.backward

    def init(self, params, *a, **k):
        params = list(params)
        adam_init(self, params, *a, **k)
        rec['hands'].append({'opt': self, 'loss': [], 'steps': 0})

    def step(self, *a, **k):
        h = rec['hands'][-1]
        if h['steps'] == 0:
            h['grad0'] = [p.grad.clone() for p in self.param_groups[0]['params']]
            h['lr0'] = self.param_groups[0]['lr']
        out = adam_step(self, *a, **k)
        if h['steps'] == 0:
            h['after0'] = [p.detach().clone() for p in self.param_groups[0]['params']]
        h.setdefault('lrs', []).append(self.param_groups[0]['lr'])
        h['steps'] += 1
        return out

    def bw(self, *a, **k):
        rec['hands'][-1]['loss'].append(float(self))
        return backward(self, *a, **k)
    torch.optim.Adam.__init__, torch.optim.Adam.step, torch.Tensor.backward = init, step, bw
    cwd = os.getcwd()
    try:
        os.chdir(tmp)
        runpy.run_path(os.path.join(SCRIPT_DIR, 'convert2mano.py'), run_name='__main__')
    finally:
        os.chdir(cwd)
        AIK.adaptive_IK = aik
        torch.optim.Adam.__init__, torch.optim.Adam.step, torch.Tensor.backward = adam_init, adam_step, backward
    out = {}
    for i, s in enumerate(('left', 'right')):
        h = rec['hands'][i]
        T, P, R = rec['aik'][i]
        params = h['opt'].param_groups[0]['params']          # OptimizationSMPL registers beta before pose
        assert tuple(params[0].shape) == (1, 10) and tuple(params[1].shape) == (1, 16, 3, 3)
        out[s] = {'joints': joints[s][f], 'template': T, 'P': P, 'aik': R, 'loss': np.array(h['loss'], np.float32), 'lrs': h['lrs'],
                  'grad0': {'pose_R': h['grad0'][1].numpy(), 'beta': h['grad0'][0].numpy()},
                  'after0': {'pose_R': h['after0'][1].numpy(), 'beta': h['after0'][0].numpy()},
                  'pose_R': params[1].detach().numpy().copy(), 'beta': params[0].detach().numpy().copy(),
                  'cur_obj': read_obj(os.path.join(tmp, 'cur_frame%d_%s.obj' % (SCRIPT_ROW, s))),
                  'ori_obj': read_obj(os.path.join(tmp, 'ori_frame%d_%s.obj' % (SCRIPT_ROW, s)))}
    return out


def aik_cases(rng):
    """Isolated (T, P) pairs: random, a flipped near-reflection palm, a kept reflection, an exactly parallel bone."""
    cases = []
    for _ in range(4):
        T = rng.normal(size=(21, 3)) * 0.05
        P = T + rng.normal(size=(21, 3)) * 0.02
        P[0] = T[0]
        cases.append(('random', T, P))
    T = rng.normal(size=(21, 3)) * 0.05
    T[[1, 5, 9, 13, 17], 2] = T[0, 2] + rng.normal(size=5) * 1e-4          # nearly planar palm: the smallest singular value < 1e-4
    P = T.copy()
    P[:, 0] = 2 * T[0, 0] - T[:, 0]                                         # mirrored about the wrist: a reflection
    P += rng.normal(size=(21, 3)) * 1e-3
    P[0] = T[0]
    cases.append(('near_reflection', T, P))
    T = rng.normal(size=(21, 3)) * 0.05
    P = T.copy()
    P[:, 0] = 2 * T[0, 0] - T[:, 0]
    P += rng.normal(size=(21, 3)) * 1e-2       # no bone left parallel to its template bone: that axis would be rounding noise
    P[0] = T[0]
    cases.append(('kept_reflection', T, P))
    # axis-aligned dyadic palm: H is diagonal, V U^T is exactly I, and the thumb's first bone of P is exactly twice its template bone
    T = np.zeros((21, 3))
    T[[1, 5, 9, 13, 17]] = [[0.5, 0, 0], [0, 0.5, 0], [0, 0, 0.5], [0.25, 0, 0], [0, 0.25, 0]]
    for a in (1, 5, 9, 13, 17):
        for s in range(1, 4):
            T[a + s] = T[a + s - 1] + np.array([0.125, 0.0625 * s, 0.25 - 0.03125 * s]) * (1 + a / 32)
    P = T.copy()
    P[[1, 5, 9, 13, 17]] *= [1.0, 1.5, 2.0]
    for a in (5, 9, 13, 17):
        P[a + 1:a + 4] = P[a] + (T[a + 1:a + 4] - T[a]) * [1.0, 0.75, 1.25] + 0.015625
    P[2] = T[1] + 2 * (T[2] - T[1])
    P[3:5] = P[2] + (T[3:5] - T[2]) * 0.5 + [[0.03125, 0, 0], [0, 0.0625, 0]]
    cases.append(('parallel_bone', T, P))
    return cases


def flat_palm_cases(rng):
    """(T, P) pairs whose wrist and five base joints lie in one plane that is not axis-aligned: exactly (to rounding) and to 1e-9,
    each rotated at random; the fingers are random.  The smallest singular value of H is then rounding-level."""
    def rot():
        q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        return q * np.sign(np.linalg.det(q))
    cases = []
    for name, flat in (('flat_palm', 0.0), ('flat_palm', 0.0), ('flat_palm_1e-9', 1e-9), ('flat_palm_1e-9', 1e-9)):
        T = rng.normal(size=(21, 3)) * 0.05
        P = T + rng.normal(size=(21, 3)) * 0.02
        for X in (T, P):
            palm = np.c_[rng.normal(size=(6, 2)) * 0.05, rng.normal(size=6) * flat] @ rot().T
            X[[0, 1, 5, 9, 13, 17]] = palm
        P += T[0] - P[0]
        cases.append((name, T, P))
    return cases


def mat2aa_cases(rng):
    def rot(axis, th):
        return _rodrigues(np.asarray(axis, np.float64) / np.linalg.norm(axis) * th)
    mats = [rot([0.2, 0.3, 0.9], 0.4), rot([1, 0.1, 0.05], 3.0), rot([0.1, 1, 0.05], 3.0), rot([0.05, 0.1, 1], 2.5), rot([1, 0.2, 0.1], 2.9),
            np.eye(3)]
    mats += [rot(rng.normal(size=3), rng.uniform(0.1, 3.1)) + rng.normal(size=(3, 3)) * 0.05 for _ in range(10)]
    return np.stack(mats).astype(np.float32)


def main():
    ref_bridge._install_chumpy_shim()
    for p in (SCRIPT_DIR, make_golden_manopth.REF_MANOPTH, ref_bridge.REF_ROOT):     # the package `utils` must shadow the script's utils.py
        if p in sys.path:
            sys.path.remove(p)
        sys.path.insert(0, p)
    saved = {k: sys.modules.get(k) for k in _stubs()}
    sys.modules.update(_stubs())
    make_golden_manopth.import_reference_layer()
    joints = take_joints()
    g = {'frames': {}, 'take': joints, 'script_row': SCRIPT_ROW}
    try:
        with tempfile.TemporaryDirectory() as tmp:
            os.makedirs(os.path.join(tmp, 'mano'))
            for s, d in mano_dicts().items():
                with open(os.path.join(tmp, 'mano', 'MANO_%s.pkl' % s.upper()), 'wb') as fh:
                    pickle.dump(d, fh)
            for f in FRAMES:
                g['frames'][f] = run_frame(tmp, joints, f)
                print('frame', f, 'final losses', [float(g['frames'][f][s]['loss'][-1]) for s in ('left', 'right')])
            import pandas as pd
            g['csv_rows'] = {f: mano_fit_ref.get_3djoints(pd.read_csv(os.path.join(tmp, CSV_NAME)), SCRIPT_ROW) for f in FRAMES[-1:]}
        from AIK import adaptive_IK
        from utils.mano_from_3djoint.utils import mat2aa
        rng = np.random.default_rng(SEED + 1)
        g['aik_cases'] = [(n, T, P, adaptive_IK(T, P)) for n, T, P in aik_cases(rng)]
        g['aik_cases'] += [(n, T, P, adaptive_IK(T, P)) for n, T, P in flat_palm_cases(np.random.default_rng(SEED + 2))]
        R = torch.from_numpy(mat2aa_cases(rng)).requires_grad_(True)
        aa = mat2aa(R)
        gup = torch.from_numpy(rng.normal(size=(R.shape[0], 3))).float()
        (aa * gup).sum().backward()
        g['mat2aa'] = {'R': R.detach().numpy(), 'aa': aa.detach().numpy(), 'g_aa': gup.numpy(), 'dR': R.grad.numpy()}
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    g['meta'] = {'source': 'utils/mano_from_3djoint/convert2mano.py executed unmodified on CPU per frame of take_joints(SEED)',
                 'torch': torch.__version__, 'numpy': np.__version__, 'seed': SEED}
    torch.save(g, GOLD, pickle_protocol=4)
    print(GOLD, os.path.getsize(GOLD), 'bytes')


if __name__ == '__main__':
    main()
