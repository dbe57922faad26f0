"""Generate tests/golden/dataset_gen_synth.pt by running the UNMODIFIED dataset preparation of the reference (utils/dataset_gen/interhand.py's
select_data and InterHand_dataset, then rendering_code/step7_gen_annotations.py's render_data and InterHand_dataset on the produced
annotations; imported in place from /root/reference) on a synthetic InterHand2.6M tree, on the CPU.

Run in the authoring container only:   python -m oracle.make_golden_dataset_gen

The tree (make_tree, rebuilt by the GPU tests from the same seed) holds N_FRAMES random 334x512 JPEG frames and the four
InterHand2.6M_{split}_{data,camera,joint_3d,MANO_NeuralAnnot}.json files with the keys load_camera / load_mano read: interacting valid
frames, a single-hand frame, an invalid-hand-type frame, a frame without the left hand's MANO entry, one with a short pose and a dark
frame.  MANO is assets.synthetic_mano with the left hand's first shape direction copied from the right hand's, so that fix_shape flips it.

What is substituted: get_mano_path (the synthetic pickles), the yacs / chumpy import shims of oracle/ref_bridge, a matplotlib stub (step 7
imports it at top level), utils.vis_utils replaced by a mano_two_hands_renderer on oracle/render_ref's float64 renderer (pytorch3d is
absent), and an identity Tensor.cuda() (step 7 moves its inputs to the renderer's device).  cv.imwrite and cv.warpAffine are wrapped to
record the exact arrays and matrices each call receives.  The file stores hashes of every written array, the arrays of the first crop
and of three heatmap planes, the matrices and source hashes of every warpAffine, the annotations, the first ori_handdict labels in full
and the joints of all, and the reference's MANO vertices of the first frames: no encoded JPEG, nothing derived from real MANO data.
"""
import contextlib
import glob
import hashlib
import json
import os
import pickle
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_bridge, render_ref  # noqa: E402
from renderih_b200 import assets as rih_assets  # noqa: E402  (asset *generator* only: no kernels involved)

GOLD = os.path.join(ROOT, 'tests', 'golden', 'dataset_gen_synth.pt')
SEED, N_FRAMES, SPLIT = 11, 16, 'train'
H, W = 512, 334
SINGLE, INVALID, NO_LEFT, SHORT_POSE, DARK = 3, 5, 7, 10, 12
N_VERTS, N_ORI = 3, 3


def mano_dicts():
    """Synthetic MANO of both hands; the left hand's shapedirs[:, 0, :] is the right hand's, the case fix_shape corrects."""
    m = {s: rih_assets.synthetic_mano(0, s) for s in ('right', 'left')}
    m['left']['shapedirs'] = m['left']['shapedirs'].copy()
    m['left']['shapedirs'][:, 0, :] = m['right']['shapedirs'][:, 0, :]
    return m


def write_mano(root):
    """-> {'left','right'} pickle paths of mano_dicts() under root."""
    paths = {}
    for s, d in mano_dicts().items():
        paths[s] = os.path.join(root, 'MANO_%s.pkl' % s.upper())
        with open(paths[s], 'wb') as f:
            pickle.dump(d, f)
    return paths


def _rot(rng, scale):
    a = rng.normal(size=3) * scale
    th = np.linalg.norm(a)
    k = a / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def make_tree(root, seed=SEED, n=N_FRAMES, split=SPLIT):
    """The synthetic InterHand2.6M tree under root (images/<split>/..., annotations/<split>/...)."""
    import cv2
    rng = np.random.default_rng(seed)
    ann_dir, img_dir = os.path.join(root, 'annotations', split), os.path.join(root, 'images', split)
    os.makedirs(ann_dir, exist_ok=True)
    cams = ['400002', '400016']
    cam = {'campos': {}, 'camrot': {}, 'focal': {}, 'princpt': {}}
    for c in cams:
        R = _rot(rng, 0.2)
        cam['camrot'][c] = R.tolist()
        cam['campos'][c] = (-R.T @ np.array([0.0, 0.0, 700.0 + 200 * rng.random()])).tolist()
        cam['focal'][c] = [1200 + 100 * rng.random(), 1200 + 100 * rng.random()]
        cam['princpt'][c] = [W / 2 + 10 * rng.normal(), H / 2 + 10 * rng.normal()]
    images, annots, mano = [], [], {'0': {}}
    yy, xx = np.mgrid[0:H, 0:W]
    for i in range(n):
        name = 'Capture0/seq/cam%s/image%05d.jpg' % (cams[i % 2], i)
        images.append({'id': i, 'file_name': name, 'width': W, 'height': H, 'capture': 0, 'camera': cams[i % 2], 'frame_idx': 100 + i,
                       'seq_name': 'seq'})
        annots.append({'id': i, 'image_id': i, 'hand_type': 'right' if i == SINGLE else 'interacting', 'hand_type_valid': 0 if i == INVALID else 1})
        entry = {}
        for s, dx in (('left', -0.04), ('right', 0.04)):
            if s == 'left' and i == NO_LEFT:
                continue
            pose = (rng.normal(size=48) * 0.3).tolist()
            entry[s] = {'pose': pose[:45] if i == SHORT_POSE and s == 'right' else pose, 'shape': (rng.normal(size=10) * 0.5).tolist(),
                        'trans': [dx + 0.01 * rng.normal(), 0.01 * rng.normal(), 0.01 * rng.normal()]}
        mano['0'][str(100 + i)] = entry
        base = rng.uniform(20, 230, size=3)
        img = base + 30 * np.sin(xx[..., None] / rng.uniform(5, 40) + rng.uniform(0, 6, 3)) + rng.normal(0, 8, (H, W, 3))
        if i == DARK:
            img = rng.uniform(0, 12, (H, W, 3))
        os.makedirs(os.path.dirname(os.path.join(img_dir, name)), exist_ok=True)
        cv2.imwrite(os.path.join(img_dir, name), np.clip(img, 0, 255).astype(np.uint8))
    pre = os.path.join(ann_dir, 'InterHand2.6M_' + split)
    for suffix, obj in (('_data.json', {'images': images, 'annotations': annots}), ('_camera.json', {'0': cam}),
                        ('_joint_3d.json', {'0': {}}), ('_MANO_NeuralAnnot.json', mano)):
        with open(pre + suffix, 'w') as f:
            json.dump(obj, f)
    return root


def array_hash(a):
    a = np.ascontiguousarray(a)
    h = hashlib.sha256()
    h.update(('%s%s' % (a.dtype.str, a.shape)).encode())
    h.update(a.tobytes())
    return h.hexdigest()


def tree_hash(root):
    """sha256 over the tree's JSON files and decoded frames (what the pipeline reads)."""
    import cv2
    h = hashlib.sha256()
    for p in sorted(glob.glob(os.path.join(root, '**', '*'), recursive=True)):
        if p.endswith('.json'):
            h.update(open(p, 'rb').read())
        elif p.endswith('.jpg'):
            h.update(array_hash(cv2.imread(p)).encode())
    return h.hexdigest()


def listing(root):
    return sorted(os.path.relpath(p, root) for p in glob.glob(os.path.join(root, '**', '*'), recursive=True) if os.path.isfile(p))


class _RefRenderer:
    """mano_two_hands_renderer(img_size, device) on oracle/render_ref: render_mask / render_densepose with perspective cameras."""

    def __init__(self, img_size=224, device='cuda', **kw):
        self.S = img_size
        self.faces = render_ref.two_hand_faces(mano_dicts()['right']['f'])
        self.dense = np.concatenate([rih_assets.synthetic_assets(0)['dense_coor'] * 255] * 2).astype(np.float64)

    def _render(self, cameras, v3d_left, v3d_right, colors):
        v = torch.cat([v3d_left, v3d_right], 1).double().numpy()
        out = render_ref.render(v, self.faces, render_ref.persp_cam(cameras.double().numpy()), True, self.S, colors, False)
        return torch.from_numpy(out['img']).float(), torch.from_numpy(out['alpha']).float()

    def render_mask(self, cameras=None, v3d_left=None, v3d_right=None, **kw):
        col = np.concatenate([np.tile([0., 0., 255.], (778, 1)), np.tile([0., 255., 0.], (778, 1))])
        return self._render(cameras, v3d_left, v3d_right, col)[0]

    def render_densepose(self, cameras=None, v3d_left=None, v3d_right=None, **kw):
        return self._render(cameras, v3d_left, v3d_right, self.dense)


@contextlib.contextmanager
def reference(mano_path, record):
    """Import the two scripts with the stubs of the module docstring; record[...] collects the imwrite / warpAffine calls."""
    import cv2
    ref_bridge._install_yacs_shim()
    ref_bridge._install_chumpy_shim()
    if ref_bridge.REF_ROOT not in sys.path:
        sys.path.insert(0, ref_bridge.REF_ROOT)
    sys.path.insert(0, os.path.join(ref_bridge.REF_ROOT, 'rendering_code'))
    mpl = types.ModuleType('matplotlib')
    mpl.pyplot = types.ModuleType('matplotlib.pyplot')
    vis = types.ModuleType('utils.vis_utils')
    vis.mano_two_hands_renderer = _RefRenderer
    saved = {k: sys.modules.get(k) for k in ('matplotlib', 'matplotlib.pyplot', 'utils.vis_utils')}
    sys.modules.update({'matplotlib': mpl, 'matplotlib.pyplot': mpl.pyplot, 'utils.vis_utils': vis})
    imwrite, warp, cuda = cv2.imwrite, cv2.warpAffine, torch.Tensor.cuda

    def rec_imwrite(path, img, *a):
        record['imwrite'].append((path, np.array(img, copy=True)))
        return imwrite(path, img, *a)

    def rec_warp(img, M, *a, **k):
        record['warp'].append((array_hash(img), np.array(M, copy=True), k.get('dsize', a[0] if a else None)))
        return warp(img, M, *a, **k)
    cv2.imwrite, cv2.warpAffine, torch.Tensor.cuda = rec_imwrite, rec_warp, lambda self, *a, **k: self
    try:
        import utils.dataset_gen.interhand as ih
        import step7_gen_annotations as s7
        for m in (ih, s7):
            m.get_mano_path = lambda: dict(mano_path)
        yield ih, s7
    finally:
        cv2.imwrite, cv2.warpAffine, torch.Tensor.cuda = imwrite, warp, cuda
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def run(tmp):
    """Build the tree under tmp, run the four reference stages -> golden dict."""
    data, save = make_tree(os.path.join(tmp, 'interhand')), os.path.join(tmp, 'processed')
    mano_path = write_mano(tmp)
    record = {'imwrite': [], 'warp': []}
    with reference(mano_path, record) as (ih, s7):
        ih.select_data(data, save, SPLIT)
        n_crops = len(record['imwrite'])
        ds = ih.InterHand_dataset(save, SPLIT, 0)
        ori = [ds[i][1] for i in range(len(ds))]
        # step 7 reads RenderIH's layout: the produced crops and annotations as color_img / color_annot
        s7dir = os.path.join(save, SPLIT)
        os.rename(os.path.join(s7dir, 'img'), os.path.join(s7dir, 'color_img'))
        os.rename(os.path.join(s7dir, 'anno'), os.path.join(s7dir, 'color_annot'))
        try:
            s7.render_data(save, SPLIT, 0)
        except FileNotFoundError:       # the loop runs to start_idx + 100000 and stops at the first missing annotation
            pass
        ds7 = s7.InterHand_dataset(s7dir, SPLIT, 0)
        ori7 = [ds7[i][1] for i in range(len(ds7))]
        loader = ih.InterHandLoader(data, SPLIT, mano_path)
        kept = [i for i in range(N_FRAMES) if i not in (SINGLE, INVALID, NO_LEFT, SHORT_POSE, DARK)]
        verts = [{s: loader.load_mano(i)[1][s]['verts'][0].numpy() for s in ('left', 'right')} for i in kept[:N_VERTS]]
    annos = [pickle.load(open(os.path.join(s7dir, 'color_annot', '%d.pkl' % i), 'rb')) for i in range(len(ori))]
    writes = {os.path.relpath(p, save): array_hash(a) for p, a in record['imwrite']}
    planes = {os.path.relpath(p, save): a for p, a in record['imwrite'] if os.path.basename(p) in ('0_0_left.jpg', '0_1_left.jpg', '0_6_right.jpg')}
    return {'tree_hash': tree_hash(data), 'files': listing(save), 'imwrite': writes, 'n_crops': n_crops, 'kept_frames': kept,
            'crop0': record['imwrite'][0][1], 'planes': planes,
            'warp': {'src_hash': [w[0] for w in record['warp']], 'M': np.stack([w[1] for w in record['warp']]), 'dsize': record['warp'][0][2]},
            'anno': annos, 'ori': ori[:N_ORI], 'ori7': ori7[:1],
            'joints2d': np.stack([[d[s]['joints2d'] for s in ('left', 'right')] for d in ori]),
            'joints2d_step7': np.stack([[d[s]['joints2d'] for s in ('left', 'right')] for d in ori7]),
            'ref_verts': verts}


def main():
    with tempfile.TemporaryDirectory() as tmp:
        g = run(tmp)
    import cv2
    g['meta'] = {'source': 'utils/dataset_gen/interhand.py select_data / InterHand_dataset and rendering_code/step7_gen_annotations.py '
                           'render_data / InterHand_dataset executed unmodified on CPU on make_tree(SEED) with mano_dicts()',
                 'torch': torch.__version__, 'numpy': np.__version__, 'cv2': cv2.__version__, 'seed': SEED}
    torch.save(g, GOLD, pickle_protocol=4)
    print(GOLD, os.path.getsize(GOLD), 'bytes;', len(g['anno']), 'kept frames;', len(g['files']), 'files')


if __name__ == '__main__':
    main()
