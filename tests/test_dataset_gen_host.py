"""Host checks of dataset preparation: the float64 oracle (oracle/dataset_gen_ref.py) against the unmodified reference's outputs on the
synthetic InterHand2.6M tree (tests/golden/dataset_gen_synth.pt, oracle/make_golden_dataset_gen.py), the golden against a fresh run of the
reference where its tree is present, and the input checks of the drop-ins."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import dataset_gen_ref as ref
from oracle import make_golden_dataset_gen as mk
from oracle import ref_bridge
from renderih_b200 import dataset_gen as dg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = torch.load(os.path.join(ROOT, 'tests', 'golden', 'dataset_gen_synth.pt'), weights_only=False)
cv2 = pytest.importorskip('cv2')


@pytest.fixture(scope='module')
def tree(tmp_path_factory):
    return mk.make_tree(str(tmp_path_factory.mktemp('tree')))


def _camera(tree, i):
    """load_camera of frame i (the drop-in's host code, interhand.py:126-144)."""
    loader = dg.InterHandLoader.__new__(dg.InterHandLoader)
    base = os.path.join(tree, 'annotations', 'train', 'InterHand2.6M_train')
    with open(base + '_data.json') as f:
        loader.data_info = json.load(f)
    with open(base + '_camera.json') as f:
        loader.cam_params = json.load(f)
    return loader.load_camera(i)


def _frame(tree, i):
    return cv2.imread(os.path.join(tree, 'images', 'train', 'Capture0/seq/cam%s/image%05d.jpg' % (('400002', '400016')[i % 2], i)))


def test_tree_is_reproducible(tree):
    assert mk.tree_hash(tree) == G['tree_hash']


def test_oracle_geometry_matches_reference(tree):
    """M, the updated camera and the crop from the reference's MANO vertices; the reference's `@` sums in its BLAS's order, so M agrees
    to float32 rounding of the camera-frame vertices, and the crop of the reference's own M is byte-exact."""
    for k, verts in enumerate(G['ref_verts']):
        R, t, K = _camera(tree, G['kept_frames'][k])
        o = ref.geometry(verts, None, R, t, K, crop=True)
        assert o['valid']
        assert np.allclose(o['M'], G['warp']['M'][k], rtol=2e-6, atol=0)
        assert np.allclose(o['K'], G['anno'][k]['camera']['camera'], rtol=2e-6, atol=0)
    img = _frame(tree, G['kept_frames'][0])
    assert mk.array_hash(img) == G['warp']['src_hash'][0]
    assert np.array_equal(ref.warp_u8(img, G['warp']['M'][0], 256), G['crop0'])


def test_oracle_crops_match_reference(tree):
    frames = {mk.array_hash(img): img for img in (_frame(tree, i) for i in G['kept_frames'])}
    for k, (h, M) in enumerate(zip(G['warp']['src_hash'], G['warp']['M'])):
        assert mk.array_hash(ref.warp_u8(frames[h], M, 256)) == G['imwrite']['train/img/%d.jpg' % k]


def test_oracle_heatmaps_match_reference():
    """Every heatmap the reference wrote, from its own joints2d: the oracle's float32 maps * 255 are the arrays it passed to cv.imwrite."""
    j = G['joints2d_step7']
    for i in range(j.shape[0]):
        for h, s in enumerate(('left', 'right')):
            hms = ref.heatmaps(j[i, h] * 64 / 256, 64, 2)[0]
            for k in range(7):
                arr = hms[3 * k:3 * k + 3].transpose(1, 2, 0) * 255
                assert mk.array_hash(arr) == G['imwrite']['train/color_hms/%d_%d_%s.jpg' % (i, k, s)]
    for p, a in G['planes'].items():
        i, k, s = os.path.basename(p)[:-4].split('_')
        hms = ref.heatmaps(j[int(i), ('left', 'right').index(s)] * 64 / 256, 64, 2)[0]
        assert np.array_equal(hms[3 * int(k):3 * int(k) + 3].transpose(1, 2, 0) * 255, a)
        assert np.array_equal(ref.planes_u8(hms)[int(k)], np.where(np.isnan(a), 0, np.clip(np.rint(a), 0, 255)).astype(np.uint8))


def test_golden_bookkeeping():
    """The kept frames and files: one crop, annotation, ori_handdict, mask, dense map and 14 heatmaps per kept frame, idx from 0."""
    n = len(G['anno'])
    assert n == len(G['kept_frames']) == G['n_crops'] and [a['inter_idx'] for a in G['anno']] == list(range(n))
    assert [a['image']['id'] for a in G['anno']] == G['kept_frames']
    want = sorted(['train/color_img/%d.jpg' % i for i in range(n)] + ['train/color_annot/%d.pkl' % i for i in range(n)] +
                  ['train/ori_handdict/%d.npy' % i for i in range(n)] + ['train/color_mask/%d.jpg' % i for i in range(n)] +
                  ['train/color_dense/%d.jpg' % i for i in range(n)] +
                  ['train/color_hms/%d_%d_%s.jpg' % (i, k, s) for i in range(n) for k in range(7) for s in ('left', 'right')])
    assert G['files'] == want
    for a in G['anno']:
        assert list(a) == ['inter_idx', 'image', 'annotation', 'mano_params', 'camera']
        assert a['camera']['R'].dtype == a['camera']['t'].dtype == np.float32 and a['camera']['camera'].dtype == np.float64
        for s in ('left', 'right'):
            assert {k: v.shape for k, v in a['mano_params'][s].items()} == {'R': (1, 3, 3), 'pose': (1, 45), 'shape': (1, 10), 'trans': (1, 3)}


@pytest.mark.skipif(not ref_bridge.reference_available(), reason='the reference tree is only present where the golden is authored')
def test_golden_reproduces_from_reference(tmp_path):
    g = mk.run(str(tmp_path))
    for k in ('tree_hash', 'files', 'imwrite', 'kept_frames', 'n_crops'):
        assert g[k] == G[k], k
    assert np.array_equal(g['warp']['M'], G['warp']['M']) and np.array_equal(g['crop0'], G['crop0'])


# ------------------------------------------------------------------------------------------------------------------------ inputs
def test_malformed_inputs_raise():
    with pytest.raises(RuntimeError):
        dg.HeatmapGenerator(64, 2)(torch.zeros(21, 3, dtype=torch.float64))
    with pytest.raises(TypeError):
        dg.HeatmapGenerator(64, 2)(np.zeros((21, 3), np.int64))
    with pytest.raises(ValueError):
        dg.HeatmapGenerator(64, 2)(np.zeros((2, 21, 4)))
    with pytest.raises(ValueError):
        dg.HeatmapGenerator(64, 2)(np.zeros((1, 2, 21, 3)))
    with pytest.raises(RuntimeError):
        dg.cut_img([np.zeros((8, 8, 3), np.uint8)], [torch.zeros(5, 2, dtype=torch.float64)])
    with pytest.raises(TypeError):
        dg.cut_img([np.zeros((8, 8, 3), np.uint8)], [np.zeros((5, 2), np.int32)])
    with pytest.raises(ValueError):
        dg.cut_img([np.zeros((8, 8, 3), np.uint8)], [np.zeros((5, 3))])
    with pytest.raises(RuntimeError):
        dg.crop_u8(torch.zeros(1, 8, 8, 3, dtype=torch.uint8), torch.zeros(1, 2, 3, dtype=torch.float64))
    v = {s: torch.zeros(1, 778, 3) for s in ('left', 'right')}
    with pytest.raises(RuntimeError):
        dg.geometry(v, None, torch.zeros(1, 3, 3), torch.zeros(1, 3), torch.zeros(1, 3, 3, dtype=torch.float64))
    with pytest.raises(NotImplementedError):
        dg.plot_2d_hand(None, np.zeros((21, 2)))
