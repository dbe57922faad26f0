"""Dataset preparation on the H100 (renderih_b200/dataset_gen.py, csrc/dataset_gen.cu): heatmaps against the numpy HeatmapGenerator, crops
against cv2.warpAffine, the geometry against the float64 oracle, and the whole pipeline on the synthetic InterHand2.6M tree against the
unmodified reference's outputs (tests/golden/dataset_gen_synth.pt, oracle/make_golden_dataset_gen.py)."""
import os
import pickle

import numpy as np
import pytest
import torch

from oracle import dataset_gen_ref as ref
from oracle import make_golden_dataset_gen as mk
from oracle import render_ref
from renderih_b200 import assets
from renderih_b200 import dataset_gen as dg

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = torch.load(os.path.join(ROOT, 'tests', 'golden', 'dataset_gen_synth.pt'), weights_only=False)
cv2 = pytest.importorskip('cv2')


def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64)).max(initial=0)


# ------------------------------------------------------------------------------------------------------------------------ heatmaps
@pytest.mark.parametrize('dtype', [np.float64, np.float32])
@pytest.mark.parametrize('scale', [1, 1.7])
def test_heatmaps_match_numpy(dtype, scale):
    rng = np.random.default_rng(1)
    j = np.concatenate([rng.uniform(-4, 68, size=(5, 21, 2)), (rng.random((5, 21, 1)) > 0.2)], -1).astype(dtype)
    j[0, :6, :2] = [[0, 0], [63.999, 10], [64, 10], [10, 64], [-1e-9, 5], [5, 63.5]]       # the border and just outside it
    j[0, :6, 2] = 1
    j[1, 0, :2] = np.nan
    for res, sigma in ((64, 2), (128, -1)):
        hm = dg.HeatmapGenerator(res, sigma)
        got, planes = hm(j, scale, planes=True)
        want = ref.heatmaps(j, res, hm.sigma, scale)
        assert got.dtype == np.float32 and got.shape == want.shape
        fin = np.isfinite(want)
        assert np.array_equal(np.isnan(got), np.isnan(want)) and _ulps(got[fin], want[fin]) <= 1
        assert (got[0, 2] == 0).all() == (got[0, 3] == 0).all() == (res == 64) and (got[0, 0] != 0).any() and (got[0, 4] == 0).all()
        assert np.array_equal(planes, np.stack([ref.planes_u8(g) for g in got]))
        two = hm(j[0, :, :2].astype(dtype), scale)               # 2-D input: one frame, visibility 1
        assert _ulps(two, ref.heatmaps(j[0, :, :2], res, hm.sigma, scale)) <= 1
    t = dg.HeatmapGenerator(64, 2)(torch.from_numpy(j).cuda())
    want = ref.heatmaps(j, 64, 2)
    fin = np.isfinite(want)
    assert t.is_cuda and _ulps(t.cpu().numpy()[fin], want[fin]) <= 1


# ------------------------------------------------------------------------------------------------------------------------ crops
def _crop_matrix(rng, H, W):
    s = rng.uniform(0.4, 3.0)
    mid = rng.uniform([0, 0], [W, H])
    L = 128 / s
    return s * np.array([[1, 0, L - mid[0]], [0, 1, L - mid[1]]])


@pytest.mark.parametrize('hw', [(512, 334), (256, 256), (301, 177)])
def test_crop_equals_cv2(hw):
    rng = np.random.default_rng(hw[0] + hw[1])
    B = 6
    frames = rng.integers(0, 256, size=(B,) + hw + (3,), dtype=np.uint8)
    M = np.stack([_crop_matrix(rng, *hw) for _ in range(B)])
    M[0] = [[1.0, 0, 0], [0, 1.0, 0]]
    crops, sums = dg.crop_u8(torch.from_numpy(frames).cuda(), torch.from_numpy(M).cuda(), 256, sums=True)
    for b in range(B):
        assert np.array_equal(crops[b].cpu().numpy(), cv2.warpAffine(frames[b], M[b], dsize=(256, 256)))
        assert np.float64(sums[b].item()) / frames[b].size == frames[b].mean()


def test_cut_img_matches_oracle():
    rng = np.random.default_rng(7)
    img = rng.integers(0, 256, size=(512, 334, 3), dtype=np.uint8)
    labels = [rng.uniform(50, 250, size=(778, 2)), rng.uniform(80, 300, size=(21, 2)).astype(np.float32)]
    cam = np.array([[1200.0, 0, 160], [0, 1210, 250], [0, 0, 1]])
    M, out, K = ref.cut(np.concatenate([labels[0], labels[1].astype(np.float64)]), 0.8, 256, cam)
    imgs, labs, cam2 = dg.cut_img([img, img[:300]], labels, camera=cam, radio=0.8, img_size=256)
    assert cam2 is cam and np.allclose(cam, K, rtol=1e-12, atol=0)
    assert np.array_equal(imgs[0], cv2.warpAffine(img, M, dsize=(256, 256))) and np.array_equal(imgs[1], cv2.warpAffine(img[:300], M, dsize=(256, 256)))
    assert [lab.shape for lab in labs] == [(778, 2), (21, 2)]
    assert np.allclose(np.concatenate(labs), out, rtol=1e-12, atol=1e-9)


# ------------------------------------------------------------------------------------------------------------------------ geometry
def test_geometry_matches_oracle():
    rng = np.random.default_rng(3)
    B = 9
    v = {s: (rng.normal(size=(B, 778, 3)) * 0.05 + [dx, 0, 0]).astype(np.float32) for s, dx in (('left', -0.04), ('right', 0.04))}
    jn = {s: (rng.normal(size=(B, 21, 3)) * 0.05).astype(np.float32) for s in v}
    R = np.stack([mk._rot(rng, 0.3) for _ in range(B)]).astype(np.float32)
    t = (rng.normal(size=(B, 3)) * 0.05 + [0, 0, 0.8]).astype(np.float32)
    K = np.stack([np.array([[1200 + 50 * rng.random(), 0, 167], [0, 1190, 256], [0, 0, 1.0]]) for _ in range(B)])
    v['left'][2, 100] = np.nan                                   # the dist test: only NaN fails it
    c = lambda x: torch.from_numpy(x).cuda()
    g = dg.geometry({s: c(x) for s, x in v.items()}, {s: c(x) for s, x in jn.items()}, c(R), c(t), c(K), crop=True)
    g = {k: x.cpu().numpy() for k, x in g.items()}
    for b in range(B):
        o = ref.geometry({s: v[s][b] for s in v}, {s: jn[s][b] for s in jn}, R[b], t[b], K[b], crop=True)
        assert bool(g['valid'][b]) == o['valid'] == (b != 2)
        if b == 2:
            continue
        assert np.array_equal(g['v3d'][b], o['v3d']) and np.array_equal(g['j3d'][b], o['j3d'])
        for k in ('v2d', 'j2d', 'M', 'K', 'cut2d'):
            assert np.allclose(g[k][b], o[k], rtol=1e-12, atol=1e-12 * np.abs(o[k]).max()), k


def test_golden_crops_from_reference_matrices(tmp_path):
    """Each warpAffine of the reference (its M and source frame) gives the reference's crop byte for byte."""
    data = mk.make_tree(str(tmp_path))
    assert mk.tree_hash(data) == G['tree_hash']
    loader = dg.InterHandLoader(data, 'train', mk.mano_dicts())
    frames = {mk.array_hash(im): im for im in (loader.load_img(i) for i in G['kept_frames'])}
    src = torch.from_numpy(np.stack([frames[h] for h in G['warp']['src_hash']])).cuda()
    crops = dg.crop_u8(src, torch.from_numpy(G['warp']['M']).cuda(), 256).cpu().numpy()
    want = [G['imwrite']['train/img/%d.jpg' % k] for k in range(len(crops))]
    assert [mk.array_hash(c) for c in crops] == want
    assert np.array_equal(crops[0], G['crop0'])


# ------------------------------------------------------------------------------------------------------------------------ end to end
def _pipeline(root, batch_size):
    data = mk.make_tree(os.path.join(root, 'interhand'))
    save = os.path.join(root, 'processed')
    mano = mk.mano_dicts()
    written = {}
    imwrite = cv2.imwrite

    def rec(path, img, *a):
        written[os.path.relpath(path, save)] = np.array(img, copy=True)
        return imwrite(path, img, *a)
    cv2.imwrite = rec
    try:
        dg.select_data(data, save, 'train', mano_path=mano, batch_size=batch_size)
        ds = dg.InterHand_dataset(save, 'train', 0, mano_path=mano)
        ds.run(batch_size)
        s7 = os.path.join(save, 'train')
        os.rename(os.path.join(s7, 'img'), os.path.join(s7, 'color_img'))
        os.rename(os.path.join(s7, 'anno'), os.path.join(s7, 'color_annot'))
        dense = assets.synthetic_assets(0)['dense_coor']
        n = dg.render_data(save, 'train', 0, mano_path=mano, dense_path=dense, batch_size=batch_size)
        ds7 = dg.step7.InterHand_dataset(s7, 'train', 0, mano_path=mano)
        ds7.run(batch_size)
    finally:
        cv2.imwrite = imwrite
    return save, written, n


def _close(a, b, rtol, atol):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.allclose(a, b, rtol=rtol, atol=atol)


def _check_hand_dict(got, want):
    assert list(got) == list(want)
    for s in ('left', 'right'):
        g, w = got[s], want[s]
        assert list(g) == list(w) and g['hms'] == []
        for k in ('R', 'pose', 'shape', 'camera'):
            assert _close(g[k], w[k], 1e-6, 1e-6), k
        for k, tol in (('verts3d', 2e-6), ('joints3d', 2e-6), ('verts2d', 2e-3), ('joints2d', 2e-3)):     # metres / pixels
            assert _close(g[k], w[k], 0, tol), (k, np.abs(np.asarray(g[k], np.float64) - w[k]).max())


@pytest.fixture(scope='module')
def e2e(tmp_path_factory):
    return {bs: _pipeline(str(tmp_path_factory.mktemp('bs%d' % bs)), bs) for bs in (512, 7, 1)}


def test_end_to_end_files_and_labels(e2e):
    save, written, n = e2e[512]
    assert mk.listing(save) == G['files'] and n == len(G['anno'])
    for i, want in enumerate(G['anno']):
        got = pickle.load(open(os.path.join(save, 'train', 'color_annot', '%d.pkl' % i), 'rb'))
        assert list(got) == list(want) and got['inter_idx'] == want['inter_idx'] == i
        assert got['image'] == want['image'] and got['annotation'] == want['annotation']
        for s in ('left', 'right'):
            for k in ('R', 'pose', 'shape', 'trans'):
                assert _close(got['mano_params'][s][k], want['mano_params'][s][k], 1e-6, 1e-6), k
        for k in ('R', 't'):
            assert np.array_equal(got['camera'][k], want['camera'][k]) and got['camera'][k].dtype == np.float32
        assert _close(got['camera']['camera'], want['camera']['camera'], 1e-5, 0)
    for i, want in enumerate(G['ori']):
        _check_hand_dict(np.load(os.path.join(save, 'train', 'ori_handdict', '%d.npy' % i), allow_pickle=True).item(), want)
    _check_hand_dict(np.load(os.path.join(save, 'train', 'ori_handdict', '0.npy'), allow_pickle=True).item(), G['ori7'][0])
    j2d = np.stack([[np.load(os.path.join(save, 'train', 'ori_handdict', '%d.npy' % i), allow_pickle=True).item()[s]['joints2d']
                     for s in ('left', 'right')] for i in range(n)])
    assert np.abs(j2d - G['joints2d_step7']).max() <= 2e-3


def test_end_to_end_images(e2e):
    """Crops and heatmap planes: exactly what cv2 / the numpy HeatmapGenerator give for this pipeline's own M and joints, and the
    reference's bytes except where the float32 MANO output moved a sample across a rounding boundary."""
    save, written, n = e2e[512]
    assert sorted(written) == sorted(G['imwrite'])
    same = sum(mk.array_hash(written['train/img/%d.jpg' % k]) == G['imwrite']['train/img/%d.jpg' % k] for k in range(n))
    data = os.path.join(os.path.dirname(save), 'interhand')
    loader = dg.InterHandLoader(data, 'train', mk.mano_dicts())
    for k, i in enumerate(G['kept_frames']):
        ann = pickle.load(open(os.path.join(save, 'train', 'color_annot', '%d.pkl' % k), 'rb'))
        K0, K1 = loader.load_camera(i)[2], ann['camera']['camera']
        s_ = K1[0, 0] / K0[0, 0]
        M = np.array([[s_, 0, K1[0, 2] - K0[0, 2] * s_], [0, K1[1, 1] / K0[1, 1], K1[1, 2] - K0[1, 2] * K1[1, 1] / K0[1, 1]]])
        d = np.abs(written['train/img/%d.jpg' % k].astype(int) - cv2.warpAffine(loader.load_img(i), M, dsize=(256, 256)).astype(int))
        assert (d > 1).mean() < 1e-3, (k, (d > 1).mean())
    hm_same = sum(mk.array_hash(a) == G['imwrite'][p] for p, a in written.items() if p.startswith('train/color_hms'))
    hm_total = sum(p.startswith('train/color_hms') for p in written)
    j2d = np.stack([[np.load(os.path.join(save, 'train', 'ori_handdict', '%d.npy' % i), allow_pickle=True).item()[s]['joints2d']
                     for s in ('left', 'right')] for i in range(n)])
    for i in range(n):
        for h, s in enumerate(('left', 'right')):
            want = ref.planes_u8(ref.heatmaps(j2d[i, h] * 64 / 256, 64, 2)[0])
            for k in range(7):
                assert np.array_equal(written['train/color_hms/%d_%d_%s.jpg' % (i, k, s)], want[k])
    for p, a in G['planes'].items():      # the float32 arrays the reference passed to cv.imwrite, converted as cv.imwrite does
        assert np.abs(written[p].astype(int) - ref.planes_u8(np.moveaxis(a / np.float32(255), -1, 0))[0].astype(int)).max() <= 1
    print('crops identical to the reference: %d of %d; heatmap planes identical: %d of %d' % (same, n, hm_same, hm_total))


def test_end_to_end_masks(e2e):
    """The mask and dense map of the first frames against the float64 renderer on this pipeline's own camera-frame vertices."""
    save, written, n = e2e[512]
    faces = render_ref.two_hand_faces(mk.mano_dicts()['right']['f'])
    dense = np.concatenate([assets.synthetic_assets(0)['dense_coor'] * 255] * 2).astype(np.float64)
    mask_col = np.concatenate([np.tile([0., 0., 255.], (778, 1)), np.tile([0., 255., 0.], (778, 1))])
    for i in range(2):
        d = np.load(os.path.join(save, 'train', 'ori_handdict', '%d.npy' % i), allow_pickle=True).item()
        v = np.concatenate([d['left']['verts3d'], d['right']['verts3d']])[None].astype(np.float64)
        cam = render_ref.persp_cam(d['left']['camera'][None].astype(np.float32).astype(np.float64))
        for name, col in (('color_mask', mask_col), ('color_dense', dense)):
            r = render_ref.render(v, faces, cam, True, 256, col, False)
            ok = ~r['ambiguous'][0]
            want = ref.planes_u8(np.moveaxis((r['img'][0]).astype(np.float32), -1, 0))[0]
            got = written['train/%s/%d.jpg' % (name, i)]
            assert ok.mean() > 0.98 and np.abs(got.astype(int) - want.astype(int))[ok].max(initial=0) <= 1, name


def test_batch_size_invariance(e2e):
    """Every file is bitwise the same at batch 512, 7 and 1."""
    base = e2e[512][0]
    for bs in (7, 1):
        other = e2e[bs][0]
        assert mk.listing(other) == mk.listing(base)
        for rel in mk.listing(base):
            a, b = open(os.path.join(base, rel), 'rb').read(), open(os.path.join(other, rel), 'rb').read()
            assert a == b, (bs, rel)
