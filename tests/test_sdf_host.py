"""The float64 SDF oracle (oracle/sdf_ref.py) against closed forms, and the default closed-hand faces when the reference assets exist.
No GPU needed."""
import os

import numpy as np
import pytest
import torch

from oracle import sdf_ref as S
from oracle.sdf_ref import box, icosphere


def _box_dist(p, lo, hi):
    lo, hi = np.asarray(lo), np.asarray(hi)
    return np.minimum(p - lo, hi - p).min(1)


def _inside_box(p, lo, hi):
    return np.all((p > np.asarray(lo)) & (p < np.asarray(hi)), 1)


def test_box_is_distance_to_nearest_plane():
    G = 16
    lo, hi = (-0.41, -0.53, -0.29), (0.33, 0.22, 0.47)          # corners off the voxel centres
    v, f = box(lo, hi)
    phi, amb = S.grid(f, v, G)
    c = S.centers(G)
    inside = _inside_box(c, lo, hi)
    ok = ~amb.ravel()
    assert amb.mean() < 0.01 and inside.sum() > 50
    p = phi.ravel()
    assert np.allclose(p[ok & inside], _box_dist(c, lo, hi)[ok & inside], rtol=0, atol=1e-12)
    assert (p[ok & ~inside] == 0).all()


def test_two_disjoint_boxes():
    G = 17
    b1, b2 = ((-0.9, -0.7, -0.6), (-0.1, 0.3, 0.55)), ((0.12, -0.37, -0.8), (0.81, 0.61, 0.05))
    (v1, f1), (v2, f2) = box(*b1), box(*b2)
    v, f = np.concatenate([v1, v2]), np.concatenate([f1, f2 + 8])
    phi, amb = S.grid(f, v, G)
    c = S.centers(G)
    i1, i2 = _inside_box(c, *b1), _inside_box(c, *b2)
    ok, p = ~amb.ravel(), phi.ravel()
    assert i1.sum() > 20 and i2.sum() > 20
    assert np.allclose(p[ok & i1], _box_dist(c, *b1)[ok & i1], atol=1e-12)
    assert np.allclose(p[ok & i2], _box_dist(c, *b2)[ok & i2], atol=1e-12)
    assert (p[ok & ~i1 & ~i2] == 0).all()


def test_icosphere_between_inscribed_and_circumscribed():
    G = 17
    r = 0.7
    v, f = icosphere(r)
    tri = v[f]
    n = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    r_in = np.abs((n * tri[:, 0]).sum(1) / np.linalg.norm(n, axis=1)).min()
    phi, amb = S.grid(f, v, G)
    c = S.centers(G)
    rad = np.linalg.norm(c, axis=1)
    ok, p = ~amb.ravel(), phi.ravel()
    surely_in, surely_out = rad < r_in, rad > r
    assert (p[ok & surely_in] > 0).all() and (p[ok & surely_out] == 0).all()
    assert np.all(p[ok & surely_in] >= r_in - rad[ok & surely_in] - 1e-12)
    assert np.all(p[ok & surely_in] <= r - rad[ok & surely_in] + 1e-12)


def test_half_voxel_centres_at_g4():
    c = S.centers(4)
    assert np.allclose(np.unique(c[:, 0]), [-2 / 3, 0, 2 / 3, 4 / 3])       # -1 + (idx + 0.5) * 2/3: half a voxel off the nodes
    assert np.allclose(c[1], [0, -2 / 3, -2 / 3]) and np.allclose(c[4], [-2 / 3, 0, -2 / 3]) and np.allclose(c[16], [-2 / 3, -2 / 3, 0])
    lo, hi = (-0.2, -0.9, -0.85), (0.25, 0.3, 0.5)
    v, f = box(lo, hi)
    phi, amb = S.grid(f, v, 4)
    assert not amb.any()
    want = np.zeros((4, 4, 4))
    for k in (0, 1):
        for j in (0, 1):
            want[k, j, 1] = _box_dist(np.array([[0.0, c[4 * j, 1], c[16 * k, 2]]]), lo, hi)[0]
    assert np.allclose(phi, want, atol=1e-12)


@pytest.mark.parametrize('G', [2, 5, 32])
def test_trilinear_matches_grid_sample(G):
    rng = np.random.default_rng(G)
    phi = rng.random((G, G, G)) * (rng.random((G, G, G)) > 0.4)
    d = 2.0 / (G - 1)
    x = np.concatenate([
        rng.uniform(-1.2, 1.2, (400, 3)),                                 # some outside the grid
        rng.choice([-1.0, 1.0], (20, 3)),                                 # grid corners
        -1.0 + rng.integers(0, G, (20, 3)) * d,                           # exactly on nodes
        np.stack([np.full(10, -1.0 - d / 3), rng.uniform(-1, 1, 10), rng.uniform(-1, 1, 10)], 1),   # within a cell of the border
        np.stack([rng.uniform(-1, 1, 10), np.full(10, 1.0 + d / 3), rng.uniform(-1, 1, 10)], 1),
        np.array([[5.0, 0.0, 0.0], [0.0, -7.0, 0.2]]),                  # far outside
    ])
    p, dp = S.trilinear(phi, x)
    xt = torch.from_numpy(x).requires_grad_(True)
    out = torch.nn.functional.grid_sample(torch.from_numpy(phi)[None, None], xt.view(1, -1, 1, 1, 3), align_corners=True,
                                          padding_mode='zeros').view(-1)
    (gx,) = torch.autograd.grad(out.sum(), xt)
    assert np.allclose(p, out.detach().numpy(), rtol=0, atol=1e-13)
    assert np.allclose(dp, gx.numpy(), rtol=0, atol=1e-11)


def test_part_counts_and_frame():
    m = S.part_counts([[0, 1, 1, 2], [2, 3], {0, 2}], 5)
    assert m.tolist() == [2, 1, 3, 1, 0]
    v = np.array([[0.0, 1.0, 2.0], [1.0, -1.0, 3.0], [0.5, 0.0, 2.5]], np.float32)
    c, s = S.frame(v, 0.1)
    assert np.allclose(c, [0.5, 0.0, 2.5]) and np.isclose(s, 0.55 * 2.0)


def _asset(*rel):
    from renderih_b200.assets import default_asset_root
    return os.path.join(default_asset_root(), *rel)


def test_default_closed_faces():
    from renderih_b200 import sdf as rs
    path = _asset(rs.CLOSED_HAND_OBJ)
    mano = _asset('misc', 'mano', 'MANO_RIGHT.pkl')
    if not (os.path.exists(path) and os.path.exists(mano)):
        pytest.skip('reference assets not present under the asset root')
    f = rs.load_obj_faces(path)
    assert f.shape == (1552, 3)
    edges = {}
    for a, b, c in f:
        for e in ((a, b), (b, c), (c, a)):
            k = (min(e), max(e))
            edges[k] = edges.get(k, 0) + 1
    assert set(edges.values()) == {2}
    from renderih_b200.assets import load_mano_dict
    assert np.array_equal(f[:1538], np.asarray(load_mano_dict(mano)['f'], np.int64))
    parts = rs.load_part_vert(_asset(rs.PART_VERT))
    assert len(parts) == 16 and sum(len(p) for p in parts) == 934
    assert set(np.concatenate([list(p) for p in parts]).tolist()) == set(range(778))
