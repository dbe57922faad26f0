"""Host checks of the collision and validity oracles (oracle/collision_ref.py) and of the filter's record assembly: the float64
Guigue-Devillers predicate against an independent exact test (separating axes in rational arithmetic), the oracle's counts and
scores against the golden files made by the unmodified reference, and collision.filtered_records against the reference's dict_add."""
import os
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import collision_ref as C
from renderih_b200 import collision

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


# ------------------------------------------------------------------------------------------------------------------------ exact reference
def _fsub(a, b):
    return [x - y for x, y in zip(a, b)]


def _fcross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _fdot(a, b):
    return sum(x * y for x, y in zip(a, b))


def exact_intersect(t1, t2):
    """Closed triangles in exact rational arithmetic, by separating axes: the two normals, the nine edge-edge cross products and the six
    in-plane edge normals.  A triangle with zero area intersects nothing (the predicate's definition)."""
    t1 = [[Fraction(float(x)) for x in p] for p in t1]
    t2 = [[Fraction(float(x)) for x in p] for p in t2]
    n1 = _fcross(_fsub(t1[1], t1[0]), _fsub(t1[2], t1[0]))
    n2 = _fcross(_fsub(t2[1], t2[0]), _fsub(t2[2], t2[0]))
    if not any(n1) or not any(n2):
        return False
    e1 = [_fsub(t1[(k + 1) % 3], t1[k]) for k in range(3)]
    e2 = [_fsub(t2[(k + 1) % 3], t2[k]) for k in range(3)]
    axes = [n1, n2] + [_fcross(a, b) for a in e1 for b in e2] + [_fcross(n1, e) for e in e1] + [_fcross(n2, e) for e in e2]
    for ax in axes:
        if not any(ax):
            continue
        p1 = [_fdot(ax, p) for p in t1]
        p2 = [_fdot(ax, p) for p in t2]
        if max(p1) < min(p2) or max(p2) < min(p1):
            return False
    return True


def oracle(t1, t2):
    h, f = C.tri_tri(np.asarray([t1], np.float64), np.asarray([t2], np.float64))
    return bool(h[0]), bool(f[0])


T = [[0.0, 0, 0], [1, 0, 0], [0, 1, 0]]
CASES = {
    'piercing': ([[0.2, 0.2, -1], [0.3, 0.2, 1], [0.2, 0.3, 1]], True),
    'crossing': ([[0.5, -0.5, -0.5], [0.5, 2, -0.5], [0.5, 0.2, 0.7]], True),
    'separated': ([[0, 0, 0.5], [1, 0, 0.5], [0, 1, 0.5]], False),
    'separated_in_plane_of_edge': ([[2, 0, -1], [3, 0, 1], [2, 1, 0]], False),
    'shared_vertex': ([[0, 0, 0], [-1, 0, 1], [0, -1, 1]], True),
    'vertex_on_face': ([[0.25, 0.25, 0], [0.25, 1, 1], [1, 0.25, 1]], True),
    'edge_touching_face': ([[0.25, 0.1, 0], [0.25, 0.6, 0], [0.25, 0.3, 1]], True),
    'edge_touching_edge': ([[0.5, 0.5, -1], [0.5, 0.5, 1], [2, 2, 0]], True),
    'edge_missing_edge': ([[0.6, 0.6, -1], [0.6, 0.6, 1], [2, 2, 0]], False),
    'coplanar_overlapping': ([[0.2, 0.2, 0], [2, 0.2, 0], [0.2, 2, 0]], True),
    'coplanar_contained': ([[0.1, 0.1, 0], [0.3, 0.1, 0], [0.1, 0.3, 0]], True),
    'coplanar_edge_contact': ([[1, 0, 0], [0, 1, 0], [1, 1, 0]], True),
    'coplanar_vertex_contact': ([[1, 0, 0], [2, 0, 0], [2, -1, 0]], True),
    'coplanar_disjoint': ([[0.6, 0.6, 0], [2, 0.6, 0], [0.6, 2, 0]], False),
    'perpendicular_shared_edge': ([[0, 0, 0], [0, 1, 0], [0, 0, 1]], True),
    'zero_area_face': ([[0.2, 0.2, -1], [0.2, 0.2, 0], [0.2, 0.2, 1]], False),
}


@pytest.mark.parametrize('name', sorted(CASES))
def test_hand_built_cases(name):
    other, want = CASES[name]
    assert exact_intersect(T, other) == want
    for a, b in ((T, other), (other, T), (T[::-1], other), (T, [other[1], other[2], other[0]])):
        assert oracle(a, b)[0] == want, (name, a, b)


@pytest.mark.parametrize('dim', [3, 2])
def test_small_integer_triangles_exact(dim):
    """Coordinates in -3..3: every float64 operation is exact, so the predicate must equal the exact test on every pair, touching and
    coplanar ones included (dim 2: both triangles in z = 0)."""
    rng = np.random.default_rng(5 + dim)
    t1 = rng.integers(-3, 4, size=(3000, 3, 3)).astype(np.float64)
    t2 = rng.integers(-3, 4, size=(3000, 3, 3)).astype(np.float64)
    if dim == 2:
        t1[..., 2] = t2[..., 2] = 0
    h, _ = C.tri_tri(t1, t2)
    want = np.array([exact_intersect(a, b) for a, b in zip(t1, t2)])
    assert (h == want).all(), np.nonzero(h != want)[0][:5]
    assert 0.2 < want.mean() < 0.8


def test_near_degenerate_pairs():
    """Random pairs built to sit on or near each other's planes, edges and vertices, at hand scale: the float64 answer may differ from
    the exact one only where the oracle flags the pair as fragile."""
    rng = np.random.default_rng(11)
    n = 3000
    t1 = rng.normal(size=(n, 3, 3)) * 0.02
    t2 = rng.normal(size=(n, 3, 3)) * 0.02
    u, v = rng.random((n, 1)), rng.random((n, 1))
    w = (u + v > 1)[:, 0]
    u[w], v[w] = 1 - u[w], 1 - v[w]
    on = t1[:, 0] + u * (t1[:, 1] - t1[:, 0]) + v * (t1[:, 2] - t1[:, 0])
    kind = np.arange(n) % 4
    t2[kind == 0, 0] = on[kind == 0]                                                       # a vertex on the other face
    t2[kind == 1, 0] = t1[kind == 1, 0]                                                    # a shared vertex
    t2[kind == 2, 0] = on[kind == 2] + rng.normal(size=((kind == 2).sum(), 3)) * 1e-17   # within rounding of the face
    nrm = np.cross(t1[:, 1] - t1[:, 0], t1[:, 2] - t1[:, 0])
    t2[kind == 3] = t1[kind == 3] + 0.3 * (t2[kind == 3] - t2[kind == 3].mean(1, keepdims=True))   # nearly coplanar copies
    t2[kind == 3] += nrm[kind == 3, None] * 1e-16
    h, f = C.tri_tri(t1, t2)
    want = np.array([exact_intersect(a, b) for a, b in zip(t1, t2)])
    bad = (h != want) & ~f
    assert not bad.any(), np.nonzero(bad)[0][:5]
    assert f.sum() < n and want.sum() > 0


def test_oracle_counts_equal_golden():
    g = torch.load(os.path.join(GOLD, 'collision_synth.pt'), weights_only=False)
    xl = g['lv'].double().numpy() + g['left_loc'].numpy()[:, None]
    xr = g['rv'].double().numpy() + g['right_loc'].numpy()[:, None]
    cnt, frag = C.counts(xr, xl, g['faces'].numpy())
    assert cnt.tolist() == g['counts'].tolist()
    assert frag.tolist() == g['fragile'].tolist()
    assert (cnt <= g['max_contacts']).tolist() == g['kept']


def test_valid_judge_oracle_equals_golden():
    g = torch.load(os.path.join(GOLD, 'valid_judge_synth.pt'), weights_only=False)
    for side in ('left', 'right'):
        s = C.valid_scores(g['quat'][side].numpy(), side, *g['converter'][side])
        assert np.abs(s - g['scores'][side].double().numpy()).max() < 2e-5
    assert C.invalid_rate(g['scores']['left'].numpy(), g['scores']['right'].numpy()) == pytest.approx(float(g['rate']))


# ------------------------------------------------------------------------------------------------------------------------ records
def _dict_add_loop(raw, kept):
    """CollisionFilter.py:9-25 restated: copy_dict_struct, then dict_add per kept frame."""
    def struct(d):
        return {k: struct(v) for k, v in d.items()} if isinstance(d, dict) else np.asarray([])

    def add(t, r, i):
        for k in r:
            if isinstance(r[k], dict):
                t[k] = add(t[k], r[k], i)
            else:
                if len(t[k]) == 0:
                    t[k] = r[k][i:i + 1]
                t[k] = np.vstack([t[k], r[k][i:i + 1]])
        return t
    out = struct(raw)
    for i in kept:
        add(out, raw, i)
    return out


def _same(a, b):
    if isinstance(a, dict):
        assert isinstance(b, dict) and list(a) == list(b)
        for k in a:
            _same(a[k], b[k])
    else:
        assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b)


@pytest.mark.parametrize('kept', [[], [3], [0, 2, 3, 6]])
def test_filtered_records(kept):
    rng = np.random.default_rng(0)
    raw = {'right': {'rot': rng.normal(size=(7, 16, 3)), 'loc': rng.normal(size=(7, 3)), 'shape': rng.normal(size=(7, 1, 10))},
           'left': {'rot': rng.normal(size=(7, 16, 3)).astype(np.float32), 'extra': {'id': np.arange(7) * 3}},
           'capture_frame_id': np.arange(7, dtype=np.int64) + 100}
    mask = np.zeros(7, bool)
    mask[kept] = True
    _same(collision.filtered_records(raw, mask), _dict_add_loop(raw, kept))
