"""The renderer's float64 oracle (oracle/render_ref.py) against closed forms, on the CPU: exact lattice counts of one triangle under both
cameras (with pixel centres exactly on an edge), the silhouette area of a closed UV sphere, the depth test, the orthographic camera's
identity with `projection_batch` at S = 256, and the semantics of compute_maskiou's `bm0`."""
from fractions import Fraction

import numpy as np

from oracle import render_ref as R

S = 64


def _lattice_count(P, S):
    """Pixel centres strictly inside the triangle P (3 exact (u, v) Fractions), counted exactly."""
    def edge(a, b, p):
        return (b[0] - a[0]) * (p[1] - a[1]) - (b[1] - a[1]) * (p[0] - a[0])
    n = 0
    for r in range(S):
        for c in range(S):
            p = (Fraction(2 * c + 1, 2), Fraction(2 * r + 1, 2))
            w = [edge(P[1], P[2], p), edge(P[2], P[0], p), edge(P[0], P[1], p)]
            n += all(x > 0 for x in w) or all(x < 0 for x in w)
    return n


# pixel-space vertices: dyadic, so every float64 step of the oracle is exact; the first edge is horizontal through the centres of row 3
TRI_UV = [(Fraction(5, 2), Fraction(7, 2)), (Fraction(61, 2), Fraction(7, 2)), (Fraction(41, 4), Fraction(163, 4))]


def test_triangle_lattice_count_orthographic():
    scale, t = 0.25, (0.125, -0.25)             # u = 16 x + 32 (t + 1)
    a, bu, bv = S * scale, S / 2 * (t[0] + 1), S / 2 * (t[1] + 1)
    verts = np.array([[(float(u) - bu) / a, (float(v) - bv) / a, 0.3] for u, v in TRI_UV])
    cams = R.ortho_cam([scale], [t])
    u, v, _ = R.project(verts, cams[0], False, S)
    assert np.array_equal(u, [float(p[0]) for p in TRI_UV]) and np.array_equal(v, [float(p[1]) for p in TRI_UV])
    fr = R.raster_image(verts, [[0, 1, 2]], cams[0], False, S)
    n = _lattice_count(TRI_UV, S)
    assert n > 300
    assert int((fr['pix_to_face'] >= 0).sum()) == n
    assert not (fr['pix_to_face'][3] >= 0).any()          # centres on the horizontal edge are outside
    assert fr['ambiguous'][3].sum() > 0                  # ... and flagged
    cov = fr['pix_to_face'] >= 0
    assert np.allclose(fr['zbuf'][cov], 10.3) and np.allclose(fr['bary'][cov].sum(-1), 1)
    # reversed winding covers the same pixels (no back-face culling)
    assert np.array_equal(R.raster_image(verts, [[1, 0, 2]], cams[0], False, S)['pix_to_face'] >= 0, cov)


def test_triangle_lattice_count_perspective():
    K = np.array([[[32.0, 0, 24.0], [0, 16.0, 40.0], [0, 0, 1]]])
    z = np.array([2.0, 4.0, 0.5])
    verts = np.array([[(float(u) - 24.0) * zz / 32.0, (float(v) - 40.0) * zz / 16.0, zz] for (u, v), zz in zip(TRI_UV, z)])
    cam = R.persp_cam(K)[0]
    fr = R.raster_image(verts, [[0, 1, 2]], cam, True, S)
    assert int((fr['pix_to_face'] >= 0).sum()) == _lattice_count(TRI_UV, S)
    # perspective-correct barycentrics interpolate 1/z linearly in screen space: zbuf = 1 / sum(b_screen / z)
    cov = np.argwhere(fr['pix_to_face'] >= 0)
    r, c = cov[len(cov) // 2]
    b = fr['bary'][r, c]
    assert np.isclose(fr['zbuf'][r, c], (b * z).sum())
    # a vertex at z <= 0 removes the face
    verts[2, 2] = -0.5
    assert (R.raster_image(verts, [[0, 1, 2]], cam, True, S)['pix_to_face'] < 0).all()


def _uv_sphere(n_lon, n_lat, radius):
    verts = [[0, 0, radius], [0, 0, -radius]]
    for i in range(1, n_lat):
        th = np.pi * i / n_lat
        for j in range(n_lon):
            ph = 2 * np.pi * j / n_lon
            verts.append([radius * np.sin(th) * np.cos(ph), radius * np.sin(th) * np.sin(ph), radius * np.cos(th)])
    ring = lambda i, j: 2 + (i - 1) * n_lon + j % n_lon
    faces = []
    for j in range(n_lon):
        faces.append([0, ring(1, j), ring(1, j + 1)])
        faces.append([1, ring(n_lat - 1, j + 1), ring(n_lat - 1, j)])
        for i in range(1, n_lat - 1):
            faces += [[ring(i, j), ring(i + 1, j), ring(i + 1, j + 1)], [ring(i, j), ring(i + 1, j + 1), ring(i, j + 1)]]
    return np.array(verts), np.array(faces)


def test_sphere_silhouette_area():
    n_lon, n_lat, radius, scale, S2 = 96, 48, 0.4, 0.9, 128
    verts, faces = _uv_sphere(n_lon, n_lat, radius)
    fr = R.raster_image(verts, faces, R.ortho_cam([scale], [[0.03, -0.05]])[0], False, S2)
    Rpx = S2 * scale * radius
    n = int((fr['pix_to_face'] >= 0).sum())
    # the silhouette lies between the inscribed equatorial polygon and the circle; pixel counting adds at most the perimeter
    poly = 0.5 * n_lon * Rpx ** 2 * np.sin(2 * np.pi / n_lon)
    assert poly - 2 * np.pi * Rpx <= n <= np.pi * Rpx ** 2 + 2 * np.pi * Rpx, (n, np.pi * Rpx ** 2)
    assert fr['ambiguous'].mean() < 1e-3


def test_depth_order_swaps_with_z_offsets():
    quad = np.array([[-0.3, -0.3, 0], [0.3, -0.3, 0], [0.3, 0.3, 0], [-0.3, 0.3, 0]])
    faces = np.array([[0, 1, 2], [0, 2, 3], [4, 5, 6], [4, 6, 7]])
    cam = R.ortho_cam([0.5], [[0.0, 0.0]])[0]
    for za, zb, front in ((0.1, 0.2, (0, 1)), (0.2, 0.1, (2, 3))):
        verts = np.concatenate([quad + [0, 0, za], quad * 0.8 + [0.02, 0.01, zb]])
        fr = R.raster_image(verts, faces, cam, False, S)
        inner = R.raster_image(verts[4:], faces[:2], cam, False, S)['pix_to_face'] >= 0
        ok = inner & ~fr['ambiguous']                   # ambiguous: centres on the front quad's diagonal, covered by neither of its faces
        assert ok.sum() > 0.9 * inner.sum()
        assert np.isin(fr['pix_to_face'][ok], front).all()
        assert np.allclose(fr['zbuf'][ok], 10 + min(za, zb))
    # equal depths (up to float64 rounding of the interpolation) are flagged: the kernels resolve fp32 ties by face index
    verts = np.concatenate([quad, quad * 0.8])
    fr = R.raster_image(verts, faces[::-1], cam, False, S)
    inner = R.raster_image(verts[4:], faces[:2], cam, False, S)['pix_to_face'] >= 0
    assert fr['ambiguous'][inner].all()


def test_orthographic_camera_is_projection_batch_at_256():
    rng = np.random.RandomState(0)
    scale, trans2d, v = rng.rand(3) * 3 + 0.5, rng.randn(3, 2) * 0.2, rng.randn(3, 50, 3) * 0.1
    cams = R.ortho_cam(scale, trans2d)
    for b in range(3):
        u, vv, d = R.project(v[b], cams[b], False, 256)
        # utils/manoutils.py:26-44: scale * 256 * xy + (trans2d * 128 + 128)
        ref = (scale[b] * 256) * v[b, :, :2] + (trans2d[b] * 256 / 2 + 256 / 2)
        assert np.allclose(np.stack([u, vv], 1), ref, rtol=0, atol=1e-12)
        assert np.allclose(d, v[b, :, 2] + 10)


def test_bm0_semantics():
    a = np.zeros((8, 8)); b = np.zeros((8, 8))
    assert np.isnan(R.bm0(a, b))
    a[2:5, 2:5] = 1
    assert R.bm0(a, b) == 0 and R.bm0(a, a) == 1
    b[3:6, 3:6] = 1
    assert R.bm0(a, b) == 4 / (9 + 9 - 4)
    # mask_iou over rasterised hands: one triangle against itself and against a disjoint copy
    tri = np.array([[[-0.3, -0.3, 0], [0.3, -0.2, 0], [0.0, 0.3, 0]]])
    cams = R.ortho_cam([0.4, 0.4], [[0, 0], [0, 0]])
    far = tri + [5.0, 0, 0]
    iou, amb, uni = R.mask_iou(np.concatenate([tri, tri]), np.concatenate([tri, far]), [[0, 1, 2]], cams, False, S)
    assert iou[0] == 1 and iou[1] == 0 and uni[0] > 0
    iou, _, uni = R.mask_iou(far, far, [[0, 1, 2]], cams[:1], False, S)
    assert np.isnan(iou[0]) and uni[0] == 0


def test_two_hand_faces_and_orth_map():
    rf = np.array([[0, 1, 2], [3, 4, 5]])
    f = R.two_hand_faces(rf)
    assert f.tolist() == [[1, 0, 2], [4, 3, 5], [778, 779, 780], [781, 782, 783]]
    # the right hand lands where its own camera would put it: S*sl*(s*x + d) + S/2*(tl+1) == S*sr*x + S/2*(tr+1)
    sl, sr, tl, tr = np.array([2.0]), np.array([2.5]), np.array([[0.1, -0.2]]), np.array([[-0.3, 0.05]])
    v = np.random.RandomState(1).randn(1, 10, 3).astype(np.float32) * 0.1
    vr = R.orth_right_into_left(sl, tl, sr, tr, v)
    u_l = np.stack(R.project(vr[0], R.ortho_cam(sl, tl)[0], False, 256)[:2], 1)
    u_r = np.stack(R.project(v[0], R.ortho_cam(sr, tr)[0], False, 256)[:2], 1)
    assert np.allclose(u_l, u_r, atol=1e-4)
